#!/usr/bin/env python
"""Cost of the in-batch retrieval metrics (siglip_request_metrics) on the single-GPU fused step at B=16384, D=1024, bf16.

Two arms on one engine, interleaved in blocks in the sustained power state (alternating to cancel drift):
  off   plain steps
  on    every step armed with top-1 rates and both index vectors
Prints per arm the step time (CUDA events around a block of steps), the loss-kernel time (SIGLIP_OPT_KERNEL_TIMING, a
separate block), and for the armed arm the memset and finalisation kernel times (torch.profiler), with the card's name,
power limit and clocks read before and after the run.
"""
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi  # noqa: E402


def gpu_state() -> str:
    q = "name,power.limit,clocks.sm,clocks.max.sm,temperature.gpu"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def main() -> int:
    dev = torch.device("cuda", 0)
    B, D = 16384, 1024
    steps, rounds = 30, 4
    print("gpu before:", gpu_state(), flush=True)
    g = torch.Generator().manual_seed(1234)
    img = torch.nn.functional.normalize(torch.randn(B, D, generator=g)).to(torch.bfloat16).to(dev)
    txt = torch.nn.functional.normalize(torch.randn(B, D, generator=g)).to(torch.bfloat16).to(dev)
    tp, bs = torch.tensor([math.log(10.0)], device=dev), torch.tensor([-10.0], device=dev)
    eng = SigmoidLossEngine(B, D, dev)
    top1 = torch.empty(2, device=dev)
    i2t = torch.empty(B, device=dev, dtype=torch.int64)
    t2i = torch.empty(B, device=dev, dtype=torch.int64)

    def step(on):
        if on:
            eng.request_metrics(top1, i2t, t2i)
        eng.fwd_bwd(img, txt, tp, bs, torch.bfloat16)

    for _ in range(100):                 # sustained power state, both arms warmed up
        step(False)
        step(True)
    torch.cuda.synchronize()
    acc = {arm: [0.0, 0, 0.0, 0] for arm in (False, True)}
    for _ in range(rounds):
        for arm in (False, True):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                step(arm)
            e1.record()
            torch.cuda.synchronize()
            eng.set_option(_capi.SIGLIP_OPT_KERNEL_TIMING, 1)
            for _ in range(steps):
                step(arm)
            lm, ln, _, _ = eng.kernel_times()
            eng.set_option(_capi.SIGLIP_OPT_KERNEL_TIMING, 0)
            a = acc[arm]
            a[0] += e0.elapsed_time(e1)
            a[1] += steps
            a[2] += lm
            a[3] += ln
    # memset + finalisation of an armed step, from the profiler's kernel records
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step(True)
        torch.cuda.synchronize()
    fin_us = mem_us = 0.0
    for ev in prof.key_averages():
        if "metrics_finalize" in ev.key:
            fin_us = ev.device_time_total / ev.count
        elif "memset" in ev.key.lower():
            mem_us = ev.device_time_total / ev.count
    a0, a1 = acc[False], acc[True]
    s0, s1 = a0[0] / a0[1], a1[0] / a1[1]
    l0, l1 = a0[2] / a0[3], a1[2] / a1[3]
    print(f"B={B} D={D} bf16, fused single-GPU step, {rounds} x {steps} steps per arm", flush=True)
    print(f"{'arm':5s} {'step ms':>8s} {'vs off':>7s} {'loss ms':>8s} {'vs off':>7s}")
    print(f"{'off':5s} {s0:8.3f} {'':>7s} {l0:8.3f}")
    print(f"{'on':5s} {s1:8.3f} {100.0 * (s1 / s0 - 1.0):+6.1f}% {l1:8.3f} {100.0 * (l1 / l0 - 1.0):+6.1f}%")
    print(f"armed step extras: finalisation kernel {fin_us:.1f} us, key memset {mem_us:.1f} us", flush=True)
    print("gpu after:", gpu_state(), flush=True)
    eng.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
