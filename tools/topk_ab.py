#!/usr/bin/env python
"""Cost of the top-K retrieval (siglip_request_topk) at B=16384, D=1024, bf16, single GPU.

Four arms on one engine, interleaved in blocks in the sustained power state (alternating to cancel drift):
  off      plain steps
  top1     every step armed with the top-1 retrieval metrics (siglip_request_metrics)
  k5       every step armed with top-K, K = 5
  k10      every step armed with top-K, K = 10
for the fused step and the no-grad forward. Prints per arm the step time (CUDA events around a block of steps) and the
loss-kernel time (SIGLIP_OPT_KERNEL_TIMING, a separate block), the finalisation kernel's time (torch.profiler), and the
card's name, power limit and clocks before, during (with unarmed steps queued) and after the run.
"""
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi  # noqa: E402

ARMS = ("off", "top1", "k5", "k10")


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
    steps, rounds = 20, 4
    print("gpu before:", gpu_state(), flush=True)
    g = torch.Generator().manual_seed(1234)
    img = torch.nn.functional.normalize(torch.randn(B, D, generator=g)).to(torch.bfloat16).to(dev)
    txt = torch.nn.functional.normalize(torch.randn(B, D, generator=g)).to(torch.bfloat16).to(dev)
    tp, bs = torch.tensor([math.log(10.0)], device=dev), torch.tensor([-10.0], device=dev)
    eng = SigmoidLossEngine(B, D, dev)
    top1 = torch.empty(2, device=dev)
    i2t = torch.empty(B, device=dev, dtype=torch.int64)
    t2i = torch.empty(B, device=dev, dtype=torch.int64)
    recall = torch.empty(20, device=dev)
    i2t_k = torch.empty(B * 10, device=dev, dtype=torch.int64)
    t2i_k = torch.empty(B * 10, device=dev, dtype=torch.int64)

    def step(kind, arm):
        if arm == "top1":
            eng.request_metrics(top1, i2t, t2i)
        elif arm != "off":
            k = int(arm[1:])
            eng.request_topk(k, recall[:2 * k], i2t_k[:B * k].view(B, k), t2i_k[:B * k].view(B, k))
        if kind == "fused":
            eng.fwd_bwd(img, txt, tp, bs, torch.bfloat16)
        else:
            eng.fwd(img, txt, tp, bs)

    for kind in ("fused", "fwd"):
        for _ in range(40):                 # sustained power state, every arm warmed up
            for arm in ARMS:
                step(kind, arm)
        torch.cuda.synchronize()
        acc = {arm: [0.0, 0, 0.0, 0] for arm in ARMS}
        for _ in range(rounds):
            for arm in ARMS:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(steps):
                    step(kind, arm)
                e1.record()
                torch.cuda.synchronize()
                eng.set_option(_capi.SIGLIP_OPT_KERNEL_TIMING, 1)
                for _ in range(steps):
                    step(kind, arm)
                lm, ln, _, _ = eng.kernel_times()
                eng.set_option(_capi.SIGLIP_OPT_KERNEL_TIMING, 0)
                a = acc[arm]
                a[0] += e0.elapsed_time(e1)
                a[1] += steps
                a[2] += lm
                a[3] += ln
        for _ in range(300):                # 0.3 to 0.9 s of unarmed steps queued: the card's state under load
            step(kind, "off")
        under = gpu_state()
        torch.cuda.synchronize()
        s0, l0 = acc["off"][0] / acc["off"][1], acc["off"][2] / acc["off"][3]
        print(f"B={B} D={D} bf16, {kind} single-GPU step, {rounds} x {steps} steps per arm, interleaved", flush=True)
        print(f"gpu under load (name, power limit, SM clock, max SM clock, temperature): {under}", flush=True)
        print(f"{'arm':8s} {'step ms':>8s} {'vs off':>7s} {'loss ms':>8s} {'vs off':>7s}")
        for arm in ARMS:
            a = acc[arm]
            s, lk = a[0] / a[1], a[2] / a[3]
            print(f"{arm:8s} {s:8.3f} {100.0 * (s / s0 - 1.0):+6.1f}% {lk:8.3f} {100.0 * (lk / l0 - 1.0):+6.1f}%",
                  flush=True)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step("fused", "k10")
        torch.cuda.synchronize()
    for ev in prof.key_averages():
        if "topk_finalize" in ev.key or "memset" in ev.key.lower():
            print(f"armed step extra: {ev.key[:60]} {ev.device_time_total / ev.count:.1f} us", flush=True)
    print("gpu after:", gpu_state(), flush=True)
    eng.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
