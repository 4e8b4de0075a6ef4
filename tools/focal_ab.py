#!/usr/bin/env python
"""Cost of the focal pair loss (SIGLIP_OPT_FOCAL) on the single-GPU fused step at B=16384, D=1024, bf16.

Four arms, interleaved in blocks in the sustained power state (same process, same GPU; the order of the arms rotates
from round to round, so that each arm takes each position once):
  off        the SigLIP step (kModeLoss)
  g0         focal with gamma = 0, no alpha: the SigLIP terms through the kModeFocal kernel
  g2a25      focal with gamma = 2, alpha = 0.25
  g2a25+sl   the same with per-sample losses requested every step
Prints per arm the step time (CUDA events around a block of steps), the loss- and gradient-kernel times
(SIGLIP_OPT_KERNEL_TIMING, a separate block, per launch), and the card's name, power limit and clocks read before and
after.
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
    arms = {"off": None, "g0": (0.0, None), "g2a25": (2.0, 0.25), "g2a25+sl": (2.0, 0.25)}
    engines = {}
    for name, focal in arms.items():
        eng = SigmoidLossEngine(B, D, dev)
        if focal is not None:
            eng.set_option(_capi.SIGLIP_OPT_FOCAL, 1)
            eng.set_focal(*focal)
        engines[name] = eng
    il = torch.empty(B, device=dev)
    tl = torch.empty(B, device=dev)

    def step(name):
        eng = engines[name]
        if name.endswith("+sl"):
            eng.request_sample_losses(il, tl)
        eng.fwd_bwd(img, txt, tp, bs, torch.bfloat16)

    for _ in range(100):                 # sustained power state, every arm warmed up
        for name in arms:
            step(name)
    torch.cuda.synchronize()
    acc = {name: [0.0, 0, 0.0, 0, 0.0, 0] for name in arms}
    names = list(arms)
    for rnd in range(rounds):
        for name in names[rnd % len(names):] + names[:rnd % len(names)]:
            eng = engines[name]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                step(name)
            e1.record()
            torch.cuda.synchronize()
            eng.set_option(_capi.SIGLIP_OPT_KERNEL_TIMING, 1)
            for _ in range(steps):
                step(name)
            lm, ln, gm, gn = eng.kernel_times()
            eng.set_option(_capi.SIGLIP_OPT_KERNEL_TIMING, 0)
            a = acc[name]
            a[0] += e0.elapsed_time(e1)
            a[1] += steps
            a[2] += lm
            a[3] += ln
            a[4] += gm
            a[5] += gn
    base = acc["off"][0] / acc["off"][1]
    print(f"B={B} D={D} bf16, fused single-GPU step, {rounds} x {steps} steps per arm", flush=True)
    print(f"{'arm':10s} {'step ms':>8s} {'vs off':>7s} {'loss ms':>8s} {'grad ms':>8s}")
    for name in arms:
        a = acc[name]
        st = a[0] / a[1]
        print(f"{name:10s} {st:8.3f} {100.0 * (st / base - 1.0):+6.1f}% {a[2] / a[3]:8.3f} {a[4] / a[5]:8.3f}",
              flush=True)
    print("gpu after:", gpu_state(), flush=True)
    for eng in engines.values():
        eng.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
