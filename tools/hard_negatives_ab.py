#!/usr/bin/env python
"""Cost of hard-negative captions on the single-GPU fused step at B=16384, D=1024, bf16.

Three arms, one engine each, interleaved in blocks in the sustained power state (alternating to cancel drift):
  plain   siglip_ctx_create, T = B
  K=4096  siglip_ctx_create_texts, T = B + 4096
  K=16384 one hard negative per image, T = 2 B
Prints per arm the step time (CUDA events around a block of steps), the loss- and gradient-kernel times
(SIGLIP_OPT_KERNEL_TIMING, a separate block), and the FLOP-normalised rate 6 B T D / t (the three contractions of the
step: logits, dimg, dtxt), with the card's name, power limit and clocks read before and after the run.
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
    steps, rounds = 20, 4
    print("gpu before:", gpu_state(), flush=True)
    g = torch.Generator().manual_seed(1234)
    unit = lambda n: torch.nn.functional.normalize(torch.randn(n, D, generator=g)).to(torch.bfloat16).to(dev)  # noqa
    img = unit(B)
    txt_all = unit(2 * B)                     # paired captions, then up to B hard negatives
    tp, bs = torch.tensor([math.log(10.0)], device=dev), torch.tensor([-10.0], device=dev)
    arms = []
    for K in (0, 4096, 16384):
        eng = SigmoidLossEngine(B, D, dev, texts_per_rank=[B + K] if K else None)
        arms.append((K, eng, txt_all[:B + K].contiguous()))

    def step(arm):
        _, eng, txt = arm
        eng.fwd_bwd(img, txt, tp, bs, torch.bfloat16)

    for _ in range(30):                       # sustained power state, every arm warmed up
        for a in arms:
            step(a)
    torch.cuda.synchronize()
    acc = {a[0]: [0.0, 0, 0.0, 0, 0.0, 0] for a in arms}
    for _ in range(rounds):
        for a in arms:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                step(a)
            e1.record()
            torch.cuda.synchronize()
            eng = a[1]
            eng.set_option(_capi.SIGLIP_OPT_KERNEL_TIMING, 1)
            for _ in range(steps):
                step(a)
            lm, ln, gm, gn = eng.kernel_times()
            eng.set_option(_capi.SIGLIP_OPT_KERNEL_TIMING, 0)
            r = acc[a[0]]
            r[0] += e0.elapsed_time(e1)
            r[1] += steps
            r[2] += lm
            r[3] += ln
            r[4] += gm
            r[5] += gn
    print(f"B={B} D={D} bf16, fused single-GPU step, {rounds} x {steps} steps per arm, interleaved", flush=True)
    print(f"{'arm':8s} {'T':>6s} {'step ms':>8s} {'vs plain':>8s} {'loss ms':>8s} {'grad ms':>8s} {'TFLOP/s':>8s}")
    base = None
    for K, _, _ in arms:
        r = acc[K]
        s, lms, gms = r[0] / r[1], r[2] / r[3], r[4] / r[5]
        T = B + K
        rate = 6.0 * B * T * D / (s * 1e-3) / 1e12
        base = s if base is None else base
        name = "plain" if K == 0 else f"K={K}"
        print(f"{name:8s} {T:6d} {s:8.3f} {100.0 * (s / base - 1.0):+7.1f}% {lms:8.3f} {gms:8.3f} {rate:8.1f}",
              flush=True)
    print("gpu after:", gpu_state(), flush=True)
    for _, eng, _ in arms:
        eng.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
