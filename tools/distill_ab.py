#!/usr/bin/env python
"""Cost of distillation from a frozen teacher on the single-GPU fused step: B=16384, D=1024, bf16.

Three arms, one engine each, interleaved in blocks in the sustained power state (alternating to cancel drift):
  (a) plain    no teacher: the default loss kernel
  (b) D_T=1024 distillation (lambda = 0.5) with a teacher of width 1024
  (c) D_T=768  distillation with a teacher of width 768
Every distillation arm sets its teacher before each step. Prints per arm the step time (CUDA events around a block of
steps), the loss- and gradient-kernel times (SIGLIP_OPT_KERNEL_TIMING, a separate block), the ratio to (a) and, for the
loss kernel, the ratio the teacher GEMM's FLOPs predict (1 + D_T / D), with the card's name, power limit and clocks read
before and after the run.
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
    txt = torch.nn.functional.normalize(img.float() + 0.5 * unit(B).float()).to(torch.bfloat16)
    tp, bs = torch.tensor([math.log(10.0)], device=dev), torch.tensor([-10.0], device=dev)
    ttp, tbs = torch.tensor([math.log(20.0)], device=dev), torch.tensor([-12.0], device=dev)

    def teacher(DT):
        # a teacher whose embeddings are correlated with the student's pairs: the usual soft-target regime
        tu = lambda n: torch.nn.functional.normalize(torch.randn(n, DT, generator=g)).to(dev)  # noqa: E731
        ti = tu(B)
        tt = torch.nn.functional.normalize(ti + 0.5 * tu(B))
        return ti.to(torch.bfloat16), tt.to(torch.bfloat16)

    def engine(DT):
        eng = SigmoidLossEngine(B, D, dev, teacher_dim=DT)
        if DT:
            eng.set_option(_capi.SIGLIP_OPT_DISTILL, 1)
        return eng

    arms = [  # name, engine, teacher (images, texts) or None, D_T
        ("plain", engine(0), None, 0),
        ("D_T=1024", engine(1024), teacher(1024), 1024),
        ("D_T=768", engine(768), teacher(768), 768),
    ]

    def step(arm):
        _, eng, t, _ = arm
        if t is not None:
            eng.set_teacher(t[0], t[1], ttp, tbs, 0.5)
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
    print(f"B={B}, D={D} bf16, fused single-GPU step, {rounds} x {steps} steps per arm, interleaved", flush=True)
    print(f"{'arm':8s} {'step ms':>8s} {'arm/(a)':>8s} {'loss ms':>8s} {'arm/(a)':>8s} {'predict':>8s} {'grad ms':>8s} "
          f"{'arm/(a)':>8s}")
    base = None
    for name, _, _, DT in arms:
        r = acc[name]
        s, lms, gms = r[0] / r[1], r[2] / r[3], r[4] / r[5]
        base = (s, lms, gms) if base is None else base
        print(f"{name:8s} {s:8.3f} {s / base[0]:8.3f} {lms:8.3f} {lms / base[1]:8.3f} {1 + DT / D:8.3f} {gms:8.3f} "
              f"{gms / base[2]:8.3f}", flush=True)
    print("gpu after:", gpu_state(), flush=True)
    for a in arms:
        a[1].close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
