#!/usr/bin/env python
"""Cost of the options under distillation on the single-GPU fused step: B=16384, D=D_T=1024, bf16, lambda = 0.5.

Six arms, one engine each, interleaved in blocks in the sustained power state:
  (a) distill       plain distillation: the kModeDistill loss kernel (every arm's engine is created with
                    distill_options=True, siglip_ctx_create_distill_extras)
  (b) +losses       per-sample losses armed every step (kModeDistillOpts)
  (c) +topk5        top-K retrieval, K = 5, armed every step
  (d) +groups       excluded groups, 1000 classes over images and texts
  (e) +sets         label sets, M = 2 (a class and a super-class of 50)
  (f) +neg4096      4096 hard-negative captions with their teacher rows
Every arm sets its teacher (and its per-step options) before each step. Prints per arm the step time (CUDA events around
a block of steps), the loss- and gradient-kernel times (SIGLIP_OPT_KERNEL_TIMING, a separate block) and the ratios to
(a), with the card's name, power limit and clocks read before and after the run.
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
    B, D, DT, K = 16384, 1024, 1024, 4096
    steps, rounds = 20, 4
    print("gpu before:", gpu_state(), flush=True)
    g = torch.Generator().manual_seed(1234)
    unit = lambda n, d=D: torch.nn.functional.normalize(torch.randn(n, d, generator=g)).to(dev)  # noqa: E731
    img = unit(B)
    txt = torch.nn.functional.normalize(img + 0.5 * unit(B)).to(torch.bfloat16)
    neg = unit(K).to(torch.bfloat16)
    img = img.to(torch.bfloat16)
    timg = unit(B, DT)
    ttxt = torch.nn.functional.normalize(timg + 0.5 * unit(B, DT)).to(torch.bfloat16)
    tneg = unit(K, DT).to(torch.bfloat16)
    timg = timg.to(torch.bfloat16)
    ttxt_neg = torch.cat([ttxt, tneg])
    txt_neg = torch.cat([txt, neg])
    tp, bs = torch.tensor([math.log(10.0)], device=dev), torch.tensor([-10.0], device=dev)
    ttp, tbs = torch.tensor([math.log(20.0)], device=dev), torch.tensor([-12.0], device=dev)
    cls = torch.randint(0, 1000, (B,), generator=g).to(dev)
    sets = torch.stack([cls, 1000 + cls % 50], dim=1)
    il, tl = torch.empty(B, device=dev), torch.empty(B, device=dev)
    recall = torch.empty(10, device=dev)

    def engine(texts=None, labels=0):
        eng = SigmoidLossEngine(B, D, dev, teacher_dim=DT, texts_per_rank=texts, labels=labels,
                                distill_options=True)
        eng.set_option(_capi.SIGLIP_OPT_DISTILL, 1)
        return eng

    groups = engine()
    groups.set_option(_capi.SIGLIP_OPT_EXCLUDE_GROUPS, 1)
    labelled = engine(labels=2)
    labelled.set_option(_capi.SIGLIP_OPT_LABEL_SETS, 1)
    arms = [  # name, engine, per-step set-up, texts, teacher texts
        ("distill", engine(), None, txt, ttxt),
        ("+losses", engine(), lambda e: e.request_sample_losses(il, tl), txt, ttxt),
        ("+topk5", engine(), lambda e: e.request_topk(5, recall), txt, ttxt),
        ("+groups", groups, lambda e: e.set_groups(cls, cls), txt, ttxt),
        ("+sets", labelled, lambda e: e.set_label_sets(sets), txt, ttxt),
        ("+neg4096", engine(texts=[B + K]), None, txt_neg, ttxt_neg),
    ]

    def step(arm):
        _, eng, setup, t, tt = arm
        eng.set_teacher(timg, tt, ttp, tbs, 0.5)
        if setup is not None:
            setup(eng)
        eng.fwd_bwd(img, t, tp, bs, torch.bfloat16)

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
    print(f"B={B}, D=D_T={D} bf16, lambda=0.5, fused single-GPU step, {rounds} x {steps} steps per arm, interleaved",
          flush=True)
    print(f"{'arm':9s} {'step ms':>8s} {'arm/(a)':>8s} {'loss ms':>8s} {'arm/(a)':>8s} {'grad ms':>8s} {'arm/(a)':>8s}")
    base = None
    for a in arms:
        r = acc[a[0]]
        s, lms, gms = r[0] / r[1], r[2] / r[3], r[4] / r[5]
        base = (s, lms, gms) if base is None else base
        print(f"{a[0]:9s} {s:8.3f} {s / base[0]:8.3f} {lms:8.3f} {lms / base[1]:8.3f} {gms:8.3f} {gms / base[2]:8.3f}",
              flush=True)
    print("gpu after:", gpu_state(), flush=True)
    for a in arms:
        a[1].close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
