#!/usr/bin/env python
"""Several captions per image on the single-GPU fused step: B=4096 images with M=4 captions each (16384 texts),
D=1024, bf16.

Four arms, one engine each, interleaved in blocks in the sustained power state (alternating to cancel drift):
  (a) repeat   multi_positive with every image repeated M times: 16384 x 16384 pairs, ids shared by an image's copies
  (b) extra    extra_texts: caption 0 paired, captions 1..3 as extras carrying their image's id: 4096 x 16384 pairs
  (c) hn+ids   hard negatives + sample ids at the shape of (b): the same kernels, no extra ever matches (what the
               matches cost)
  (d) hn       hard negatives without ids, same shape
Every arm that uses ids sets them before each step (stream copies, part of the step). Prints per arm the step time
(CUDA events around a block of steps), the loss- and gradient-kernel times (SIGLIP_OPT_KERNEL_TIMING, a separate
block), the FLOP-normalised rate 6 B T D / t and the speed-up of each arm over (a), with the card's name, power limit
and clocks read before and after the run.
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
    B, M, D = 4096, 4, 1024
    T = M * B
    steps, rounds = 20, 4
    print("gpu before:", gpu_state(), flush=True)
    g = torch.Generator().manual_seed(1234)
    unit = lambda n: torch.nn.functional.normalize(torch.randn(n, D, generator=g)).to(torch.bfloat16).to(dev)  # noqa
    img = unit(B)
    # caption m of image i is row m * B + i: a perturbed copy of the image, so the positives carry weight
    txt = torch.nn.functional.normalize(img.float().repeat(M, 1) + 0.5 * unit(T).float()).to(torch.bfloat16)
    ids = torch.arange(B, device=dev, dtype=torch.int64)
    tp, bs = torch.tensor([math.log(10.0)], device=dev), torch.tensor([-10.0], device=dev)

    def engine(batch, texts, sample_ids, extra_ids):
        eng = SigmoidLossEngine(batch, D, dev, texts_per_rank=[texts] if texts != batch else None)
        if sample_ids:
            eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 1)
        if extra_ids:
            eng.set_option(_capi.SIGLIP_OPT_EXTRA_TEXT_IDS, 1)
        return eng

    arms = [  # name, engine, images, sample ids, extra ids
        ("repeat", engine(T, T, True, False), img.repeat(M, 1), ids.repeat(M), None),
        ("extra", engine(B, T, True, True), img, ids, ids.repeat(M - 1)),
        ("hn+ids", engine(B, T, True, False), img, ids, None),
        ("hn", engine(B, T, False, False), img, None, None),
    ]

    def step(arm):
        _, eng, im, sid, eid = arm
        if sid is not None:
            eng.set_sample_ids(sid)
        if eid is not None:
            eng.set_extra_text_ids(eid)
        eng.fwd_bwd(im, txt, tp, bs, torch.bfloat16)

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
    print(f"B={B} images x M={M} captions (T={T} texts), D={D} bf16, fused single-GPU step, {rounds} x {steps} steps "
          f"per arm, interleaved", flush=True)
    print(f"{'arm':8s} {'pairs':>13s} {'step ms':>8s} {'(a)/arm':>8s} {'loss ms':>8s} {'grad ms':>8s} {'TFLOP/s':>8s}")
    base = None
    for name, _, im, _, _ in arms:
        r = acc[name]
        s, lms, gms = r[0] / r[1], r[2] / r[3], r[4] / r[5]
        rows = im.shape[0]
        rate = 6.0 * rows * T * D / (s * 1e-3) / 1e12
        base = s if base is None else base
        print(f"{name:8s} {rows:5d} x {T:5d} {s:8.3f} {base / s:7.2f}x {lms:8.3f} {gms:8.3f} {rate:8.1f}", flush=True)
    print("gpu after:", gpu_state(), flush=True)
    for a in arms:
        a[1].close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
