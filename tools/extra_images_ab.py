#!/usr/bin/env python
"""Several images per caption on the single-GPU fused step: B=4096 captions with M=4 images each (16384 images),
D=1024, bf16.

Four arms, one engine each, interleaved in blocks in the sustained power state (alternating to cancel drift):
  (a) repeat   multi_positive with every caption repeated M times: 16384 x 16384 pairs, ids shared by a caption's copies
  (b) extra    extra_images with ids: image 0 paired, images 1..3 as extras carrying their caption's id: 16384 x 4096
               pairs
  (c) hn-img   hard-negative images without ids at the shape of (b)
  (d) plain    the plain step at B=4096 (4096 x 4096 pairs)
Every arm that uses ids sets them before each step (stream copies, part of the step). Prints per arm the step time
(CUDA events around a block of steps), the loss- and gradient-kernel times per launch (SIGLIP_OPT_KERNEL_TIMING, a
separate block), the FLOP-normalised rate 6 R T D / t and the speed-up of each arm over (a), with the card's name,
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
    B, M, D = 4096, 4, 1024
    R = M * B
    steps, rounds = 20, 4
    print("gpu before:", gpu_state(), flush=True)
    g = torch.Generator().manual_seed(1234)
    unit = lambda n: torch.nn.functional.normalize(torch.randn(n, D, generator=g)).to(torch.bfloat16).to(dev)  # noqa
    txt = unit(B)
    # image m of caption i is row m * B + i: a perturbed copy of the caption, so the positives carry weight
    img = torch.nn.functional.normalize(txt.float().repeat(M, 1) + 0.5 * unit(R).float()).to(torch.bfloat16)
    ids = torch.arange(B, device=dev, dtype=torch.int64)
    tp, bs = torch.tensor([math.log(10.0)], device=dev), torch.tensor([-10.0], device=dev)

    def engine(batch, images, sample_ids, extra_ids):
        eng = SigmoidLossEngine(batch, D, dev, images_per_rank=[images] if images != batch else None)
        if sample_ids:
            eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 1)
        if extra_ids:
            eng.set_option(_capi.SIGLIP_OPT_EXTRA_IMAGE_IDS, 1)
        return eng

    arms = [  # name, engine, images, texts, sample ids, extra-image ids
        ("repeat", engine(R, R, True, False), img, txt.repeat(M, 1), ids.repeat(M), None),
        ("extra", engine(B, R, True, True), img, txt, ids, ids.repeat(M - 1)),
        ("hn-img", engine(B, R, False, False), img, txt, None, None),
        ("plain", engine(B, B, False, False), img[:B].contiguous(), txt, None, None),
    ]

    def step(arm):
        _, eng, im, tx, sid, eid = arm
        if sid is not None:
            eng.set_sample_ids(sid)
        if eid is not None:
            eng.set_extra_image_ids(eid)
        eng.fwd_bwd(im, tx, tp, bs, torch.bfloat16)

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
    print(f"B={B} captions x M={M} images (R={R} images), D={D} bf16, fused single-GPU step, {rounds} x {steps} "
          f"steps per arm, interleaved", flush=True)
    print(f"{'arm':8s} {'pairs':>13s} {'step ms':>8s} {'(a)/arm':>8s} {'loss ms':>8s} {'grad ms':>8s} {'TFLOP/s':>8s}")
    base = None
    for name, _, im, tx, _, _ in arms:
        r = acc[name]
        s, lms, gms = r[0] / r[1], r[2] / r[3], r[4] / r[5]
        rows, cols = im.shape[0], tx.shape[0]
        rate = 6.0 * rows * cols * D / (s * 1e-3) / 1e12
        base = s if base is None else base
        print(f"{name:8s} {rows:5d} x {cols:5d} {s:8.3f} {base / s:7.2f}x {lms:8.3f} {gms:8.3f} {rate:8.1f}", flush=True)
    print("gpu after:", gpu_state(), flush=True)
    for a in arms:
        a[1].close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
