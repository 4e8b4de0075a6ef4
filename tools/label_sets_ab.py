#!/usr/bin/env python
"""Cost of multi-label positives (SIGLIP_OPT_LABEL_SETS) on the single-GPU fused step at B=16384, D=1024, bf16.

Five arms, interleaved in blocks in the sustained power state (same process, same GPU, alternating to cancel drift):
  off      no labels: positional pairs only
  ids      multi_positive sample ids from 1000 classes (SIGLIP_OPT_SAMPLE_IDS)
  m1       label sets with M = 1 holding the same 1000 classes: the same positives as ids
  tree4    M = 4, a 4-level hierarchy: leaf class c of 1000, then 1000 + c // 10, 2000 + c // 100, 3000 + c // 250
  tags4    M = 4 random tags of 1000 per sample, 30 % of the slots empty
Prints per arm the step time (CUDA events around a block of steps, every step including its label copies), the loss-
and gradient-kernel times (SIGLIP_OPT_KERNEL_TIMING, a separate block, per launch), the share of 16 x 32 warp slabs of
the own chunk that hold a positive off the diagonal, and the card's name, power limit and clocks read before and after.
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


def slab_share(sets: torch.Tensor) -> float:
    """Share of 16 x 32 warp slabs of the own-chunk B x B tile grid holding a positive off the diagonal (two sets that
    share a label >= 0), computed in row blocks on the device."""
    B, M = sets.shape
    hit = 0
    for r0 in range(0, B, 1024):
        a = sets[r0:r0 + 1024]
        pos = torch.zeros(a.shape[0], B, dtype=torch.bool, device=sets.device)
        for p in range(M):
            for q in range(M):
                pos |= (a[:, p, None] == sets[None, :, q]) & (a[:, p, None] >= 0)
        pos[torch.arange(a.shape[0]), torch.arange(r0, r0 + a.shape[0])] = False
        hit += int(pos.reshape(a.shape[0] // 16, 16, B // 32, 32).any(dim=3).any(dim=1).sum())
    return hit / ((B // 16) * (B // 32))


def main() -> int:
    dev = torch.device("cuda", 0)
    B, D = 16384, 1024
    steps, rounds = 30, 4
    print("gpu before:", gpu_state(), flush=True)
    g = torch.Generator().manual_seed(1234)
    img = torch.nn.functional.normalize(torch.randn(B, D, generator=g)).to(torch.bfloat16).to(dev)
    txt = torch.nn.functional.normalize(torch.randn(B, D, generator=g)).to(torch.bfloat16).to(dev)
    tp, bs = torch.tensor([math.log(10.0)], device=dev), torch.tensor([-10.0], device=dev)
    classes = torch.randint(0, 1000, (B,), generator=g)
    tree = torch.stack([classes, 1000 + classes // 10, 2000 + classes // 100, 3000 + classes // 250], dim=1)
    tags = torch.randint(0, 1000, (B, 4), generator=g)
    tags[torch.rand(B, 4, generator=g) < 0.3] = -1
    arms = {"off": None, "ids": classes, "m1": classes[:, None].contiguous(), "tree4": tree, "tags4": tags}
    arms = {k: (None if v is None else v.to(dev)) for k, v in arms.items()}
    engines = {}
    for name, lab in arms.items():
        if name in ("m1", "tree4", "tags4"):
            eng = SigmoidLossEngine(B, D, dev, labels=lab.shape[1])
            eng.set_option(_capi.SIGLIP_OPT_LABEL_SETS, 1)
        else:
            eng = SigmoidLossEngine(B, D, dev)
            if name == "ids":
                eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 1)
        engines[name] = eng

    def step(name):
        eng = engines[name]
        if name == "ids":
            eng.set_sample_ids(arms[name])
        elif arms[name] is not None:
            eng.set_label_sets(arms[name])
        eng.fwd_bwd(img, txt, tp, bs, torch.bfloat16)

    for _ in range(100):                 # sustained power state, every arm warmed up
        for name in arms:
            step(name)
    torch.cuda.synchronize()
    acc = {name: [0.0, 0, 0.0, 0, 0.0, 0] for name in arms}
    for _ in range(rounds):
        for name in arms:
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
    print(f"{'arm':8s} {'step ms':>8s} {'vs off':>7s} {'loss ms':>8s} {'grad ms':>8s} {'slabs w/ positive':>18s}")
    for name, lab in arms.items():
        a = acc[name]
        st = a[0] / a[1]
        share = 0.0 if lab is None else slab_share(lab if lab.dim() == 2 else lab[:, None])
        print(f"{name:8s} {st:8.3f} {100.0 * (st / base - 1.0):+6.1f}% {a[2] / a[3]:8.3f} {a[4] / a[5]:8.3f} "
              f"{100.0 * share:17.1f}%", flush=True)
    print("gpu after:", gpu_state(), flush=True)
    for eng in engines.values():
        eng.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
