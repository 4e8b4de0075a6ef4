#!/usr/bin/env python
"""Cost of excluded same-group pairs (SIGLIP_OPT_EXCLUDE_GROUPS) on the single-GPU fused step at B=16384, D=1024, bf16.

Five arms, interleaved in blocks in the sustained power state (same process, same GPU, alternating to cancel drift):
  off       the option off
  unique    groups on, every group distinct: no pair is excluded, so the cost is the per-slab group comparisons alone
  classes   groups on, 1000 classes drawn at random (class-label captions: ~1/1000 of the pairs excluded)
  dups1     groups on, 1 % of the samples in near-duplicate pairs (a dedup cluster of two), the rest without a group
  ids       groups as in classes, together with multi-positive sample ids (unique ids)
Prints per arm the step time (CUDA events around a block of steps, every step including its siglip_set_groups
copies), the loss- and gradient-kernel times (SIGLIP_OPT_KERNEL_TIMING, a separate block), the share of 16 x 32 warp
slabs of the own chunk that hold an excluded pair, and the card's name, power limit and clocks read before and after.
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


def slab_share(groups: torch.Tensor) -> float:
    """Share of 16 x 32 warp slabs of the own-chunk B x B tile grid holding an excluded pair (same group >= 0, off the
    diagonal)."""
    B = groups.shape[0]
    m = (groups[:, None] == groups[None, :]) & (groups[:, None] >= 0)
    m.fill_diagonal_(False)
    return float(m.reshape(B // 16, 16, B // 32, 32).any(dim=3).any(dim=1).float().mean())


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
    dups = torch.full((B,), -1, dtype=torch.int64)
    pick = torch.randperm(B, generator=g)[: B // 100]
    dups[pick] = torch.arange(pick.numel()) // 2          # pairs of near-duplicates at random positions
    arms = {"off": None, "unique": torch.randperm(B, generator=g), "classes": classes, "dups1": dups, "ids": classes}
    arms = {k: (None if v is None else v.to(dev)) for k, v in arms.items()}
    ids = torch.arange(B, device=dev)
    engines = {}
    for name, grp in arms.items():
        eng = SigmoidLossEngine(B, D, dev)
        if grp is not None:
            eng.set_option(_capi.SIGLIP_OPT_EXCLUDE_GROUPS, 1)
        if name == "ids":
            eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 1)
        engines[name] = eng

    def step(name):
        eng = engines[name]
        if name == "ids":
            eng.set_sample_ids(ids)
        if arms[name] is not None:
            eng.set_groups(arms[name], arms[name])
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
    print(f"{'arm':8s} {'step ms':>8s} {'vs off':>7s} {'loss ms':>8s} {'grad ms':>8s} {'slabs w/ excluded':>18s}")
    for name, grp in arms.items():
        a = acc[name]
        st = a[0] / a[1]
        share = 0.0 if grp is None else slab_share(grp.cpu())
        print(f"{name:8s} {st:8.3f} {100.0 * (st / base - 1.0):+6.1f}% {a[2] / a[3]:8.3f} {a[4] / a[5]:8.3f} "
              f"{100.0 * share:17.1f}%", flush=True)
    print("gpu after:", gpu_state(), flush=True)
    for eng in engines.values():
        eng.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
