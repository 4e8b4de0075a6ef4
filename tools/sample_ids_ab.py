#!/usr/bin/env python
"""Cost of multi-positive labels (SIGLIP_OPT_SAMPLE_IDS) on the single-GPU fused step at B=16384, D=1024, bf16.

Four arms, interleaved in blocks in the sustained power state (same process, same GPU, alternating to cancel drift):
  off       positional labels (the option off)
  unique    ids on, every id distinct: the same labels, so the cost is the per-slab id comparisons alone
  classes   ids on, 1000 classes drawn at random (~40 % of the 16x32 warp slabs hold an off-diagonal positive)
  groups4   ids on, groups of 4 consecutive duplicates
Prints per arm the step time (CUDA events around a block of steps, every step including its siglip_set_sample_ids
copy), the loss- and gradient-kernel times (SIGLIP_OPT_KERNEL_TIMING, a separate block), the share of warp slabs the
ids send to the general path, and the card's name, power limit and clocks read before and after the run.
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


def slab_share(ids: torch.Tensor) -> float:
    """Share of 16 x 32 warp slabs of the own-chunk B x B tile grid holding a positive other than the diagonal."""
    B = ids.shape[0]
    m = ids[:, None] == ids[None, :]
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
    arms = {
        "off": None,
        "unique": ((torch.randperm(B, generator=g) - B // 2) * 8589934597).to(dev),
        "classes": torch.randint(0, 1000, (B,), generator=g).to(dev),
        "groups4": (torch.arange(B) // 4).to(dev),
    }
    engines = {}
    for name, ids in arms.items():
        eng = SigmoidLossEngine(B, D, dev)
        if ids is not None:
            eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 1)
        engines[name] = eng

    def step(name):
        if arms[name] is not None:
            engines[name].set_sample_ids(arms[name])
        engines[name].fwd_bwd(img, txt, tp, bs, torch.bfloat16)

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
    print(f"{'arm':8s} {'step ms':>8s} {'vs off':>7s} {'loss ms':>8s} {'grad ms':>8s} {'slabs w/ off-diag +':>20s}")
    for name, ids in arms.items():
        a = acc[name]
        st = a[0] / a[1]
        share = 0.0 if ids is None else slab_share(ids)
        print(f"{name:8s} {st:8.3f} {100.0 * (st / base - 1.0):+6.1f}% {a[2] / a[3]:8.3f} {a[4] / a[5]:8.3f} "
              f"{100.0 * share:19.1f}%", flush=True)
    print("gpu after:", gpu_state(), flush=True)
    for eng in engines.values():
        eng.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
