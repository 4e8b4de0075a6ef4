#!/usr/bin/env python
"""Cost of the row panels of SIGLIP_OPT_SIGMA_BUDGET_MIB (bf16, fused step), three arms:

  1. B = 32768, D = 1024, single GPU, where the unbounded step fits: the unbounded step and the panelled step at 2, 4
     and 8 panels, on separate engines, interleaved in blocks in the sustained power state (alternating cancels drift);
  2. B = 131072 single GPU at D = 768 and D = 1024 under a 4 GiB budget (8 panels), where the unbounded sigma operand
     alone would take 32 GiB;
  3. with >= 2 GPUs, W ranks (one process each, NCCL only for the handle exchange) at B = 131072 per rank, D = 1024,
     under a 4 GiB budget. Skipped ("not measured") with one GPU.

Prints per configuration the step time (CUDA events around a block of steps), the loss and gradient kernel time per
step and launch counts (SIGLIP_OPT_KERNEL_TIMING, a separate block), the panel count and workspace_bytes, and the card's
name, power limit and clocks before and after the run.
"""
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi  # noqa: E402

MIB = 1 << 20


def gpu_state() -> str:
    q = "name,power.limit,clocks.sm,clocks.max.sm,temperature.gpu"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def inputs(B, D, dev, seed):
    g = torch.Generator().manual_seed(seed)
    img = torch.nn.functional.normalize(torch.randn(B, D, generator=g)).to(torch.bfloat16).to(dev)
    txt = torch.nn.functional.normalize(torch.randn(B, D, generator=g)).to(torch.bfloat16).to(dev)
    return img, txt


def budget_for_panels(eng, n):
    """Smallest whole-MiB budget that gives exactly n panels (None when no budget does)."""
    lo, hi = 1, 1 << 20
    while lo < hi:
        mid = (lo + hi) // 2
        eng.set_sigma_budget(mid * MIB)
        rows, got, _ = eng.sigma_panels()
        if rows and got <= n:
            hi = mid
        else:
            lo = mid + 1
    eng.set_sigma_budget(lo * MIB)
    return lo * MIB if eng.sigma_panels()[1] == n else None


def measure(eng, img, txt, steps):
    dev = img.device
    tp, bs = torch.tensor([math.log(10.0)], device=dev), torch.tensor([-10.0], device=dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        eng.fwd_bwd(img, txt, tp, bs, torch.bfloat16)
    e1.record()
    torch.cuda.synchronize()
    eng.set_option(_capi.SIGLIP_OPT_KERNEL_TIMING, 1)
    for _ in range(steps):
        eng.fwd_bwd(img, txt, tp, bs, torch.bfloat16)
    lm, ln, gm, gn = eng.kernel_times()
    eng.set_option(_capi.SIGLIP_OPT_KERNEL_TIMING, 0)
    return e0.elapsed_time(e1), lm, ln, gm, gn


def report(tag, eng, acc, base=None):
    t, n, lm, ln, gm, gn = acc
    s = t / n
    rel = f"{100.0 * (s / base - 1.0):+6.1f}%" if base else "      "
    print(f"{tag:28s} panels {eng.sigma_panels()[1]:2d}  step {s:8.3f} ms {rel}  loss {lm / n:7.3f} ms ({ln // n} "
          f"launches)  grad {gm / n:7.3f} ms ({gn // n} launches)  workspace {eng.workspace_bytes / 2**30:6.2f} GiB",
          flush=True)
    return s


def arm_unbounded_vs_panels(dev, steps=10, rounds=3):
    B, D = 32768, 1024
    img, txt = inputs(B, D, dev, 1)
    engines = {"unbounded": SigmoidLossEngine(B, D, dev)}
    for n in (2, 4, 8):
        e = SigmoidLossEngine(B, D, dev)
        if budget_for_panels(e, n) is None:
            print(f"no budget gives {n} panels at B={B}", flush=True)
            e.close()
            continue
        engines[f"{n} panels"] = e
    tp, bs = torch.tensor([math.log(10.0)], device=dev), torch.tensor([-10.0], device=dev)
    for _ in range(10):
        for e in engines.values():
            e.fwd_bwd(img, txt, tp, bs, torch.bfloat16)
    torch.cuda.synchronize()
    acc = {k: [0.0, 0, 0.0, 0, 0.0, 0] for k in engines}
    for _ in range(rounds):
        for k, e in engines.items():
            t, lm, ln, gm, gn = measure(e, img, txt, steps)
            a = acc[k]
            a[0] += t
            a[1] += steps
            a[2] += lm
            a[3] += ln
            a[4] += gm
            a[5] += gn
    print(f"arm 1: B={B} D={D} bf16 single GPU, {rounds} x {steps} steps per configuration, interleaved", flush=True)
    base = None
    for k, e in engines.items():
        s = report(k, e, acc[k], base)
        base = base or s
        e.close()


def arm_large_single(dev, steps=3):
    for D in (768, 1024):
        B = 131072
        img, txt = inputs(B, D, dev, 2)
        e = SigmoidLossEngine(B, D, dev)
        e.set_sigma_budget(4 << 30)
        tp, bs = torch.tensor([math.log(10.0)], device=dev), torch.tensor([-10.0], device=dev)
        e.fwd_bwd(img, txt, tp, bs, torch.bfloat16)
        torch.cuda.synchronize()
        t, lm, ln, gm, gn = measure(e, img, txt, steps)
        print(f"arm 2: B={B} D={D} bf16 single GPU, 4 GiB sigma budget, {steps} steps", flush=True)
        report(f"B={B} D={D}", e, [t, steps, lm, ln, gm, gn])
        e.close()
        del img, txt
        torch.cuda.empty_cache()


def _rank_main(rank, world, path):
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", init_method=f"file://{path}", rank=rank, world_size=world)
    dev = torch.device("cuda", rank)
    B, D, steps = 131072, 1024, 3
    img, txt = inputs(B, D, dev, 10 + rank)
    e = SigmoidLossEngine(B, D, dev)
    e.set_sigma_budget(4 << 30)
    tp, bs = torch.tensor([math.log(10.0)], device=dev), torch.tensor([-10.0], device=dev)
    e.fwd_bwd(img, txt, tp, bs, torch.bfloat16)
    torch.cuda.synchronize()
    dist.barrier()
    t, lm, ln, gm, gn = measure(e, img, txt, steps)
    if rank == 0:
        print(f"arm 3: W={world} ranks, B={B} per rank, D={D}, 4 GiB sigma budget, {steps} steps (rank 0)", flush=True)
        report(f"W={world} B={B}", e, [t, steps, lm, ln, gm, gn])
    dist.barrier()
    e.close()
    dist.destroy_process_group()


def arm_multi_gpu():
    world = torch.cuda.device_count()
    if world < 2:
        print("arm 3: W ranks at B=131072: not measured (one GPU visible)", flush=True)
        return
    import tempfile

    import torch.multiprocessing as mp
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_rank_main, args=(world, os.path.join(d, "store")), nprocs=world, join=True)


def main() -> int:
    dev = torch.device("cuda", 0)
    print("gpu before:", gpu_state(), flush=True)
    arm_unbounded_vs_panels(dev)
    arm_large_single(dev)
    torch.cuda.empty_cache()
    arm_multi_gpu()
    print("gpu after:", gpu_state(), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
