#!/usr/bin/env python
"""Cost of a group that spans nodes, on one host with two or more GPUs, one process per GPU:

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29721 \
        tools/cross_node_ab.py [--batch 16384] [--dim 1024] [--steps 20] [--warmup 5]

Times the same global batch (bf16, B per rank, forward + backward through DDPSigmoidLoss) as one node of P GPUs
(ranks_per_node = P: the in-kernel exchange alone) and as P "nodes" of one GPU (ranks_per_node = 1: every remote text
arrives through the all-to-all), alternating the two, and times the forward all-to-all of the texts and the backward
one of their gradients on their own. The exchange here runs over NVLink, not InfiniBand, so this is a lower bound on
the cost of real nodes. Prints one JSON line on rank 0 with the card's name and power limit."""
from __future__ import annotations

import argparse
import datetime
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from distributed_sigmoid_loss_b200 import DDPSigmoidLoss  # noqa: E402
from distributed_sigmoid_loss_b200.cross_node import Topology, return_rows, send_rows  # noqa: E402


def timed(fn, steps: int, warmup: int) -> float:
    """Median ms of fn over `steps` calls, CUDA events around each, a barrier before each."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(steps):
        dist.barrier()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return sorted(ms)[len(ms) // 2]


def card() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        name, power = [x.strip() for x in q.strip().split(",")]
        return dict(gpu=name, power_limit=power)
    except Exception as e:  # the timing stands without it, but say so
        return dict(gpu=torch.cuda.get_device_name(), power_limit=f"unknown ({e})")


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16384)
    ap.add_argument("--dim", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    dist.init_process_group("nccl", timeout=datetime.timedelta(seconds=300))
    rank, world = dist.get_rank(), dist.get_world_size()
    if world < 2:
        raise SystemExit("needs two or more GPUs")
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", rank)))
    torch.cuda.set_device(dev)
    B, D = args.batch, args.dim
    g = torch.Generator(device=dev).manual_seed(1 + rank)
    img = torch.nn.functional.normalize(torch.randn(B, D, device=dev, generator=g)).bfloat16().requires_grad_(True)
    txt = torch.nn.functional.normalize(torch.randn(B, D, device=dev, generator=g)).bfloat16().requires_grad_(True)
    mods = {L: DDPSigmoidLoss(B, ranks_per_node=L).to(dev) for L in (world, 1)}

    def step(L):
        def run():
            img.grad = txt.grad = None
            mods[L](img, txt).backward()
        return run

    for L in mods:   # build both engines before timing
        step(L)()
    res = {}
    for _ in range(2):   # alternate the two configurations
        for L in mods:
            res.setdefault(L, []).append(timed(step(L), args.steps, args.warmup))
    topo = Topology(rank, world, 1)
    tpr = [B] * world
    rows = txt.detach()
    remote = torch.zeros((world - 1) * B, D, device=dev, dtype=torch.bfloat16)
    fwd_ms = timed(lambda: send_rows(rows, topo, tpr, None), args.steps, args.warmup)
    bwd_ms = timed(lambda: return_rows(remote, rows, topo, tpr, None), args.steps, args.warmup)
    if rank == 0:
        out = dict(metric="cross_node_step_ms", batch_per_rank=B, dim=D, ranks=world,
                   one_node_step_ms=min(res[world]), one_gpu_nodes_step_ms=min(res[1]),
                   forward_all_to_all_ms=fwd_ms, backward_all_to_all_ms=bwd_ms,
                   exchange="NCCL over NVLink on one host: a lower bound on InfiniBand", **card())
        print(json.dumps(out), flush=True)
    dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
