#!/usr/bin/env python
"""Check of a process group that spans nodes, one process per rank:

    python -m torch.distributed.run --nnodes=1 --nproc-per-node P --master-addr 127.0.0.1 --master-port PORT \
        tools/cross_node_check.py --ranks-per-node L [--backend gloo|nccl] [--same-device] [--compare-single-node]

Every rank builds the same seeded global batch (tests/cross_node_oracle.make_problem), takes its slice and runs
DDPSigmoidLoss(ranks_per_node=L): N = P / L "nodes" whose contexts hold their own texts and their counterparts'.
Loss, image and text gradients (extras included), t_prime / bias gradients and per-sample losses are compared with the
float64 global-batch oracle at 1e-3 (norm-relative; bf16 gradients at 4e-3, their rounding), for every option the
exchange carries data for, fp32 inputs under normalize_inputs, a sigma budget that forces row panels, both schedules,
and sync_scalar_grads (bit-identical on every rank). --same-device puts every rank on cuda:0 (L = 1 only: the contexts
of one-rank nodes share no memory). --compare-single-node also runs the same data as one node (ranks_per_node = P,
the in-kernel exchange alone) and compares the two. Exit code 0 only if every rank passes."""
from __future__ import annotations

import argparse
import datetime
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from cross_node_oracle import OPTIONS, global_results, make_problem  # noqa: E402
from distributed_sigmoid_loss_b200 import DDPSigmoidLoss  # noqa: E402

TOL = 1e-3
TOL_BF16 = 4e-3   # bf16 gradients: the 2^-9 rounding of each element of the fp32 result


def rel(a, b) -> float:
    a = torch.as_tensor(np.asarray(a, np.float64)) if not isinstance(a, torch.Tensor) else a.detach().double().cpu()
    b = torch.as_tensor(np.asarray(b, np.float64))
    return float((a - b).norm() / max(float(b.norm()), 1e-30))


def normalized_oracle(p):
    """The oracle of normalize_inputs: the problem on L2-normalised rows, gradients through F.normalize."""
    q = dict(p)
    q["img"] = [x / np.linalg.norm(x, axis=1, keepdims=True) for x in p["img"]]
    q["txt"] = [x / np.linalg.norm(x, axis=1, keepdims=True) for x in p["txt"]]
    out = global_results(q)
    for g, o in enumerate(out):
        for key, raw, hat in (("dimg", p["img"][g], q["img"][g]), ("dtxt", p["txt"][g], q["txt"][g])):
            d = o[key]
            o[key] = (d - hat * (hat * d).sum(axis=1, keepdims=True)) / np.linalg.norm(raw, axis=1, keepdims=True)
    return out


def module_kwargs(p):
    o, K = p["option"], p["K"]
    kw = dict(batch_per_rank=p["Bs"])
    if o in ("ids", "extra_texts", "extra_images"):
        kw["multi_positive"] = True
    if o == "extra_texts":
        kw["extra_texts"] = K
    if o == "hard_negatives":
        kw["hard_negatives"] = K
    if o in ("weights", "focal"):
        kw["sample_weights"] = True
    if o == "groups":
        kw["exclude_groups"] = True
    if o == "label_sets":
        kw.update(multi_label=2, extra_texts=K)
    if o == "focal":
        kw.update(focal_gamma=p["focal"][0], focal_alpha=p["focal"][1])
    if o == "extra_images":
        kw["extra_images"] = p["K_img"]
    return kw


def run_rank(p, g, dev, dtype, ranks_per_node, fwd=None, **extra):
    """One rank's step: (loss, dimg [R], dtxt [T], dt', dbias, image_loss, text_loss) as host tensors."""
    B, K, Ki = p["Bs"][g], p["K"], p["K_img"]
    mod = DDPSigmoidLoss(B, ranks_per_node=ranks_per_node, **module_kwargs(p), **extra).to(dev)
    with torch.no_grad():
        mod.t_prime.fill_(p["t_prime"])
        mod.bias.fill_(p["bias"])

    def t(x, dt=dtype):
        return torch.tensor(np.asarray(x), dtype=dt, device=dev)

    img = t(p["img"][g][:B]).requires_grad_(True)
    txt = t(p["txt"][g][:B]).requires_grad_(True)
    kw = dict(return_sample_losses=True, **(fwd or {}))
    if K:
        ext = t(p["txt"][g][B:]).requires_grad_(True)
        kw["negative_text" if p["hard_negatives"] else "extra_text"] = ext
    if Ki:
        xim = t(p["img"][g][B:]).requires_grad_(True)
        kw["extra_image"] = xim
    if "ids" in p:
        kw["sample_ids"] = t(p["ids"][g], torch.int64)
    if "extra_text_ids" in p:
        kw["extra_text_ids"] = t(p["extra_text_ids"][g], torch.int64)
    if "extra_image_ids" in p:
        kw["extra_image_ids"] = t(p["extra_image_ids"][g], torch.int64)
    if "image_weights" in p:
        kw["image_weights"] = t(p["image_weights"][g], torch.float32)
        kw["text_weights"] = t(p["text_weights"][g], torch.float32)
    if "image_groups" in p:
        kw["image_groups"] = t(p["image_groups"][g], torch.int64)
        kw["text_groups"] = t(p["text_groups"][g], torch.int64)
    if p["multi_label"]:
        kw["sample_labels"] = t(p["sample_labels"][g], torch.int64)
        kw["extra_text_labels"] = t(p["extra_text_labels"][g], torch.int64)
    loss, sl = mod(img, txt, **kw)
    loss.backward()
    torch.cuda.synchronize(dev)
    dimg = torch.cat([img.grad] + ([xim.grad] if Ki else []))
    dtxt = torch.cat([txt.grad] + ([ext.grad] if K else []))
    cpu = lambda x: x.detach().double().cpu()  # noqa: E731
    return dict(loss=float(loss), dimg=cpu(dimg), dtxt=cpu(dtxt), dt_prime=float(mod.t_prime.grad),
                dbias=float(mod.bias.grad), image_loss=cpu(sl["image_loss"]), text_loss=cpu(sl["text_loss"]),
                raw_scalars=torch.stack([mod.t_prime.grad.detach().double(), mod.bias.grad.detach().double()]).cpu(),
                mod=mod)


def compare(name, got, want, grad_tol, rank, fails):
    errs = {}
    for k in ("loss", "dt_prime", "dbias"):
        errs[k] = abs(got[k] - want[k]) / max(abs(want[k]), 1e-30)
    for k in ("dimg", "dtxt"):
        errs[k] = rel(got[k], want[k])
    for k in ("image_loss", "text_loss"):
        errs[k] = rel(got[k], want[k])
    bad = {k: v for k, v in errs.items() if not v <= (grad_tol if k in ("dimg", "dtxt") else TOL)}
    worst = max(errs.values())
    print(f"[rank {rank}] {name}: worst rel {worst:.2e}" + (f" FAIL {bad}" if bad else " ok"), flush=True)
    if bad:
        fails.append(name)


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks-per-node", type=int, required=True)
    ap.add_argument("--backend", default="gloo", choices=["gloo", "nccl"])
    ap.add_argument("--same-device", action="store_true")
    ap.add_argument("--compare-single-node", action="store_true")
    ap.add_argument("--dim", type=int, default=64)
    args = ap.parse_args()
    dist.init_process_group(args.backend, timeout=datetime.timedelta(seconds=120))
    rank, world = dist.get_rank(), dist.get_world_size()
    L = args.ranks_per_node
    N = world // L
    dev = torch.device("cuda", 0 if args.same_device else int(os.environ.get("LOCAL_RANK", rank)))
    torch.cuda.set_device(dev)
    fails = []
    base = [40, 56, 48, 64, 40, 48, 56, 64][:world]
    for i, option in enumerate(OPTIONS):
        p = make_problem(N, L, base, args.dim, option, seed=100 + i)
        want = global_results(p)
        for fused in (True, False):
            got = run_rank(p, rank, dev, torch.float32, L, fused_step=fused)
            compare(f"{option} fp32 {'fused' if fused else 'split'}", got, want[rank], TOL, rank, fails)
    p = make_problem(N, L, base, args.dim, "plain", seed=7)
    # bf16 operands and gradients: the exchange moves the caller's dtype
    q = dict(p)
    q["img"] = [torch.tensor(x).bfloat16().double().numpy() for x in p["img"]]
    q["txt"] = [torch.tensor(x).bfloat16().double().numpy() for x in p["txt"]]
    compare("plain bf16", run_rank(q, rank, dev, torch.bfloat16, L), global_results(q)[rank], TOL_BF16, rank, fails)
    compare("normalize_inputs fp32", run_rank(p, rank, dev, torch.float32, L, normalize_inputs=True),
            normalized_oracle(p)[rank], TOL, rank, fails)
    # a sigma budget far below the fused step's two operands (5.6 MiB each at N = 2): row panels
    big = make_problem(N, L, [1024 + 16 * g for g in range(world)], args.dim, "weights", seed=8)
    got = run_rank(big, rank, dev, torch.float32, L, sigma_budget_bytes=2 << 20)
    eng = got["mod"].engine_for(big["Bs"][rank], args.dim, dev)
    panels = eng.sigma_panels()[1]
    print(f"[rank {rank}] sigma budget 2 MiB: {panels} row panels", flush=True)
    if panels < 2:
        fails.append("row panels")
    compare("sigma_budget_bytes", got, global_results(big)[rank], TOL, rank, fails)
    # sync_scalar_grads: the mean over every rank of the group, bit-identical everywhere
    want = global_results(p)
    got = run_rank(p, rank, dev, torch.float32, L, sync_scalar_grads=True)
    mean = dict(want[rank], dt_prime=float(np.mean([w["dt_prime"] for w in want])),
                dbias=float(np.mean([w["dbias"] for w in want])))
    compare("sync_scalar_grads", got, mean, TOL, rank, fails)
    all_s = [None] * world
    dist.all_gather_object(all_s, got["raw_scalars"])
    same = all(torch.equal(x, all_s[0]) for x in all_s)
    print(f"[rank {rank}] sync_scalar_grads bit-identical on every rank: {same}", flush=True)
    if not same:
        fails.append("sync bit-identical")
    if args.compare_single_node:
        one = run_rank(p, rank, dev, torch.float32, world)
        assert one["mod"].engine_for(p["Bs"][rank], args.dim, dev).topology is None
        compare("single node (in-kernel exchange only)", one, want[rank], TOL, rank, fails)
        nodes = run_rank(p, rank, dev, torch.float32, L)
        d = max(rel(nodes[k], one[k].numpy()) for k in ("dimg", "dtxt", "image_loss", "text_loss"))
        print(f"[rank {rank}] {N} nodes vs one node: worst rel {d:.2e}", flush=True)
        if not d <= TOL:
            fails.append("nodes vs one node")
    # refusals name the option and say "across nodes"
    try:
        run_rank(p, rank, dev, torch.float32, L, fwd=dict(return_metrics=True))
        fails.append("return_metrics not refused")
    except RuntimeError as e:
        if "across nodes" not in str(e):
            fails.append(f"return_metrics refusal: {e}")
    flags = [None] * world
    dist.all_gather_object(flags, len(fails))
    ok = all(f == 0 for f in flags)
    if rank == 0:
        print("CROSS-NODE CHECK " + ("PASS" if ok else "FAIL"), flush=True)
    dist.destroy_process_group()
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
