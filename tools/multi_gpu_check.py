#!/usr/bin/env python
"""Multi-GPU parity + timing check, one rank per GPU:

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29533 \
        tools/multi_gpu_check.py [--time]

Every rank builds the same seeded global batch, takes its slice, runs the module (NVSwitch peer pulls of the text
chunks, per-owner dtxt slots, cross-rank reduction) and compares with
  * the float64 closed form over the GLOBAL batch (oracle.closed_form) at a small shape, and
  * fp32 autograd of the same math at a larger one (the text gradient reference is all-reduced over ranks).
Exit code 0 only if every rank passes.
"""
from __future__ import annotations

import argparse
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402


def rel_f(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-300))


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--time", action="store_true")
    ap.add_argument("--batch", type=int, default=16384)
    ap.add_argument("--dim", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--all-variants", action="store_true", help="also time the non-overlapped variants")
    ap.add_argument("--skip-parity", action="store_true")
    ap.add_argument("--sample-ids", action="store_true",
                    help="also check multi-positive labels from sample ids (duplicates across ranks) against the oracle")
    ap.add_argument("--metrics", action="store_true",
                    help="also check the in-batch retrieval metrics (return_metrics=True) against the float64 oracle, with "
                         "and without shared sample ids, uneven batches, fused and split schedules")
    ap.add_argument("--hard-negatives", action="store_true",
                    help="also check hard-negative captions (extra texts per rank, negatives for every image) against the "
                         "float64 oracle: the module with the same K on every rank (fused and split, uneven batches) and "
                         "an engine with a different K per rank")
    ap.add_argument("--extra-texts", action="store_true",
                    help="also check extra captions with ids (several captions per image) against the float64 oracle: "
                         "extras that caption images of other ranks, extras that match nothing, fused and split")
    ap.add_argument("--extra-images", action="store_true",
                    help="also check extra images per rank against the float64 oracle: hard-negative images, and with ids "
                         "extra images whose ids caption texts of other ranks, with extra texts too, fused and split, "
                         "and the retrieval metrics over the published extra-image ids")
    ap.add_argument("--weights", action="store_true",
                    help="also check per-sample loss weights against the float64 oracle: random weights with zeros on "
                         "every rank, the text weights travelling with the text, uneven batches, with and without sample "
                         "ids and hard negatives, fused and split")
    ap.add_argument("--distill", action="store_true",
                    help="also check distillation from a frozen teacher against the float64 oracle: the teacher text "
                         "travelling with the student text through the peer pulls, a teacher width different from the "
                         "student's, uneven batches, with and without sample ids and weights, fused and split")
    ap.add_argument("--distill-options", action="store_true",
                    help="also check distillation with the other options against the float64 oracle: hard negatives "
                         "and label sets with extras (each with the teacher's rows of the extras travelling with the "
                         "text), excluded groups and weights, per-sample losses, uneven batches, fused and split")
    ap.add_argument("--sample-losses", action="store_true",
                    help="also check the per-sample losses (return_sample_losses=True) against the float64 oracle: "
                         "text_loss combines every rank's column partials of the own chunk, uneven batches, hard "
                         "negatives, ids and weights, fused / split / forward-only, and the cross-rank sum identity")
    ap.add_argument("--metrics-topk", action="store_true",
                    help="also check the top-K retrieval (metrics_topk=10) against the float64 oracle on exact "
                         "small-integer embeddings: t2i merges every rank's column lists of the own chunk, uneven "
                         "batches, hard negatives, ids with duplicates, fused / split / forward-only")
    ap.add_argument("--exclude-groups", action="store_true",
                    help="also check excluded same-group pairs (exclude_groups=True) against the float64 oracle, with "
                         "and without ids and with hard negatives, on both schedules")
    ap.add_argument("--label-sets", action="store_true",
                    help="also check multi-label positives (multi_label=M) against the float64 oracle, with extra texts "
                         "and extra images carrying label sets")
    ap.add_argument("--focal", action="store_true",
                    help="also check the focal pair loss (focal_gamma / focal_alpha) against the float64 oracle, "
                         "positional, with label sets and extras, and with weights and excluded groups")
    ap.add_argument("--row-panels", action="store_true",
                    help="also check the fused step in row panels (sigma_budget_bytes forcing several panels) against "
                         "the float64 closed form and against the unbounded step on the same peers: uneven batches "
                         "(DDPSigmoidLoss), bidir (SigLipLoss), two steps each")
    ap.add_argument("--soak", type=int, default=0,
                    help="N > 0: that many back-to-back steps at the --batch/--dim shape mixing the fused step, the split "
                         "API and forward-only calls; same inputs, so every step of a kind must reproduce its first result "
                         "bit for bit")
    args = ap.parse_args()
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, _capi
    from oracle.siglip_oracle import closed_form, torch_reference_fp32

    ok = True

    def report(tag, errs, tol=1e-3):
        nonlocal ok
        good = all(v <= tol for v in errs.values())
        ok &= good
        print(f"[rank {rank}] {tag}: " + " ".join(f"{k}={v:.2e}" for k, v in errs.items()) + (" OK" if good else " FAIL"),
              flush=True)

    # ---- small: float64 closed form over the global batch -------------------------------------------------
    for (B, D, tp, bias) in ([] if args.skip_parity else [(96, 64, math.log(10.0), -10.0), (512, 256, math.log(20.0), -5.0)]):
        g = torch.Generator().manual_seed(99)
        img_all = torch.nn.functional.normalize(torch.randn(world * B, D, generator=g)).to(torch.bfloat16)
        txt_all = torch.nn.functional.normalize(torch.randn(world * B, D, generator=g)).to(torch.bfloat16)
        ref = closed_form(img_all.float().numpy(), txt_all.float().numpy(), tp, bias, world)[rank]
        mod = DDPSigmoidLoss(B).to(dev)
        with torch.no_grad():
            mod.t_prime.fill_(tp)
            mod.bias.fill_(bias)
        eng = mod.engine_for(B, D, dev)
        img = img_all[rank * B:(rank + 1) * B].to(dev).contiguous()
        txt = txt_all[rank * B:(rank + 1) * B].to(dev).contiguous()
        for rep in range(2):   # second repetition exercises the step-to-step flag protocol
            loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, torch.tensor([tp], device=dev),
                                                    torch.tensor([bias], device=dev))
            loss_f = eng.fwd(img, txt, torch.tensor([tp], device=dev), torch.tensor([bias], device=dev))
            torch.cuda.synchronize()
            report(f"closed-form B={B} D={D} rep{rep}", dict(
                loss=abs(float(loss) - ref["loss"]) / abs(ref["loss"]),
                loss_fwd=abs(float(loss_f) - ref["loss"]) / abs(ref["loss"]),
                dimg=rel_f(dimg.cpu(), torch.from_numpy(ref["dimg"])),
                dtxt=rel_f(dtxt.cpu(), torch.from_numpy(ref["dtxt"])),
                dtp=abs(float(dtp) - ref["dt_prime"]) / abs(ref["dt_prime"]),
                db=abs(float(db) - ref["dbias"]) / abs(ref["dbias"])))
        # the split forward / backward API (one sigma operand per chunk, helper-kernel flags) on the same peers
        tpt, bt = torch.tensor([tp], device=dev), torch.tensor([bias], device=dev)
        for rep in range(2):
            ls = eng.forward(img, txt, tpt, bt, True)
            dimg_s, dtxt_s, dtp_s, db_s = eng.backward(img, txt, tpt, None)
            torch.cuda.synchronize()
            report(f"split API B={B} D={D} rep{rep}", dict(
                loss=abs(float(ls) - ref["loss"]) / abs(ref["loss"]),
                dimg=rel_f(dimg_s.cpu(), torch.from_numpy(ref["dimg"])),
                dtxt=rel_f(dtxt_s.cpu(), torch.from_numpy(ref["dtxt"])),
                dtp=abs(float(dtp_s) - ref["dt_prime"]) / abs(ref["dt_prime"]),
                db=abs(float(db_s) - ref["dbias"]) / abs(ref["dbias"]),
                vs_fused_dtxt=rel_f(dtxt_s, dtxt)), tol=1e-3)
        # the fused step with the flags handled by separate helper kernels (SIGLIP_OPT_INKERNEL_SYNC = 0)
        eng.set_option(_capi.SIGLIP_OPT_INKERNEL_SYNC, 0)
        for rep in range(2):
            l0, dimg0, dtxt0, dtp0, db0 = eng.fwd_bwd(img, txt, tpt, bt)
            torch.cuda.synchronize()
            report(f"fused, helper-kernel flags B={B} rep{rep}", dict(
                loss=abs(float(l0) - ref["loss"]) / abs(ref["loss"]),
                dimg=rel_f(dimg0.cpu(), torch.from_numpy(ref["dimg"])),
                dtxt=rel_f(dtxt0.cpu(), torch.from_numpy(ref["dtxt"])),
                bitwise_vs_inkernel=0.0 if (torch.equal(dimg0, dimg) and torch.equal(dtxt0, dtxt)) else 1.0))
        eng.set_option(_capi.SIGLIP_OPT_INKERNEL_SYNC, 1)
        # module surface (fused schedule by default on a multi-rank group; split schedule on request)
        for fused in (None, False):
            modx = DDPSigmoidLoss(B, fused_step=fused).to(dev)
            with torch.no_grad():
                modx.t_prime.fill_(tp)
                modx.bias.fill_(bias)
            a, b = img.clone().requires_grad_(True), txt.clone().requires_grad_(True)
            l2 = modx(a, b)
            l2.backward()
            torch.cuda.synchronize()
            report(f"module fused_step={fused} B={B}", dict(
                loss=abs(float(l2) - ref["loss"]) / abs(ref["loss"]),
                dimg=rel_f(a.grad.float().cpu(), torch.from_numpy(ref["dimg"])),
                dtxt=rel_f(b.grad.float().cpu(), torch.from_numpy(ref["dtxt"])),
                dtp=abs(float(modx.t_prime.grad) - ref["dt_prime"]) / abs(ref["dt_prime"]),
                db=abs(float(modx.bias.grad) - ref["dbias"]) / abs(ref["dbias"])), tol=4e-3)
            del modx

    # ---- fp32 callers: raw fp32 inputs -> fp16(16 x) operands, text chunks exchanged in that format ---------------
    if not args.skip_parity:
        B, D, tp, bias = 160, 96, math.log(10.0), -10.0
        g = torch.Generator().manual_seed(123)
        img_all = torch.nn.functional.normalize(torch.randn(world * B, D, generator=g))
        txt_all = torch.nn.functional.normalize(torch.randn(world * B, D, generator=g))
        ref = closed_form(img_all.numpy(), txt_all.numpy(), tp, bias, world)[rank]
        mod = DDPSigmoidLoss(B).to(dev)
        a = img_all[rank * B:(rank + 1) * B].to(dev).requires_grad_(True)
        b = txt_all[rank * B:(rank + 1) * B].to(dev).requires_grad_(True)
        for rep in range(2):
            a.grad = b.grad = mod.t_prime.grad = mod.bias.grad = None
            lf = mod(a, b)
            lf.backward()
            torch.cuda.synchronize()
            report(f"fp32 inputs (fp16x16 operands) B={B} D={D} rep{rep}", dict(
                loss=abs(float(lf.detach()) - ref["loss"]) / abs(ref["loss"]),
                dimg=rel_f(a.grad.cpu(), torch.from_numpy(ref["dimg"])),
                dtxt=rel_f(b.grad.cpu(), torch.from_numpy(ref["dtxt"])),
                dtp=abs(float(mod.t_prime.grad) - ref["dt_prime"]) / abs(ref["dt_prime"]),
                db=abs(float(mod.bias.grad) - ref["dbias"]) / abs(ref["dbias"])))

    # ---- SURVEY §8f-4: ranks with different batch sizes (B_r = 72 + 24 r), float64 closed form over the global set ----
    if not args.skip_parity:
        from distributed_sigmoid_loss_b200 import SigmoidLossEngine
        Bs = [72 + 24 * r for r in range(world)]
        D, tp, bias = 136, math.log(10.0), -9.0
        g = torch.Generator().manual_seed(321)
        imgs = [torch.nn.functional.normalize(torch.randn(b, D, generator=g)).to(torch.bfloat16) for b in Bs]
        txts = [torch.nn.functional.normalize(torch.randn(b, D, generator=g)).to(torch.bfloat16) for b in Bs]
        t = math.exp(tp)
        i64 = imgs[rank].double()
        loss_ref, dimg_ref, dtp_ref, db_ref = 0.0, torch.zeros_like(i64), 0.0, 0.0
        for c in range(world):
            s_ = i64 @ txts[c].double().T
            z = t * s_ + bias
            y = -torch.ones_like(z)
            if c == rank:
                y.fill_diagonal_(1.0)
            gmat = -y * torch.sigmoid(-y * z) / Bs[rank]
            loss_ref += float(torch.nn.functional.softplus(-y * z).sum() / Bs[rank])
            dimg_ref += t * (gmat @ txts[c].double())
            dtp_ref += float(t * (gmat * s_).sum())
            db_ref += float(gmat.sum())
        # text gradient of MY chunk: sum over all ranks r of t * G_{r,me}^T img_r
        dtxt_ref = torch.zeros(Bs[rank], D, dtype=torch.float64)
        for r in range(world):
            s_ = imgs[r].double() @ txts[rank].double().T
            z = t * s_ + bias
            y = -torch.ones_like(z)
            if r == rank:
                y.fill_diagonal_(1.0)
            gmat = -y * torch.sigmoid(-y * z) / Bs[r]
            dtxt_ref += t * (gmat.T @ imgs[r].double())
        engu = SigmoidLossEngine(Bs[rank], D, dev, batch_per_rank=Bs)
        tpt, bt = torch.tensor([tp], device=dev), torch.tensor([bias], device=dev)
        for rep in range(2):
            lu, dimg_u, dtxt_u, dtp_u, db_u = engu.fwd_bwd(imgs[rank].to(dev), txts[rank].to(dev), tpt, bt)
            torch.cuda.synchronize()
            report(f"uneven batches {Bs} rep{rep}", dict(
                loss=abs(float(lu) - loss_ref) / abs(loss_ref), dimg=rel_f(dimg_u.cpu(), dimg_ref),
                dtxt=rel_f(dtxt_u.cpu(), dtxt_ref), dtp=abs(float(dtp_u) - dtp_ref) / abs(dtp_ref),
                db=abs(float(db_u) - db_ref) / abs(db_ref)))
        engu.close()

    # ---- multi-positive labels from sample ids: 40 classes over the global batch, so most ranks share ids with every
    # other rank (cross-chunk positives); the ids travel with the text through the peer exchange -----------------------
    if args.sample_ids:
        sys.path.insert(0, os.path.join(ROOT, "tests"))      # the ids oracle lives with the tests
        from sample_ids_oracle import closed_form_ids
        for (B, D, tp, bias) in [(96, 64, math.log(10.0), -10.0), (200, 136, math.log(10.0), -8.0)]:
            g = torch.Generator().manual_seed(77)
            img_all = torch.nn.functional.normalize(torch.randn(world * B, D, generator=g)).to(torch.bfloat16)
            txt_all = torch.nn.functional.normalize(torch.randn(world * B, D, generator=g)).to(torch.bfloat16)
            ids_all = torch.randint(-(2 ** 40), -(2 ** 40) + 40, (world * B,), generator=g)
            blk = lambda x, r: x[r * B:(r + 1) * B]  # noqa: E731
            ref = closed_form_ids([blk(img_all, r).float().numpy() for r in range(world)],
                                  [blk(txt_all, r).float().numpy() for r in range(world)],
                                  [blk(ids_all, r).numpy() for r in range(world)], tp, bias)
            mine = ref[rank]
            dtxt_ref = torch.from_numpy(sum(ref[r]["contrib"][rank] for r in range(world)))
            img, txt = blk(img_all, rank).to(dev).contiguous(), blk(txt_all, rank).to(dev).contiguous()
            ids = blk(ids_all, rank).to(dev).contiguous()
            for fused in (None, False):
                modx = DDPSigmoidLoss(B, fused_step=fused, multi_positive=True).to(dev)
                with torch.no_grad():
                    modx.t_prime.fill_(tp)
                    modx.bias.fill_(bias)
                for rep in range(2):
                    a, b = img.float().requires_grad_(True), txt.float().requires_grad_(True)
                    l2 = modx(a, b, sample_ids=ids)
                    l2.backward()
                    torch.cuda.synchronize()
                    report(f"sample ids fused_step={fused} B={B} D={D} rep{rep}", dict(
                        loss=abs(float(l2) - mine["loss"]) / abs(mine["loss"]),
                        dimg=rel_f(a.grad.cpu(), torch.from_numpy(mine["dimg"])),
                        dtxt=rel_f(b.grad.cpu(), dtxt_ref),
                        dtp=abs(float(modx.t_prime.grad) - mine["dt_prime"]) / abs(mine["dt_prime"]),
                        db=abs(float(modx.bias.grad) - mine["dbias"]) / abs(mine["dbias"])))
                del modx

    # ---- in-batch retrieval metrics: texts are perturbed images under a permutation (a fifth of them point at another
    # rank's sample), so the top-1 of every direction crosses ranks; uneven batches; ids shared across ranks ----------
    if args.metrics:
        sys.path.insert(0, os.path.join(ROOT, "tests"))      # the oracle lives with the tests
        from retrieval_metrics_oracle import hits, retrieval_metrics
        from distributed_sigmoid_loss_b200 import SigmoidLossEngine
        Bs = [96 + 40 * r for r in range(world)]
        D, tp, bias = 128, math.log(10.0), -10.0
        g = torch.Generator().manual_seed(555)
        n = sum(Bs)
        img_all = torch.nn.functional.normalize(torch.randn(n, D, generator=g))
        perm = torch.arange(n)
        sel = torch.randperm(n, generator=g)[: n // 5]
        perm[sel] = sel.roll(1)
        txt_all = torch.nn.functional.normalize(img_all[perm] + 0.1 * torch.randn(n, D, generator=g))
        img_all, txt_all = img_all.to(torch.bfloat16), txt_all.to(torch.bfloat16)
        ids_all = torch.arange(n) % (n // 2)                 # every id twice, mostly on two different ranks
        imgs, txts, idss = (list(torch.split(x, Bs)) for x in (img_all, txt_all, ids_all))
        off = sum(Bs[:rank])
        for with_ids in (False, True):
            res = retrieval_metrics([x.float().numpy() for x in imgs], [x.float().numpy() for x in txts],
                                    [x.numpy() for x in idss] if with_ids else None)[rank]
            eng = SigmoidLossEngine(Bs[rank], D, dev, batch_per_rank=Bs)
            if with_ids:
                eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 1)
            tpt, bt = torch.tensor([tp], device=dev), torch.tensor([bias], device=dev)
            img, txt = imgs[rank].to(dev), txts[rank].to(dev)
            for sched in ("fused", "split", "fwd", "fused"):
                top1 = torch.empty(2, device=dev)
                i2t = torch.empty(Bs[rank], device=dev, dtype=torch.int64)
                t2i = torch.empty(Bs[rank], device=dev, dtype=torch.int64)
                if with_ids:
                    eng.set_sample_ids(idss[rank].to(dev))
                eng.request_metrics(top1, i2t, t2i)
                if sched == "fused":
                    eng.fwd_bwd(img, txt, tpt, bt)
                elif sched == "split":
                    eng.forward(img, txt, tpt, bt, True)
                    eng.backward(img, txt, tpt, None)
                else:
                    eng.fwd(img, txt, tpt, bt)
                torch.cuda.synchronize()
                gi, gt = i2t.cpu().numpy(), t2i.cpu().numpy()
                ok_i, ok_t = res["i2t_margin"] > 1e-3, res["t2i_margin"] > 1e-3
                hi, ht = hits(gi, res["gid"], off), hits(gt, res["gid"], off)
                report(f"retrieval metrics ids={with_ids} {sched} B={Bs}", dict(
                    i2t_index=float((gi != res["i2t_index"])[ok_i].mean()),
                    t2i_index=float((gt != res["t2i_index"])[ok_t].mean()),
                    i2t_top1=abs(float(top1[0]) - hi.mean()), t2i_top1=abs(float(top1[1]) - ht.mean()),
                    unclear_rows=float(1.0 - min(ok_i.mean(), ok_t.mean())) / 50), tol=1e-6)
            eng.close()

    # ---- per-sample losses: the column sums of my chunk add every rank's fixed-point partials after flag kind 5; the
    # totals over ranks of image_loss and text_loss agree --------------------------------------------------------------
    if args.row_panels:
        from distributed_sigmoid_loss_b200 import SigLipLoss
        for (Bs, D, bidir) in ([[1000 - 100 * (p % 3) for p in range(world)], 136, False],
                               [[960] * world, 264, True]):   # SigLipLoss: equal batches
            B = Bs[rank]
            off = [sum(Bs[:p]) for p in range(world + 1)]
            g = torch.Generator().manual_seed(7)
            img_all = torch.nn.functional.normalize(torch.randn(off[-1], D, generator=g)).to(torch.bfloat16)
            txt_all = torch.nn.functional.normalize(img_all.float() + 0.6 * torch.randn(off[-1], D, generator=g))
            txt_all = txt_all.to(torch.bfloat16)
            img = img_all[off[rank]:off[rank + 1]].to(dev).contiguous()
            txt = txt_all[off[rank]:off[rank + 1]].to(dev).contiguous()
            tpt, bt = torch.tensor([math.log(10.0)], device=dev), torch.tensor([-10.0], device=dev)
            outs = []
            for budget in (None, 1 << 20):
                mod = (SigLipLoss(rank=rank, world_size=world, bidir=True, sigma_budget_bytes=budget) if bidir else
                       DDPSigmoidLoss(B, batch_per_rank=Bs, sigma_budget_bytes=budget)).to(dev)
                eng = mod._cache.get(B, D, dev)
                if budget:
                    rows, n, _ = eng.sigma_panels()
                    assert n >= 2, (rows, n)
                for rep in range(2):
                    out = [x.clone() for x in eng.fwd_bwd(img, txt, tpt, bt)]
                torch.cuda.synchronize()
                outs.append(out)
            # every rank's loss over its rows: the closed form over the global batch (uneven: per-rank blocks)
            x, y = img_all.double(), txt_all.double()
            z = 10.0 * (x[off[rank]:off[rank + 1]] @ y.T) - 10.0
            lab = -torch.ones_like(z)
            lab[torch.arange(B), off[rank] + torch.arange(B)] = 1.0
            loss_ref = float(torch.nn.functional.softplus(-lab * z).sum() / B)
            gz = -lab * torch.sigmoid(-lab * z) * 10.0 / B
            dimg_ref = gz @ y
            unb, pan = outs
            report(f"row panels W={world} Bs={Bs} D={D} bidir={bidir} vs float64", dict(
                loss=abs(float(pan[0]) - loss_ref) / abs(loss_ref),
                dimg=rel_f(pan[1].cpu(), dimg_ref.float())))
            report(f"row panels W={world} Bs={Bs} D={D} bidir={bidir} vs unbounded",
                   {k: rel_f(a.cpu().float(), b.cpu().float()) for k, a, b in
                    zip(("loss", "dimg", "dtxt", "dt_prime", "dbias"), pan, unb)}, tol=1e-5)

    if args.sample_losses:
        sys.path.insert(0, os.path.join(ROOT, "tests"))      # the oracle lives with the tests
        from extra_images_oracle import label_blocks
        from sample_losses_oracle import sample_losses
        from distributed_sigmoid_loss_b200 import SigmoidLossEngine
        Bs = [160 + 24 * r for r in range(world)]
        Ts = [b + 8 + 4 * r for r, b in enumerate(Bs)]
        D, tp, bias = 136, math.log(10.0), -8.0
        g = torch.Generator().manual_seed(777)
        imgs = [torch.nn.functional.normalize(torch.randn(b, D, generator=g)).to(torch.bfloat16) for b in Bs]
        txts = [torch.nn.functional.normalize(torch.randn(t, D, generator=g)).to(torch.bfloat16) for t in Ts]
        idss = [torch.randint(0, sum(Bs) // 2, (b,), generator=g) for b in Bs]
        wis = [torch.rand(b, generator=g) * (torch.rand(b, generator=g) > 0.2) for b in Bs]
        wts = [torch.rand(t, generator=g) * (torch.rand(t, generator=g) > 0.2) for t in Ts]
        for with_ids in (False, True):
            labels = label_blocks(Bs, Bs, Ts, [x.numpy() for x in idss] if with_ids else None)
            ref = sample_losses([x.float().numpy() for x in imgs], [x.float().numpy() for x in txts], Bs, tp, bias,
                                labels, [x.numpy() for x in wis], [x.numpy() for x in wts])
            eng = SigmoidLossEngine(Bs[rank], D, dev, batch_per_rank=Bs, texts_per_rank=Ts)
            if with_ids:
                eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 1)
            eng.set_option(_capi.SIGLIP_OPT_SAMPLE_WEIGHTS, 1)
            tpt, bt = torch.tensor([tp], device=dev), torch.tensor([bias], device=dev)
            img, txt = imgs[rank].to(dev), txts[rank].to(dev)
            for sched in ("fused", "split", "fwd", "fused"):
                il = torch.empty(Bs[rank], device=dev)
                tl = torch.empty(Ts[rank], device=dev)
                if with_ids:
                    eng.set_sample_ids(idss[rank].to(dev))
                eng.set_sample_weights(wis[rank].to(dev), wts[rank].to(dev))
                eng.request_sample_losses(il, tl)
                if sched == "fused":
                    loss = eng.fwd_bwd(img, txt, tpt, bt)[0]
                elif sched == "split":
                    loss = eng.forward(img, txt, tpt, bt, True)
                    eng.backward(img, txt, tpt, None)
                else:
                    loss = eng.fwd(img, txt, tpt, bt)
                torch.cuda.synchronize()
                tot = torch.tensor([il.double().sum(), tl.double().sum()], device=dev)
                dist.all_reduce(tot)
                want_i, want_t = ref[rank]["image_loss"], ref[rank]["text_loss"]

                def max_rel(got, want):
                    got = got.double().cpu().numpy()
                    keep = want > 0
                    return float(np.max(np.abs(got[keep] - want[keep]) / want[keep]))

                report(f"sample losses ids={with_ids} {sched} B={Bs} T={Ts}", dict(
                    image_loss=max_rel(il, want_i), text_loss=max_rel(tl, want_t),
                    zero_weights=float((il.cpu()[wis[rank] == 0] != 0).any() or (tl.cpu()[wts[rank] == 0] != 0).any()),
                    loss_identity=abs(float(il.double().sum()) / Bs[rank] - float(loss)) / abs(float(loss)),
                    cross_rank_sums=abs(float(tot[0] - tot[1])) / float(tot[0])), tol=1e-3)
            eng.close()

    if args.metrics_topk:
        sys.path.insert(0, os.path.join(ROOT, "tests"))      # the oracle lives with the tests
        from retrieval_topk_oracle import recall_counts, topk_retrieval
        from distributed_sigmoid_loss_b200 import SigmoidLossEngine
        Bs = [160 + 24 * r for r in range(world)]
        Ts = [b + 8 + 4 * r for r, b in enumerate(Bs)]
        D, K = 136, 10
        gn = np.random.default_rng(4242)
        # small integers / 8: exact bf16 operands, exact fp32 logits, so the lists compare exactly (ties included)
        base = [gn.integers(-2, 3, (b, D)) for b in Bs]
        imgs = [torch.from_numpy(x / 8).to(torch.bfloat16) for x in base]
        txts = [torch.from_numpy(np.concatenate([x + gn.integers(-1, 2, x.shape), gn.integers(-2, 3, (t - b, D))]) / 8)
                .to(torch.bfloat16) for x, b, t in zip(base, Bs, Ts)]
        idss = [gn.integers(0, sum(Bs) // 2, b).astype(np.int64) for b in Bs]
        for with_ids in (False, True):
            ref = topk_retrieval([x.double().numpy() for x in imgs], [x.double().numpy() for x in txts], Bs, K,
                                 img_ids=idss if with_ids else None, txt_ids=idss if with_ids else None)[rank]
            eng = SigmoidLossEngine(Bs[rank], D, dev, batch_per_rank=Bs, texts_per_rank=Ts)
            if with_ids:
                eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 1)
            tpt, bt = torch.tensor([math.log(10.0)], device=dev), torch.tensor([-8.0], device=dev)
            img, txt = imgs[rank].to(dev), txts[rank].to(dev)
            for sched in ("fused", "split", "fwd", "fused"):
                recall = torch.empty(2 * K, device=dev)
                i2t = torch.empty(Bs[rank], K, device=dev, dtype=torch.int64)
                t2i = torch.empty(Bs[rank], K, device=dev, dtype=torch.int64)
                if with_ids:
                    eng.set_sample_ids(torch.from_numpy(idss[rank]).to(dev))
                eng.request_topk(K, recall, i2t, t2i)
                if sched == "fused":
                    eng.fwd_bwd(img, txt, tpt, bt)
                elif sched == "split":
                    eng.forward(img, txt, tpt, bt, True)
                    eng.backward(img, txt, tpt, None)
                else:
                    eng.fwd(img, txt, tpt, bt)
                torch.cuda.synchronize()
                want = np.concatenate([recall_counts(ref["i2t_first"], K), recall_counts(ref["t2i_first"], K)])
                report(f"top-K ids={with_ids} {sched} B={Bs} T={Ts}", dict(
                    i2t_lists=float((i2t.cpu().numpy() != ref["i2t_topk"]).mean()),
                    t2i_lists=float((t2i.cpu().numpy() != ref["t2i_topk"]).mean()),
                    recall=float(np.abs(recall.cpu().numpy() - want).max())), tol=0.0)
            eng.close()

    # ---- hard-negative captions: every rank's extras are pulled with its text and scored against every image; their
    # text gradient sums every rank's contribution through the dtxt exchange -------------------------------------------
    if args.hard_negatives:
        sys.path.insert(0, os.path.join(ROOT, "tests"))      # the oracle lives with the tests
        from hard_negatives_oracle import closed_form_hard_negatives
        from distributed_sigmoid_loss_b200 import SigmoidLossEngine
        Bs = [160 + 24 * r for r in range(world)]
        D, tp, bias = 136, math.log(10.0), -8.0
        g = torch.Generator().manual_seed(4242)
        unit = lambda n: torch.nn.functional.normalize(torch.randn(n, D, generator=g)).to(torch.bfloat16)  # noqa: E731
        imgs, txts = [unit(b) for b in Bs], [unit(b) for b in Bs]
        for Ks in ([37] * world, [8 + 40 * r for r in range(world)]):
            extras = [unit(k) for k in Ks]
            ref = closed_form_hard_negatives([x.float().numpy() for x in imgs], [x.float().numpy() for x in txts],
                                             [x.float().numpy() for x in extras], tp, bias)
            mine = ref[rank]
            dtxt_ref = torch.from_numpy(sum(ref[r]["contrib"][rank] for r in range(world)))
            img, txt, ext = imgs[rank].to(dev), txts[rank].to(dev), extras[rank].to(dev)
            same_k = len(set(Ks)) == 1
            for fused in ((None, False) if same_k else ("engine",)):
                for rep in range(2):
                    if fused == "engine":
                        if rep == 0:
                            eng = SigmoidLossEngine(Bs[rank], D, dev, batch_per_rank=Bs,
                                                    texts_per_rank=[b + k for b, k in zip(Bs, Ks)])
                        l2, gi, gt, dtp, db = eng.fwd_bwd(img, torch.cat([txt, ext]), torch.tensor([tp], device=dev),
                                                          torch.tensor([bias], device=dev))
                        dtp, db = float(dtp), float(db)
                    else:
                        if rep == 0:
                            modx = DDPSigmoidLoss(Bs[rank], fused_step=fused, batch_per_rank=Bs,
                                                  hard_negatives=Ks[0]).to(dev)
                            with torch.no_grad():
                                modx.t_prime.fill_(tp)
                                modx.bias.fill_(bias)
                        modx.zero_grad()
                        a, b, e = (x.float().requires_grad_(True) for x in (img, txt, ext))
                        l2 = modx(a, b, negative_text=e)
                        l2.backward()
                        gi, gt = a.grad, torch.cat([b.grad, e.grad])
                        dtp, db = float(modx.t_prime.grad), float(modx.bias.grad)
                    torch.cuda.synchronize()
                    report(f"hard negatives {fused} B={Bs} K={Ks} D={D} rep{rep}", dict(
                        loss=abs(float(l2) - mine["loss"]) / abs(mine["loss"]),
                        dimg=rel_f(gi.float().cpu(), torch.from_numpy(mine["dimg"])),
                        dtxt=rel_f(gt.float().cpu(), dtxt_ref),
                        dneg=rel_f(gt[Bs[rank]:].float().cpu(), dtxt_ref[Bs[rank]:]),
                        dtp=abs(dtp - mine["dt_prime"]) / abs(mine["dt_prime"]),
                        db=abs(db - mine["dbias"]) / abs(mine["dbias"])))
            if not same_k:
                eng.close()

    # ---- extra captions with ids: an extra of one rank is a positive for the images with its id on every rank; the
    # ids travel with the text through the peer pulls --------------------------------------------------------------
    if args.extra_texts:
        sys.path.insert(0, os.path.join(ROOT, "tests"))      # the oracle lives with the tests
        from extra_text_ids_oracle import closed_form_extra_text_ids
        Bs = [160 + 24 * r for r in range(world)]
        K, D, tp, bias = 300, 136, math.log(10.0), -8.0
        g = torch.Generator().manual_seed(4343)
        unit = lambda n: torch.nn.functional.normalize(torch.randn(n, D, generator=g)).to(torch.bfloat16)  # noqa: E731
        imgs, txts, extras = [unit(b) for b in Bs], [unit(b) for b in Bs], [unit(K) for _ in Bs]
        ids = list(torch.split(torch.arange(sum(Bs), dtype=torch.int64) * 2, Bs))
        # extra j of rank r: a caption of image j of rank (r + 1) % world (its id), every fourth one an id no image has
        eids = []
        for r in range(world):
            own = ids[(r + 1) % world]
            e = own[torch.arange(K) % len(own)].clone()
            e[::4] = -1 - torch.arange(len(e[::4]))
            eids.append(e)
        ref = closed_form_extra_text_ids([x.float().numpy() for x in imgs], [x.float().numpy() for x in txts],
                                         [x.float().numpy() for x in extras], [x.numpy() for x in ids],
                                         [x.numpy() for x in eids], tp, bias)
        mine = ref[rank]
        dtxt_ref = torch.from_numpy(sum(ref[r]["contrib"][rank] for r in range(world)))
        img, txt, ext = imgs[rank].to(dev), txts[rank].to(dev), extras[rank].to(dev)
        for fused in (None, False):
            modx = DDPSigmoidLoss(Bs[rank], fused_step=fused, batch_per_rank=Bs, multi_positive=True,
                                  extra_texts=K).to(dev)
            with torch.no_grad():
                modx.t_prime.fill_(tp)
                modx.bias.fill_(bias)
            for rep in range(2):
                modx.zero_grad()
                a, b, e = (x.float().requires_grad_(True) for x in (img, txt, ext))
                l2 = modx(a, b, sample_ids=ids[rank].to(dev), extra_text=e, extra_text_ids=eids[rank].to(dev))
                l2.backward()
                torch.cuda.synchronize()
                gt = torch.cat([b.grad, e.grad])
                report(f"extra texts {fused} B={Bs} K={K} D={D} rep{rep}", dict(
                    loss=abs(float(l2) - mine["loss"]) / abs(mine["loss"]),
                    dimg=rel_f(a.grad.float().cpu(), torch.from_numpy(mine["dimg"])),
                    dtxt=rel_f(gt.float().cpu(), dtxt_ref),
                    dextra=rel_f(e.grad.float().cpu(), dtxt_ref[Bs[rank]:]),
                    dtp=abs(float(modx.t_prime.grad) - mine["dt_prime"]) / abs(mine["dt_prime"]),
                    db=abs(float(modx.bias.grad) - mine["dbias"]) / abs(mine["dbias"])))

    # ---- extra images: they never leave their rank; their ids meet the texts of every rank, and a metrics step
    # publishes them for the other ranks' t2i hit test ----------------------------------------------------------------
    if args.extra_images:
        sys.path.insert(0, os.path.join(ROOT, "tests"))      # the oracle lives with the tests
        from extra_images_oracle import closed_form_extras, label_blocks, retrieval_metrics_extras
        Bs = [160 + 24 * r for r in range(world)]
        K, Kt, D, tp, bias = 200, 40, 136, math.log(10.0), -8.0
        Rs, Ts = [b + K for b in Bs], [b + Kt for b in Bs]
        g = torch.Generator().manual_seed(4545)
        unit = lambda n: torch.nn.functional.normalize(torch.randn(n, D, generator=g)).to(torch.bfloat16)  # noqa: E731
        imgs, txts = [unit(r) for r in Rs], [unit(t) for t in Ts]
        ids = [np.arange(sum(Bs[:r]), sum(Bs[:r + 1]), dtype=np.int64) * 2 for r in range(world)]
        xt = [ids[r][np.arange(Kt) % Bs[r]].copy() for r in range(world)]
        xi = []
        for r in range(world):   # extra image j of rank r: an image of a caption of rank (r + 1) % world, or of nothing
            e = ids[(r + 1) % world][np.arange(K) % Bs[(r + 1) % world]].copy()
            e[::4] = -1 - np.arange(len(e[::4]))
            xi.append(e)
        for multi in (False, True):
            labels = label_blocks(Bs, Rs, Ts, ids if multi else None, xt if multi else None, xi if multi else None)
            ref = closed_form_extras([x.float().numpy() for x in imgs], [x.float().numpy() for x in txts], Bs, tp, bias,
                                     labels)
            mine = ref[rank]
            dtxt_ref = torch.from_numpy(sum(ref[r]["contrib"][rank] for r in range(world)))
            met = retrieval_metrics_extras([x.float().numpy() for x in imgs], [x.float().numpy() for x in txts], Bs,
                                           ids if multi else None, xt if multi else None, xi if multi else None)[rank]
            img, txt = imgs[rank].to(dev), txts[rank].to(dev)
            for fused in (None, False):
                kw = dict(multi_positive=True, extra_texts=Kt) if multi else dict(hard_negatives=Kt)
                modx = DDPSigmoidLoss(Bs[rank], fused_step=fused, batch_per_rank=Bs, extra_images=K, **kw).to(dev)
                with torch.no_grad():
                    modx.t_prime.fill_(tp)
                    modx.bias.fill_(bias)
                for rep in range(2):
                    modx.zero_grad()
                    a, e = img[:Bs[rank]].float().requires_grad_(True), img[Bs[rank]:].float().requires_grad_(True)
                    b, x = txt[:Bs[rank]].float().requires_grad_(True), txt[Bs[rank]:].float().requires_grad_(True)
                    fw = dict(extra_image=e, return_metrics=True)
                    if multi:
                        fw.update(sample_ids=torch.from_numpy(ids[rank]).to(dev), extra_text=x,
                                  extra_text_ids=torch.from_numpy(xt[rank]).to(dev),
                                  extra_image_ids=torch.from_numpy(xi[rank]).to(dev))
                    else:
                        fw.update(negative_text=x)
                    l2, m = modx(a, b, **fw)
                    l2.backward()
                    torch.cuda.synchronize()
                    clear = met["t2i_margin"] > 1e-4
                    t2i_bad = int(((m["t2i_index"].cpu().numpy() != met["t2i_index"]) & clear).sum())
                    report(f"extra images ids={multi} {fused} B={Bs} K={K} D={D} rep{rep}", dict(
                        loss=abs(float(l2) - mine["loss"]) / abs(mine["loss"]),
                        dimg=rel_f(torch.cat([a.grad, e.grad]).float().cpu(), torch.from_numpy(mine["dimg"])),
                        dtxt=rel_f(torch.cat([b.grad, x.grad]).float().cpu(), dtxt_ref),
                        dtp=abs(float(modx.t_prime.grad) - mine["dt_prime"]) / abs(mine["dt_prime"]),
                        db=abs(float(modx.bias.grad) - mine["dbias"]) / abs(mine["dbias"]),
                        t2i_rows_off=float(t2i_bad)))

    # ---- per-sample weights: image weights stay local, text weights travel with the text through the peer pulls ----
    if args.weights:
        sys.path.insert(0, os.path.join(ROOT, "tests"))      # the oracle lives with the tests
        from sample_weights_oracle import closed_form_weighted, label_blocks
        Bs = [160 + 24 * r for r in range(world)]
        D, tp, bias = 136, math.log(10.0), -8.0
        g = torch.Generator().manual_seed(4444)
        unit = lambda n: torch.nn.functional.normalize(torch.randn(n, D, generator=g)).to(torch.bfloat16)  # noqa: E731
        for K, with_ids in ((0, False), (0, True), (37, True)):
            Ts = [b + K for b in Bs]
            imgs, texts = [unit(b) for b in Bs], [unit(t) for t in Ts]
            ids = list(torch.split(torch.randint(0, 200, (sum(Bs),), generator=g), Bs)) if with_ids else None

            def weights(n):
                w = torch.rand(n, generator=g)
                w[torch.rand(n, generator=g) < 0.1] = 0.0
                return w
            iws, tws = [weights(b) for b in Bs], [weights(t) for t in Ts]
            f = lambda xs: [x.double().numpy() for x in xs]  # noqa: E731
            ref = closed_form_weighted(f(imgs), f(texts), tp, bias, f(iws), f(tws),
                                       label_blocks(Bs, Ts, f(ids) if ids else None))
            mine = ref[rank]
            dtxt_ref = torch.from_numpy(sum(ref[r]["contrib"][rank] for r in range(world)))
            img, txt = imgs[rank].to(dev), texts[rank].to(dev)
            for fused in (None, False):
                modx = DDPSigmoidLoss(Bs[rank], fused_step=fused, batch_per_rank=Bs, multi_positive=with_ids,
                                      hard_negatives=K, sample_weights=True).to(dev)
                with torch.no_grad():
                    modx.t_prime.fill_(tp)
                    modx.bias.fill_(bias)
                for rep in range(2):
                    modx.zero_grad()
                    a, b = (x.float().requires_grad_(True) for x in (img, txt))
                    kw = dict(image_weights=iws[rank].to(dev), text_weights=tws[rank].to(dev))
                    if with_ids:
                        kw["sample_ids"] = ids[rank].to(dev)
                    if K:
                        l2 = modx(a, b[:Bs[rank]], negative_text=b[Bs[rank]:], **kw)
                    else:
                        l2 = modx(a, b, **kw)
                    l2.backward()
                    torch.cuda.synchronize()
                    report(f"weights {fused} B={Bs} K={K} ids={with_ids} D={D} rep{rep}", dict(
                        loss=abs(float(l2) - mine["loss"]) / abs(mine["loss"]),
                        dimg=rel_f(a.grad.float().cpu(), torch.from_numpy(mine["dimg"])),
                        dtxt=rel_f(b.grad.float().cpu(), dtxt_ref),
                        dtp=abs(float(modx.t_prime.grad) - mine["dt_prime"]) / abs(mine["dt_prime"]),
                        db=abs(float(modx.bias.grad) - mine["dbias"]) / abs(mine["dbias"])))

    # ---- excluded groups: each rank's text groups travel with its ids through the peer pulls ------------------------
    if args.exclude_groups:
        sys.path.insert(0, os.path.join(ROOT, "tests"))      # the oracle lives with the tests
        from exclude_groups_oracle import closed_form_groups, clustered, group_labels
        from sample_weights_oracle import label_blocks
        Bs = [160 + 24 * r for r in range(world)]
        D, tp, bias, n_groups = 136, math.log(10.0), -5.0, 7
        rng = np.random.default_rng(5555)
        for K, with_ids in ((0, False), (0, True), (37, False)):
            Ts = [b + K for b in Bs]
            tgs = [rng.integers(0, n_groups, t) for t in Ts]
            igs = [tg[:b].copy() for tg, b in zip(tgs, Bs)]   # image i shares text i's group
            imgs = [torch.from_numpy(clustered(ig, D, n_groups, 1, 10 + r)).to(torch.bfloat16) for r, ig in enumerate(igs)]
            texts = [torch.from_numpy(clustered(tg, D, n_groups, 1, 50 + r)).to(torch.bfloat16) for r, tg in enumerate(tgs)]
            for gr in igs + tgs:
                gr[rng.random(len(gr)) < 0.2] = -1
            ids = [torch.from_numpy(rng.integers(0, 200, b)) for b in Bs] if with_ids else None
            f = lambda xs: [x.double().numpy() for x in xs]  # noqa: E731
            labels = group_labels(label_blocks(Bs, Ts, [x.numpy() for x in ids] if ids else None), igs, tgs)
            ref = closed_form_groups(f(imgs), f(texts), tp, bias, labels, Bs)
            mine = ref[rank]
            dtxt_ref = torch.from_numpy(sum(ref[r]["contrib"][rank] for r in range(world)))
            img, txt = imgs[rank].to(dev), texts[rank].to(dev)
            for fused in (None, False):
                modx = DDPSigmoidLoss(Bs[rank], fused_step=fused, batch_per_rank=Bs, multi_positive=with_ids,
                                      hard_negatives=K, exclude_groups=True).to(dev)
                with torch.no_grad():
                    modx.t_prime.fill_(tp)
                    modx.bias.fill_(bias)
                for rep in range(2):
                    modx.zero_grad()
                    a, b = (x.float().requires_grad_(True) for x in (img, txt))
                    kw = dict(image_groups=torch.from_numpy(igs[rank]).to(dev),
                              text_groups=torch.from_numpy(tgs[rank]).to(dev))
                    if with_ids:
                        kw["sample_ids"] = ids[rank].to(dev)
                    if K:
                        l2 = modx(a, b[:Bs[rank]], negative_text=b[Bs[rank]:], **kw)
                    else:
                        l2 = modx(a, b, **kw)
                    l2.backward()
                    torch.cuda.synchronize()
                    report(f"exclude groups {fused} B={Bs} K={K} ids={with_ids} D={D} rep{rep}", dict(
                        loss=abs(float(l2) - mine["loss"]) / abs(mine["loss"]),
                        dimg=rel_f(a.grad.float().cpu(), torch.from_numpy(mine["dimg"])),
                        dtxt=rel_f(b.grad.float().cpu(), dtxt_ref),
                        dtp=abs(float(modx.t_prime.grad) - mine["dt_prime"]) / abs(mine["dt_prime"]),
                        db=abs(float(modx.bias.grad) - mine["dbias"]) / abs(mine["dbias"])))

    # ---- label sets: each rank's text sets travel with its ids slot through the peer pulls -------------------------
    if args.label_sets:
        sys.path.insert(0, os.path.join(ROOT, "tests"))      # the oracle lives with the tests
        from exclude_groups_oracle import clustered
        from label_sets_oracle import closed_form_sets, dense_labels, topk_retrieval_sets
        Bs = [160 + 24 * r for r in range(world)]
        D, tp, bias = 136, math.log(10.0), -5.0
        rng = np.random.default_rng(6666)
        for M, K, E in ((1, 0, 0), (4, 29, 0), (2, 0, 17)):
            Ts, Rs = [b + K for b in Bs], [b + E for b in Bs]
            ss = [rng.integers(0, 12, (b, M)) for b in Bs]
            for s_ in ss:
                s_[rng.random(s_.shape) < 0.3] = -1
            tsets = [np.concatenate([s_, rng.integers(-1, 12, (K, M))]) for s_ in ss]
            isets = [np.concatenate([s_, rng.integers(-1, 12, (E, M))]) for s_ in ss]
            key = lambda x: np.where(x[:, 0] >= 0, x[:, 0], 99)  # noqa: E731
            imgs = [torch.from_numpy(clustered(key(x), D, 13, 1, 10 + r)).to(torch.bfloat16) for r, x in enumerate(isets)]
            texts = [torch.from_numpy(clustered(key(x), D, 13, 1, 50 + r)).to(torch.bfloat16) for r, x in enumerate(tsets)]
            f = lambda xs: [x.double().numpy() for x in xs]  # noqa: E731
            ref = closed_form_sets(f(imgs), f(texts), tp, bias, isets, tsets, Bs)
            mine = ref[rank]
            dtxt_ref = torch.from_numpy(sum(ref[r]["contrib"][rank] for r in range(world)))
            img, txt = imgs[rank].to(dev), texts[rank].to(dev)
            B = Bs[rank]
            for fused in (None, False):
                modx = DDPSigmoidLoss(B, fused_step=fused, batch_per_rank=Bs, multi_label=M, extra_texts=K,
                                      extra_images=E).to(dev)
                with torch.no_grad():
                    modx.t_prime.fill_(tp)
                    modx.bias.fill_(bias)
                for rep in range(2):
                    modx.zero_grad()
                    a, b = (x.float().requires_grad_(True) for x in (img, txt))
                    kw = dict(sample_labels=torch.from_numpy(isets[rank][:B]).to(dev))
                    if K:
                        kw.update(extra_text=b[B:], extra_text_labels=torch.from_numpy(tsets[rank][B:]).to(dev))
                    if E:
                        kw.update(extra_image=a[B:], extra_image_labels=torch.from_numpy(isets[rank][B:]).to(dev))
                    kq = 3
                    if rep == 0:   # retrieval over the real peers: published text and extra-image sets
                        l2, met = modx(a[:B], b[:B], return_metrics=True, metrics_topk=kq, **kw)
                    else:
                        l2 = modx(a[:B], b[:B], **kw)
                    l2.backward()
                    torch.cuda.synchronize()
                    if rep == 0:
                        exp = topk_retrieval_sets(f(imgs), f(texts), Bs, kq, isets, tsets)[rank]
                        Y = dense_labels(isets, tsets, Bs) > 0
                        o, to = exp["off"][rank], exp["toff"][rank]
                        got_i = met["i2t_topk"].cpu().numpy()
                        got_t = met["t2i_topk"].cpu().numpy()

                        def clear(v):
                            top = np.sort(v)[::-1][:kq + 1]
                            return float(np.min(top[:-1] - top[1:])) > 1e-4

                        ci = np.array([clear(exp["S"][o + i]) for i in range(len(got_i))])
                        ct = np.array([clear(exp["S"][:, to + j]) for j in range(len(got_t))])
                        fi = np.array([next((q for q, j in enumerate(row) if Y[o + i, j]), kq)
                                       for i, row in enumerate(got_i)])
                        ft = np.array([next((q for q, g in enumerate(row) if Y[g, to + j]), kq)
                                       for j, row in enumerate(got_t)])
                        rec = np.concatenate([met["i2t_recall"].cpu().numpy(), met["t2i_recall"].cpu().numpy()])
                        want = [np.float32(np.count_nonzero(x < q)) / np.float32(len(x)) for x in (fi, ft)
                                for q in range(1, kq + 1)]
                        report(f"label sets retrieval B={Bs} M={M} K={K} E={E}", dict(
                            i2t_lists=float((got_i[ci] != exp["i2t_topk"][ci]).any(axis=1).mean()),
                            t2i_lists=float((got_t[ct] != exp["t2i_topk"][ct]).any(axis=1).mean()),
                            unclear=float(max(0.8 - ci.mean(), 0.8 - ct.mean(), 0.0)),
                            recall=float(np.abs(rec - np.array(want, np.float32)).max())), tol=0.0)
                    report(f"label sets {fused} B={Bs} M={M} K={K} E={E} D={D} rep{rep}", dict(
                        loss=abs(float(l2) - mine["loss"]) / abs(mine["loss"]),
                        dimg=rel_f(a.grad.float().cpu(), torch.from_numpy(mine["dimg"])),
                        dtxt=rel_f(b.grad.float().cpu(), dtxt_ref),
                        dtp=abs(float(modx.t_prime.grad) - mine["dt_prime"]) / abs(mine["dt_prime"]),
                        db=abs(float(modx.bias.grad) - mine["dbias"]) / abs(mine["dbias"])))

    # ---- focal pair loss: gamma and alpha are kernel parameters; the exchange is the one of the options it rides ----
    if args.focal:
        sys.path.insert(0, os.path.join(ROOT, "tests"))      # the oracle lives with the tests
        from exclude_groups_oracle import clustered, group_labels
        from focal_oracle import closed_form_focal
        from label_sets_oracle import set_labels
        Bs = [160 + 24 * r for r in range(world)]
        D, tp, bias = 136, math.log(10.0), -5.0
        rng = np.random.default_rng(7777)
        for gamma, alpha, M, K, E, extra in ((2.0, 0.25, 0, 0, 0, False), (5.0, None, 2, 29, 17, False),
                                             (0.5, 0.25, 0, 0, 0, True)):
            Ts, Rs = [b + K for b in Bs], [b + E for b in Bs]
            ss = [rng.integers(-1, 12, (b, max(M, 1))) for b in Bs]
            tsets = [np.concatenate([s_, rng.integers(-1, 12, (K, max(M, 1)))]) for s_ in ss]
            isets = [np.concatenate([s_, rng.integers(-1, 12, (E, max(M, 1)))]) for s_ in ss]
            key = lambda x: np.where(x[:, 0] >= 0, x[:, 0], 99)  # noqa: E731
            imgs = [torch.from_numpy(clustered(key(x), D, 13, 1, 20 + r)).to(torch.bfloat16) for r, x in enumerate(isets)]
            texts = [torch.from_numpy(clustered(key(x), D, 13, 1, 60 + r)).to(torch.bfloat16) for r, x in enumerate(tsets)]
            f = lambda xs: [x.double().numpy() for x in xs]  # noqa: E731
            if M:
                lab = set_labels(isets, tsets, Bs)
            else:
                lab = [[np.where((np.arange(Rs[r])[:, None] == np.arange(Ts[c])[None, :]) & (r == c), 1.0, -1.0)
                        for c in range(world)] for r in range(world)]
            iws = tws = igs = tgs = None
            if extra:   # weights and excluded groups
                iws = [rng.random(r_) for r_ in Rs]
                tws = [rng.random(t_) for t_ in Ts]
                igs = [rng.integers(-1, 6, r_) for r_ in Rs]
                tgs = [rng.integers(-1, 6, t_) for t_ in Ts]
                lab = group_labels(lab, igs, tgs)
            ref = closed_form_focal(f(imgs), f(texts), tp, bias, lab, gamma, alpha, Bs, iws, tws)
            mine = ref[rank]
            dtxt_ref = torch.from_numpy(sum(ref[r]["contrib"][rank] for r in range(world)))
            img, txt = imgs[rank].to(dev), texts[rank].to(dev)
            B = Bs[rank]
            for fused in (None, False):
                modx = DDPSigmoidLoss(B, fused_step=fused, batch_per_rank=Bs, multi_label=M or None, extra_texts=K,
                                      extra_images=E, sample_weights=extra, exclude_groups=extra, focal_gamma=gamma,
                                      focal_alpha=alpha).to(dev)
                with torch.no_grad():
                    modx.t_prime.fill_(tp)
                    modx.bias.fill_(bias)
                for rep in range(2):
                    modx.zero_grad()
                    a, b = (x.float().requires_grad_(True) for x in (img, txt))
                    kw = {}
                    if M:
                        kw["sample_labels"] = torch.from_numpy(isets[rank][:B]).to(dev)
                    if K:
                        kw.update(extra_text=b[B:], extra_text_labels=torch.from_numpy(tsets[rank][B:]).to(dev))
                    if E:
                        kw.update(extra_image=a[B:], extra_image_labels=torch.from_numpy(isets[rank][B:]).to(dev))
                    if extra:
                        kw.update(image_weights=torch.from_numpy(iws[rank]).float().to(dev),
                                  text_weights=torch.from_numpy(tws[rank]).float().to(dev),
                                  image_groups=torch.from_numpy(igs[rank]).to(dev),
                                  text_groups=torch.from_numpy(tgs[rank]).to(dev))
                    l2 = modx(a[:B] if E else a, b[:B] if K else b, **kw)
                    l2.backward()
                    torch.cuda.synchronize()
                    report(f"focal {fused} gamma={gamma} alpha={alpha} B={Bs} M={M} K={K} E={E} w/g={extra} rep{rep}",
                           dict(loss=abs(float(l2) - mine["loss"]) / abs(mine["loss"]),
                                dimg=rel_f(a.grad.float().cpu(), torch.from_numpy(mine["dimg"])),
                                dtxt=rel_f(b.grad.float().cpu(), dtxt_ref),
                                dtp=abs(float(modx.t_prime.grad) - mine["dt_prime"]) / abs(mine["dt_prime"]),
                                db=abs(float(modx.bias.grad) - mine["dbias"]) / abs(mine["dbias"])))

    # ---- distillation: each rank's teacher text travels with its text through the peer pulls ----------------------
    if args.distill:
        sys.path.insert(0, os.path.join(ROOT, "tests"))      # the oracle lives with the tests
        from distill_oracle import closed_form_distill
        from sample_weights_oracle import label_blocks
        Bs = [160 + 24 * r for r in range(world)]
        D, DT, tp, bias, ttp, tbias, lam = 136, 72, math.log(10.0), -8.0, math.log(20.0), -6.0, 0.7
        g = torch.Generator().manual_seed(5555)
        unit = lambda n, d: torch.nn.functional.normalize(torch.randn(n, d, generator=g)).to(torch.bfloat16)  # noqa: E731
        for with_ids, with_w in ((False, False), (True, True)):
            imgs, texts = [unit(b, D) for b in Bs], [unit(b, D) for b in Bs]
            timgs, ttexts = [unit(b, DT) for b in Bs], [unit(b, DT) for b in Bs]
            ids = list(torch.split(torch.randint(0, 200, (sum(Bs),), generator=g), Bs)) if with_ids else None
            iws = [torch.rand(b, generator=g) for b in Bs] if with_w else None
            tws = [torch.rand(b, generator=g) for b in Bs] if with_w else None
            f = lambda xs: None if xs is None else [x.double().numpy() for x in xs]  # noqa: E731
            ref = closed_form_distill(f(imgs), f(texts), tp, bias, f(timgs), f(ttexts), ttp, tbias, lam, f(iws), f(tws),
                                      label_blocks(Bs, Bs, f(ids)))
            mine = ref[rank]
            dtxt_ref = torch.from_numpy(sum(ref[r]["contrib"][rank] for r in range(world)))
            img, txt = imgs[rank].to(dev), texts[rank].to(dev)
            for fused in (None, False):
                modx = DDPSigmoidLoss(Bs[rank], fused_step=fused, batch_per_rank=Bs, multi_positive=with_ids,
                                      sample_weights=with_w, distill=lam).to(dev)
                with torch.no_grad():
                    modx.t_prime.fill_(tp)
                    modx.bias.fill_(bias)
                for rep in range(2):
                    modx.zero_grad()
                    # fp32 student inputs (fp16 operands, fp32 gradients), bf16 teacher: two operand formats in one step
                    a, b = (x.float().requires_grad_(True) for x in (img, txt))
                    kw = dict(teacher_image=timgs[rank].to(dev), teacher_text=ttexts[rank].to(dev),
                              teacher_t_prime=torch.tensor(ttp, device=dev), teacher_bias=torch.tensor(tbias, device=dev))
                    if with_ids:
                        kw["sample_ids"] = ids[rank].to(dev)
                    if with_w:
                        kw.update(image_weights=iws[rank].to(dev), text_weights=tws[rank].to(dev))
                    l2 = modx(a, b, **kw)
                    l2.backward()
                    torch.cuda.synchronize()
                    report(f"distill {fused} B={Bs} D={D} D_T={DT} ids={with_ids} weights={with_w} rep{rep}", dict(
                        loss=abs(float(l2) - mine["loss"]) / abs(mine["loss"]),
                        dimg=rel_f(a.grad.float().cpu(), torch.from_numpy(mine["dimg"])),
                        dtxt=rel_f(b.grad.float().cpu(), dtxt_ref),
                        dtp=abs(float(modx.t_prime.grad) - mine["dt_prime"]) / abs(mine["dt_prime"]),
                        db=abs(float(modx.bias.grad) - mine["dbias"]) / abs(mine["dbias"])))

    # ---- distillation with the other options: the teacher's rows of the extras travel with the text ----------------
    if args.distill_options:
        sys.path.insert(0, os.path.join(ROOT, "tests"))      # the oracle lives with the tests
        from distill_options_oracle import closed_form_distill_options
        from exclude_groups_oracle import group_labels
        from extra_images_oracle import label_blocks as xlabel_blocks
        from label_sets_oracle import set_labels
        Bs = [160 + 24 * r for r in range(world)]
        D, DT, tp, bias, ttp, tbias, lam = 136, 72, math.log(10.0), -8.0, math.log(20.0), -6.0, 0.6
        g = torch.Generator().manual_seed(6666)
        rng = np.random.default_rng(6666)
        unit = lambda n, d: torch.nn.functional.normalize(torch.randn(n, d, generator=g)).to(torch.bfloat16)  # noqa: E731
        for kind, K, E in (("negatives", 48, 0), ("sets", 29, 17)):
            Ts, Rs = [b + K for b in Bs], [b + E for b in Bs]
            imgs, texts = [unit(r_, D) for r_ in Rs], [unit(t_, D) for t_ in Ts]
            timgs, ttexts = [unit(r_, DT) for r_ in Rs], [unit(t_, DT) for t_ in Ts]
            if kind == "sets":
                ss = [rng.integers(-1, 12, (b, 2)) for b in Bs]
                tsets = [np.concatenate([s_, rng.integers(-1, 12, (K, 2))]) for s_ in ss]
                isets = [np.concatenate([s_, rng.integers(-1, 12, (E, 2))]) for s_ in ss]
                lab = set_labels(isets, tsets, Bs)
            else:
                lab = xlabel_blocks(Bs, Rs, Ts)
            iws = [rng.random(r_) for r_ in Rs]
            tws = [rng.random(t_) for t_ in Ts]
            igs = [rng.integers(-1, 6, r_) for r_ in Rs]
            tgs = [rng.integers(-1, 6, t_) for t_ in Ts]
            lab = group_labels(lab, igs, tgs)
            f = lambda xs: [x.double().numpy() for x in xs]  # noqa: E731
            ref = closed_form_distill_options(f(imgs), f(texts), tp, bias, f(timgs), f(ttexts), ttp, tbias, lam, lab, Bs,
                                              iws, tws)
            mine = ref[rank]
            dtxt_ref = torch.from_numpy(sum(ref[r]["contrib"][rank] for r in range(world)))
            tl_ref = torch.from_numpy(sum(ref[r]["text_part"][rank] for r in range(world)))
            img, txt = imgs[rank].to(dev), texts[rank].to(dev)
            B = Bs[rank]
            for fused in (None, False):
                modx = DDPSigmoidLoss(B, fused_step=fused, batch_per_rank=Bs, multi_label=2 if kind == "sets" else None,
                                      hard_negatives=K if kind == "negatives" else 0,
                                      extra_texts=K if kind == "sets" else 0, extra_images=E, sample_weights=True,
                                      exclude_groups=True, distill=lam, distill_options=True).to(dev)
                with torch.no_grad():
                    modx.t_prime.fill_(tp)
                    modx.bias.fill_(bias)
                for rep in range(2):
                    modx.zero_grad()
                    a, b = (x.float().requires_grad_(True) for x in (img, txt))
                    ti, tt = timgs[rank].to(dev), ttexts[rank].to(dev)
                    kw = dict(teacher_image=ti[:B], teacher_text=tt[:B], teacher_t_prime=torch.tensor(ttp, device=dev),
                              teacher_bias=torch.tensor(tbias, device=dev),
                              image_weights=torch.from_numpy(iws[rank]).float().to(dev),
                              text_weights=torch.from_numpy(tws[rank]).float().to(dev),
                              image_groups=torch.from_numpy(igs[rank]).to(dev),
                              text_groups=torch.from_numpy(tgs[rank]).to(dev))
                    if kind == "negatives":
                        kw.update(negative_text=b[B:], teacher_negative_text=tt[B:])
                    else:
                        kw.update(sample_labels=torch.from_numpy(isets[rank][:B]).to(dev),
                                  extra_text=b[B:], teacher_extra_text=tt[B:],
                                  extra_text_labels=torch.from_numpy(tsets[rank][B:]).to(dev),
                                  extra_image=a[B:], teacher_extra_image=ti[B:],
                                  extra_image_labels=torch.from_numpy(isets[rank][B:]).to(dev))
                    l2, sl = modx(a[:B] if E else a, b[:B], return_sample_losses=True, **kw)
                    l2.backward()
                    torch.cuda.synchronize()
                    report(f"distill-options {kind} {fused} B={Bs} K={K} E={E} rep{rep}", dict(
                        loss=abs(float(l2) - mine["loss"]) / abs(mine["loss"]),
                        dimg=rel_f(a.grad.float().cpu(), torch.from_numpy(mine["dimg"])),
                        dtxt=rel_f(b.grad.float().cpu(), dtxt_ref),
                        dtp=abs(float(modx.t_prime.grad) - mine["dt_prime"]) / abs(mine["dt_prime"]),
                        db=abs(float(modx.bias.grad) - mine["dbias"]) / abs(mine["dbias"]),
                        image_loss=rel_f(sl["image_loss"].cpu(), torch.from_numpy(mine["image_loss"])),
                        text_loss=rel_f(sl["text_loss"].cpu(), tl_ref)))

    # ---- larger: fp32 autograd; dtxt reference summed over ranks ------------------------------------------
    B, D, tp, bias = 2048, 768, math.log(10.0), -10.0
    g = torch.Generator().manual_seed(1234 + rank)
    img = torch.nn.functional.normalize(torch.randn(B, D, generator=g)).to(torch.bfloat16).to(dev)
    txt = torch.nn.functional.normalize(torch.randn(B, D, generator=g)).to(torch.bfloat16).to(dev)
    chunks = [torch.empty_like(txt) for _ in range(world)]
    dist.all_gather(chunks, txt)
    ref = torch_reference_fp32(img, chunks, tp, bias, rank)
    contrib = torch.stack(ref["dtxt_chunks"])             # [W, B, D] this rank's contributions
    dist.all_reduce(contrib)                              # sum over ranks
    mod = DDPSigmoidLoss(B).to(dev)
    eng = mod.engine_for(B, D, dev)
    loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, torch.tensor([tp], device=dev), torch.tensor([bias], device=dev))
    torch.cuda.synchronize()
    report(f"fp32-autograd B={B} D={D}", dict(
        loss=abs(float(loss) - ref["loss"]) / abs(ref["loss"]),
        dimg=rel_f(dimg, ref["dimg"]), dtxt=rel_f(dtxt, contrib[rank]),
        dtp=abs(float(dtp) - ref["dt_prime"]) / abs(ref["dt_prime"]),
        db=abs(float(db) - ref["dbias"]) / abs(ref["dbias"])))

    # ---- the reference's own acceptance test on GPUs: encoder-weight gradients of the W-rank job, averaged over the
    # ranks, equal those of ONE rank holding the whole batch (test_distributed_sigmoid_loss.py:122-141 test_same_gradient;
    # toy linear encoders :71-77, seeds 42 / 40 and the row partition :55-68, gradient averaging :79-83). fp32 leaves,
    # like the reference feeds them; output widths 64 and the reference's own 2 (padded to 8 inside the module) ----------
    if not args.skip_parity:
        groups = [dist.new_group([q]) for q in range(world)]       # collective: every rank creates every 1-rank group
        for out_dim in (64, 2):
            in_dim, bpr = 32, 32
            torch.manual_seed(42)
            x_img = torch.randn(world * bpr, in_dim)
            torch.manual_seed(40)
            x_txt = torch.randn(world * bpr, in_dim)

            def run(rows, group, batch):
                torch.manual_seed(42)
                enc_i = torch.nn.Linear(in_dim, out_dim, bias=False).to(dev)
                torch.manual_seed(42)
                enc_t = torch.nn.Linear(in_dim, out_dim, bias=False).to(dev)
                mod_ = DDPSigmoidLoss(batch, group=group).to(dev)
                e_i = torch.nn.functional.normalize(enc_i(x_img[rows].to(dev)))
                e_t = torch.nn.functional.normalize(enc_t(x_txt[rows].to(dev)))
                mod_(e_i, e_t).backward()
                return [enc_i.weight.grad, enc_t.weight.grad, mod_.t_prime.grad.float().reshape(1),
                        mod_.bias.grad.reshape(1)]

            multi = run(slice(rank * bpr, (rank + 1) * bpr), None, bpr)
            for gr in multi:                                        # average_gradients
                dist.all_reduce(gr)
                gr /= world
            single = run(slice(0, world * bpr), groups[rank], world * bpr)
            torch.cuda.synchronize()
            report(f"same_gradient (reference's test) out_dim={out_dim}", dict(
                img_encoder=rel_f(multi[0], single[0]), txt_encoder=rel_f(multi[1], single[1]),
                t_prime=abs(float(multi[2]) - float(single[2])) / abs(float(single[2])),
                bias=abs(float(multi[3]) - float(single[3])) / abs(float(single[3]))))

    # ---- a late rank: the last rank arrives 2.5 s after the others; they wait INSIDE their kernels (bounded by
    # SIGLIP_OPT_PEER_TIMEOUT_MS, minutes by default) and the step still gives the same numbers -----------------------
    import time
    dist.barrier()
    torch.cuda.synchronize()
    if rank == world - 1:
        time.sleep(2.5)
    t0 = time.perf_counter()
    loss_l, dimg_l, dtxt_l, dtp_l, db_l = eng.fwd_bwd(img, txt, torch.tensor([tp], device=dev),
                                                      torch.tensor([bias], device=dev))
    torch.cuda.synchronize()
    waited = time.perf_counter() - t0
    report("late rank (2.5 s)", dict(
        loss=abs(float(loss_l) - ref["loss"]) / abs(ref["loss"]),
        dimg=rel_f(dimg_l, ref["dimg"]), dtxt=rel_f(dtxt_l, contrib[rank]),
        bitwise_vs_on_time=0.0 if (torch.equal(dimg_l, dimg) and torch.equal(dtxt_l, dtxt)) else 1.0,
        waited_too_little=0.0 if (rank == world - 1 or waited > 2.0) else 1.0))

    # ---- SURVEY §8f-2: mean over ranks of the scalar gradients inside the backward (no DDP wrapper needed) -----
    both = torch.stack([dtp.reshape(()), db.reshape(())]).double()
    dist.all_reduce(both)
    both /= world
    eng.set_option(_capi.SIGLIP_OPT_SYNC_SCALAR_GRADS, 1)
    for rep in range(3):
        _, _, _, dtp_m, db_m = eng.fwd_bwd(img, txt, torch.tensor([tp], device=dev), torch.tensor([bias], device=dev))
        torch.cuda.synchronize()
        mine = torch.stack([dtp_m.reshape(()), db_m.reshape(())])
        gathered = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(gathered, mine)
        identical = all(torch.equal(gathered[0], x) for x in gathered)
        report(f"scalar-grad mean rep{rep}", dict(
            dtp=abs(float(dtp_m) - float(both[0])) / abs(float(both[0])),
            db=abs(float(db_m) - float(both[1])) / abs(float(both[1])),
            not_bit_identical=0.0 if identical else 1.0), tol=1e-5)
    eng.set_option(_capi.SIGLIP_OPT_SYNC_SCALAR_GRADS, 0)

    # ---- SURVEY §8f-3: bidirectional visiting order (same pairs, other order) against the same fp32 autograd ----
    eng.set_option(_capi.SIGLIP_OPT_BIDIR, 1)
    for rep in range(2):
        loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, torch.tensor([tp], device=dev), torch.tensor([bias], device=dev))
        torch.cuda.synchronize()
        report(f"bidir order rep{rep} B={B} D={D}", dict(
            loss=abs(float(loss) - ref["loss"]) / abs(ref["loss"]),
            dimg=rel_f(dimg, ref["dimg"]), dtxt=rel_f(dtxt, contrib[rank]),
            dtp=abs(float(dtp) - ref["dt_prime"]) / abs(ref["dt_prime"]),
            db=abs(float(db) - ref["dbias"]) / abs(ref["dbias"])))
    eng.set_option(_capi.SIGLIP_OPT_BIDIR, 0)

    # ---- timing at the headline per-rank shape -------------------------------------------------------------
    if args.time:
        B, D = args.batch, args.dim
        g = torch.Generator().manual_seed(1234 + rank)
        img = torch.nn.functional.normalize(torch.randn(B, D, generator=g)).to(torch.bfloat16).to(dev)
        txt = torch.nn.functional.normalize(torch.randn(B, D, generator=g)).to(torch.bfloat16).to(dev)
        mod = DDPSigmoidLoss(B).to(dev)
        eng = mod.engine_for(B, D, dev)
        tpt, bt = torch.tensor([math.log(10.0)], device=dev), torch.tensor([-10.0], device=dev)
        from distributed_sigmoid_loss_b200 import SigmoidLossEngine

        def timed(engine, label):
            for _ in range(3):
                engine.fwd_bwd(img, txt, tpt, bt, torch.bfloat16)
            dist.barrier()
            torch.cuda.synchronize()
            engine.set_option(_capi.SIGLIP_OPT_KERNEL_TIMING, 1)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                engine.fwd_bwd(img, txt, tpt, bt, torch.bfloat16)
            e1.record()
            torch.cuda.synchronize()
            lm, ln, gm, gn = engine.kernel_times()
            engine.set_option(_capi.SIGLIP_OPT_KERNEL_TIMING, 0)
            t = torch.tensor([e0.elapsed_time(e1) / args.steps], device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            w = engine.world
            if rank == 0:
                ms = float(t)
                print(f"[time {label} W={w}] B={B} D={D}: {ms:.3f} ms/step ({ms / w:.3f} per chunk) "
                      f"{w * B / ms * 1e3 / 1e6:.2f} Mpairs/s (global) {6.0 * B * w * B * D / ms / 1e9:.1f} TFLOP/s per GPU; "
                      f"loss kernel {lm / max(ln, 1):.3f} ms, gradient kernel {gm / max(gn, 1):.3f} ms (rank 0)",
                      flush=True)
            return float(t)

        single = SigmoidLossEngine(B, D, dev, rank_world=(0, 1))
        t1 = timed(single, "single-GPU baseline on every rank")
        single.close()
        eng.set_option(_capi.SIGLIP_OPT_OVERLAP_PULL, 1)
        eng.set_option(_capi.SIGLIP_OPT_OVERLAP_REDUCE, 1)
        tw = timed(eng, "in-kernel pull + progressive reduce")
        if rank == 0:
            print(f"[time] FLOP-normalised weak-scaling efficiency W*t(1)/t(W) = {world * t1 / tw:.3f}", flush=True)
        if args.all_variants:
            eng.set_option(_capi.SIGLIP_OPT_OVERLAP_REDUCE, 0)
            timed(eng, "in-kernel pull, reduction at the end")
            eng.set_option(_capi.SIGLIP_OPT_OVERLAP_PULL, 0)
            timed(eng, "separate copy, reduction at the end")
    # ---- soak: thousands of steps through the cross-rank protocol (monotonic flags, tickets, buffer hand-over) --------
    if args.soak > 0:
        B, D = args.batch, args.dim
        g = torch.Generator().manual_seed(4321 + rank)
        img = torch.nn.functional.normalize(torch.randn(B, D, generator=g)).to(torch.bfloat16).to(dev)
        txt = torch.nn.functional.normalize(torch.randn(B, D, generator=g)).to(torch.bfloat16).to(dev)
        mod = DDPSigmoidLoss(B).to(dev)
        eng = mod.engine_for(B, D, dev)
        tpt, bt = torch.tensor([math.log(10.0)], device=dev), torch.tensor([-10.0], device=dev)
        first = {}
        bad = 0
        import time
        dist.barrier()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pattern = ["fused", "fused", "fused", "split", "fused", "fwd", "fused", "fused"]
        for i in range(args.soak):
            kind = pattern[i % len(pattern)]
            if kind == "fused":
                out = eng.fwd_bwd(img, txt, tpt, bt, torch.bfloat16)
                res = (out[0], out[1], out[2], out[3], out[4])
            elif kind == "split":
                l_ = eng.forward(img, txt, tpt, bt, True)
                d_ = eng.backward(img, txt, tpt, None, torch.bfloat16)
                res = (l_, d_[0], d_[1], d_[2], d_[3])
            else:
                res = (eng.fwd(img, txt, tpt, bt),)
            if kind not in first:
                first[kind] = [x.clone() for x in res]
            elif i % 97 == 0 or i >= args.soak - len(pattern):      # spot checks + the last round of every kind
                bad += sum(0 if torch.equal(a, b) else 1 for a, b in zip(res, first[kind]))
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        # fused vs split schedule: loss, dimg and the scalars are the same arithmetic (bitwise); the text gradient adds the
        # same fp32 terms, the fused step with one rounding less (own term and folded peer sum meet in one fma of the
        # last gradient kernel's epilogue instead of a separate add): equal to the last bit or two, not bitwise
        f_, s_ = first["fused"], first["split"]
        same = all(torch.equal(f_[i], s_[i]) for i in (0, 1, 3, 4))
        report(f"soak {args.soak} steps B={B} D={D} ({dt:.1f} s)", dict(
            steps_that_differ_from_their_first=float(bad), fused_vs_split_not_bitwise=0.0 if same else 1.0,
            fused_vs_split_dtxt=rel_f(f_[2].float(), s_[2].float()) * 1e4), tol=0.5)
        # (x 1e4: the bf16 text gradients of the two schedules within 5e-5 relative Frobenius — an fp32 last-bit
        # difference flips the bf16 rounding of about one element in 2^16: measured 1.2e-5)
        eng.close()

    flag = torch.tensor([0 if ok else 1], device=dev)
    dist.all_reduce(flag)
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0:
        print("MULTI-GPU CHECK", "PASS" if int(flag) == 0 else "FAIL", flush=True)
    return 0 if int(flag) == 0 else 1


if __name__ == "__main__":
    sys.exit(main())
