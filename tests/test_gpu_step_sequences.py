"""Step sequences on one long-lived context on the H100 (tests/step_sequences.py), against the float64 oracle at every
step, and a DDPSigmoidLoss trained over several steps against float64 autograd at each step's actual parameters.

Per step of a sequence: fresh planted data, t', bias, lambda and upstream gradient; the options and knobs the step
changes; at W > 1 fresh loopback peers (their chunks, keys, lists, partials), fresh contributions to this rank's text
gradient and, under SIGLIP_OPT_SYNC_SCALAR_GRADS, fresh mailboxes holding the peers' own dt' and dbias. Checked: loss,
dimg, the own chunk's dtxt (less the seeded contributions) and the outgoing slots, dt' and dbias within 1e-3 (bf16
gradients within 1e-3 + 2^-8); per-sample losses within 1e-3 plus the fixed-point words; top-1, top-K lists and recall
exactly. Request buffers hold sentinels before they are armed; after an unarmed step the last request's buffers still
hold what it wrote; the launches of every step equal those of the same step repeated on a fresh context (a request left
armed, or a step that runs another's work, shows there). A refused step must leave its armed buffers untouched through the
next step, which is checked like any other.

Observed on one H100 80GB HBM3 (700 W power limit): the 16 sequences (115 steps), the two module runs and the three
engine refusals in 34 s of wall time; the largest relative errors: loss 3.5e-7, dimg 1.5e-4 (bf16 output 3.5e-3),
dtxt 1.1e-4 (bf16 3.1e-3), dtxt - sum C 2.0e-4 (bf16 5.6e-3), outgoing slots 1.6e-4, dt' 6.8e-7, dbias 7.6e-7, the
evaluation forward's loss 3.3e-7; the modules' loss 1.8e-7, bf16 gradients 3.2e-3 (their tolerance: 4e-3), dt' 6.4e-7,
dbias 9.6e-7."""
import dataclasses

import numpy as np
import pytest
import torch

import loopback_exchange as lx
import option_matrix as om
import step_sequences as ss
from exclude_groups_oracle import operand_values, torch_loss
from test_gpu_option_matrix import _check_sample_losses, _f32, _i64, _operand, _scal, _seed_peers

pytestmark = pytest.mark.gpu

BF16_TOL = om.TOL + 2.0 ** -8
OBSERVED = {}
# set_option order: what depends on an option is turned off before it and on after it
OFF_FIRST = ("FOCAL", "DISTILL", "EXTRA_TEXT_IDS", "EXTRA_IMAGE_IDS", "SAMPLE_IDS", "LABEL_SETS")
ON_LAST = ("LABEL_SETS", "SAMPLE_IDS", "EXTRA_TEXT_IDS", "EXTRA_IMAGE_IDS", "DISTILL", "FOCAL")
BY_DTYPE = ("INPUT_F16", "TPRIME_F64", "GRAD_BF16")   # the engine sets these from the tensors it is given
SENTINEL = {torch.float32: -1.0, torch.int64: -7}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(OBSERVED):
        print(f"step sequences: largest relative error of {k}: {OBSERVED[k]:.3e}")


def _dev():
    return torch.device("cuda", 0)


def _check(tag, kind, got, ref, tol):
    got = got.double().cpu().numpy() if torch.is_tensor(got) else np.asarray(got, np.float64)
    err = om.rel(got, ref)
    OBSERVED[kind] = max(OBSERVED.get(kind, 0.0), err)
    assert err <= tol, f"{tag} {kind}: relative error {err:.3e} (tolerance {tol:.2e})"


def _engine(seq):
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine

    Bs, Rs, Ts = seq.cell(seq.steps[0]).shapes()
    kw = dict(cta_group=2, rank_world=(seq.r, seq.W), loopback=seq.W > 1, batch_per_rank=Bs, labels=seq.M)
    if seq.teacher:
        kw.update(teacher_dim=om.DT, distill_options=seq.teacher == "extras")
    if Rs != Bs:
        kw.update(images_per_rank=Rs, texts_per_rank=Ts)
    elif Ts != Bs:
        kw["texts_per_rank"] = Ts
    return SigmoidLossEngine(Bs[seq.r], om.D, _dev(), **kw)


def _apply(eng, held, want):
    """Sets every option whose value differs from what the context holds (`held`, updated)."""
    from distributed_sigmoid_loss_b200 import _capi

    todo = {k: v for k, v in want.items() if k not in BY_DTYPE and held.get(k, ss.DEFAULTS[k]) != v}
    order = ([k for k in OFF_FIRST if k in todo and not todo[k]] + [k for k in todo if k not in OFF_FIRST] +
             [k for k in ON_LAST if k in todo and todo[k]])
    for k in order:
        eng.set_option(getattr(_capi, f"SIGLIP_OPT_{k}"), int(todo[k]))
        held[k] = todo[k]


def _inputs(eng, seq, st, P, skip=None):
    """The step's own inputs, given before every step; `skip` leaves out the one a take_ids refusal needs missing.
    Returns the teacher tensors, which must live until the step is enqueued."""
    o, r = st.opts, seq.r
    Bs, Rs, Ts, _, _ = P.view(o)
    if o.labels and skip != "sets":
        isets, tsets = P.sets(o)
        eng.set_label_sets(_i64(isets[r][:Bs[r]]), _i64(tsets[r][Bs[r]:]) if o.xt_sets else None,
                           _i64(isets[r][Bs[r]:]) if o.xi_sets else None)
    if o.ids and skip != "ids":
        eng.set_sample_ids(_i64(P.ids[r]))
    if o.xt_ids and skip != "extra_text_ids":
        eng.set_extra_text_ids(_i64(P.xt_ids[r][:Ts[r] - Bs[r]]))
    if o.xi_ids and skip != "extra_image_ids":
        eng.set_extra_image_ids(_i64(P.xi_ids[r][:Rs[r] - Bs[r]]))
    if o.weights and skip != "weights":
        eng.set_sample_weights(_f32(P.iw[r][:Rs[r]]), _f32(P.tw[r][:Ts[r]]))
    if o.groups and skip != "groups":
        eng.set_groups(_i64(P.ig[r][:Rs[r]]), _i64(P.tg[r][:Ts[r]]))
    if o.focal is not None and skip != "focal":
        eng.set_focal(*o.focal)
    if o.teacher and skip != "teacher":
        timgs, ttxts = P.teacher(o)
        teacher = (_operand(timgs[r], st.f16), _operand(ttxts[r], st.f16), _scal(om.TTP), _scal(om.TBIAS))
        eng.set_teacher(*teacher, st.lam)
        return teacher
    return None


def _arm(eng, o):
    """Request buffers filled with sentinels, armed for the next step."""
    dev, out = _dev(), {}
    if o.metrics:
        out["top1"] = torch.full((2,), -1.0, device=dev)
        out["i2t"] = torch.full((eng.metric_images,), -7, dtype=torch.int64, device=dev)
        out["t2i"] = torch.full((eng.metric_texts,), -7, dtype=torch.int64, device=dev)
        eng.request_metrics(out["top1"], out["i2t"], out["t2i"])
    if o.topk:
        k = o.topk
        out["recall"] = torch.full((2 * k,), -1.0, device=dev)
        out["i2t_k"] = torch.full((eng.metric_images, k), -7, dtype=torch.int64, device=dev)
        out["t2i_k"] = torch.full((eng.metric_texts, k), -7, dtype=torch.int64, device=dev)
        eng.request_topk(k, out["recall"], out["i2t_k"], out["t2i_k"])
    if o.losses:
        out["image_loss"] = torch.full((eng.images,), -1.0, device=dev)
        out["text_loss"] = torch.full((eng.texts,), -1.0, device=dev)
        eng.request_sample_losses(out["image_loss"], out["text_loss"])
    return out


def _untouched(bufs):
    return all(bool((v == SENTINEL[v.dtype]).all()) for v in bufs.values())


def _references(seq, st, P):
    o, r, g = st.opts, seq.r, st.grad_out
    res = om.oracle(P, o, st.tp, st.bias, st.lam)
    ret = om.retrieval(P, o, o.topk) if (o.keys or o.topk > 1 or seq.W > 1) else None
    stand = om.peer_stand_ins(P, o, r, res, ret, st.f16)
    x = res[r]
    ref = dict(loss=x["loss"], dimg=g * x["dimg"], contrib=[g * c for c in x["contrib"]], dt_prime=g * x["dt_prime"],
               dbias=g * x["dbias"], image_loss=x["image_loss"], text_loss=x["text_loss"])
    if seq.W > 1 and st.knob("SYNC_SCALAR_GRADS") and st.backward:
        # the mean over ranks of every rank's own dt' and dbias (the peers' stand in through their mailboxes)
        ref["mailbox"] = {p: (g * res[p]["dt_prime"], g * res[p]["dbias"]) for p in range(seq.W) if p != r}
        ref["dt_prime"] = g * np.mean([y["dt_prime"] for y in res])
        ref["dbias"] = g * np.mean([y["dbias"] for y in res])
    return ref, ret, stand


def _seed(eng, seq, st, i, P, ref, stand):
    """The peers of a W > 1 step: chunks and request stand-ins, contributions to this rank's dtxt, mailboxes."""
    if seq.W == 1:
        return None
    cell = seq.cell(st)
    _seed_peers(eng, cell, P, stand)
    for p, (a, b) in ref.get("mailbox", {}).items():
        eng.debug_set_mailbox(p, float(a), float(b))
    if not st.backward:
        return None
    C = lx.seeds(lx.XCell(cell), ref["contrib"][seq.r], i)
    for p, blk in C.items():
        eng.debug_set_peer_contribution(p, torch.from_numpy(np.ascontiguousarray(blk, np.float32)).to(_dev()))
    return sum(C.values())


def _run(eng, seq, st, P):
    """The step's calls; returns its outputs (peer slots as slot<k>) or raises what the library returned."""
    o, r = st.opts, seq.r
    _, _, _, imgs, txts = P.view(o)
    img, txt = _operand(imgs[r], st.f16), _operand(txts[r], st.f16)
    tp = torch.tensor([st.tp], device=_dev(), dtype=torch.float64 if st.tp64 else torch.float32)
    b, g = _scal(st.bias), _scal(st.grad_out)
    gdt = torch.bfloat16 if st.bf16 else torch.float32
    out = {}
    if st.refuse == "backward_unsaved":
        eng.backward(img, txt, tp, g, gdt)
    elif st.sched == "fused":
        out["loss"], out["dimg"], out["dtxt"], out["dtp"], out["db"] = eng.fwd_bwd(img, txt, tp, b, gdt)
    elif st.sched == "scaled":
        out["loss"], out["dimg"], out["dtxt"], out["dtp"], out["db"] = eng.fwd_bwd(img, txt, tp, b, gdt, g)
    elif st.sched == "fwd":
        out["loss"] = eng.fwd(img, txt, tp, b)
    else:
        out["loss"] = eng.forward(img, txt, tp, b, True)
        if st.sched == "eval":   # an evaluation forward of other data between the saving forward and its backward
            Q = om.planted(dataclasses.replace(seq.cell(st), seed=st.seed + 50))
            _, _, _, qi, qt = Q.view(o)
            out["eval_loss"] = eng.fwd(_operand(qi[r], st.f16), _operand(qt[r], st.f16), tp, b)
        out["dimg"], out["dtxt"], out["dtp"], out["db"] = eng.backward(img, txt, tp, g, gdt)
    if st.backward:
        for k in range(seq.W):
            if k != r:
                out[f"slot{k}"] = eng.debug_get_slot(k)
    torch.cuda.synchronize()
    return {k: v.clone() for k, v in out.items()}


def _prepare(eng, held, seq, st, i, P, ref, stand):
    """Options, inputs, peers and requests of the step: (request buffers, seeded dtxt sum, teacher tensors)."""
    want = seq.options(st)
    req = None
    if st.refuse in ("distill_losses", "distill_topk"):
        # the request is armed while DISTILL is off; turning it on then makes take_ids refuse the step
        _apply(eng, held, dict(want, DISTILL=0))
        req = _arm(eng, st.opts)
    _apply(eng, held, want)
    if held.get("SIGMA_BUDGET_MIB") and st.refuse is None and st.sched in ("fused", "scaled"):
        assert eng.sigma_panels()[1] > 1, f"{seq.name} step {i}: the budget does not split the rows"
    teacher = _inputs(eng, seq, st, P, st.refuse)
    total = _seed(eng, seq, st, i, P, ref, stand) if st.refuse is None else None
    if req is None:
        req = _arm(eng, st.opts)
    return req, total, teacher


def _compare(seq, st, i, out, req, ref, ret, total, P):
    o, r = st.opts, seq.r
    tag = f"{seq.name} step {i}"
    Bs, Rs, Ts, _, _ = P.view(o)
    gtol = BF16_TOL if st.bf16 else om.TOL
    bf = " (bf16)" if st.bf16 else ""
    _check(tag, "loss", out["loss"], ref["loss"], om.TOL)
    if st.backward:
        _check(tag, "dimg" + bf, out["dimg"], ref["dimg"], gtol)
        _check(tag, "dt_prime", out["dtp"], ref["dt_prime"], om.TOL)
        _check(tag, "dbias", out["db"], ref["dbias"], om.TOL)
        own = ref["contrib"][r]
        got = out["dtxt"].double().cpu().numpy()
        if total is None:
            _check(tag, "dtxt" + bf, got, own, gtol)
        else:   # the seeded contributions are exact in fp32; the output rounds |own| + |sum C|
            mag = np.abs(own) + np.abs(total)
            ratio = max(np.linalg.norm(mag) / np.linalg.norm(own), mag.max() / np.abs(own).max())
            u = 2.0 ** -8 if st.bf16 else 2.0 ** -23
            _check(tag, "dtxt - sum C" + bf, got - total, own, gtol + u * ratio)
        for k in range(seq.W):
            if k != r:
                _check(tag, "outgoing slots", out[f"slot{k}"], ref["contrib"][k], om.TOL)
    if o.losses:
        zi = P.iw[r][:Rs[r]] == 0 if o.weights else None
        zt = P.tw[r][:Ts[r]] == 0 if o.weights else None
        rows = sum((t + 127) // 128 + 1 for t in Ts)
        cols = (Rs[r] + 15) // 16 + 1 + seq.W - 1
        _check_sample_losses(f"{tag} image_loss", req["image_loss"], ref["image_loss"], zi, rows)
        _check_sample_losses(f"{tag} text_loss", req["text_loss"], ref["text_loss"], zt, cols)
    if o.metrics:
        y = ret[r]
        assert np.array_equal(req["top1"].cpu().numpy(), y["top1"]), f"{tag}: top-1 rates"
        assert np.array_equal(req["i2t"].cpu().numpy(), y["i2t_index"]), f"{tag}: i2t indices"
        assert np.array_equal(req["t2i"].cpu().numpy(), y["t2i_index"]), f"{tag}: t2i indices"
    if o.topk:
        y = ret[r]
        assert np.array_equal(req["i2t_k"].cpu().numpy(), y["i2t_topk"]), f"{tag}: i2t top-K lists"
        assert np.array_equal(req["t2i_k"].cpu().numpy(), y["t2i_topk"]), f"{tag}: t2i top-K lists"
        assert np.array_equal(req["recall"].cpu().numpy(), y["recall_f32"]), f"{tag}: recall"


def _fresh_launches(seq, st, i, P, ref, stand):
    """The launches of the same step on a fresh context, counted at its second step: the first step of a multi-rank
    context has no previous step whose flags it waits for."""
    eng = _engine(seq)
    try:
        held = {}
        for _ in range(2):
            n0 = eng.launch_count
            teacher = _prepare(eng, held, seq, st, i, P, ref, stand)  # noqa: F841
            _run(eng, seq, st, P)
        return eng.launch_count - n0
    finally:
        eng.close()


@pytest.mark.parametrize("seq", ss.SEQUENCES, ids=lambda s: s.name)
def test_step_sequence(seq):
    eng = _engine(seq)
    held, last, refused = {}, None, None
    try:
        for i, st in enumerate(seq.steps):
            tag = f"{seq.name} step {i}"
            P = om.planted(seq.cell(st))
            if st.refuse is not None:
                req, _, teacher = _prepare(eng, held, seq, st, i, P, None, None)
                with pytest.raises(RuntimeError):
                    _run(eng, seq, st, P)
                refused = req
                continue
            ref, ret, stand = _references(seq, st, P)
            n0 = eng.launch_count
            req, total, teacher = _prepare(eng, held, seq, st, i, P, ref, stand)
            out = _run(eng, seq, st, P)
            launches = eng.launch_count - n0
            _compare(seq, st, i, out, req, ref, ret, total, P)
            if st.sched == "eval":
                Q = om.planted(dataclasses.replace(seq.cell(st), seed=st.seed + 50))
                _check(tag, "evaluation loss", out["eval_loss"],
                       om.oracle(Q, st.opts, st.tp, st.bias, st.lam)[seq.r]["loss"], om.TOL)
            if refused is not None:
                assert _untouched(refused), f"{tag}: the refused step's request buffers were written"
                refused = None
            if not st.requests and last is not None:
                for k, (buf, vals) in last.items():
                    assert torch.equal(buf, vals), f"{tag}: the last request's {k} changed in an unarmed step"
            if st.requests:
                last = {k: (v, v.clone()) for k, v in req.items()}
            fresh = _fresh_launches(seq, st, i, P, ref, stand)
            assert launches == fresh, f"{tag}: {launches} launches, {fresh} on a fresh context"
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# a DDPSigmoidLoss trained over several steps: t' and bias by SGD from the kernel's own gradients, bf16 and fp32
# inputs alternating on one module (INPUT_F16 flips on one context), a no_grad fp32 evaluation forward between steps,
# metrics every other step, and the loss scaled by 2^k before backward (grad_out != 1)
# ---------------------------------------------------------------------------------------------------------------------
MODULE_STEPS = 8
LR = 0.05


@pytest.mark.parametrize("fused", [False, True], ids=["split", "fused"])
def test_module_sequence_matches_autograd_at_every_step(fused):
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss

    dev = _dev()
    B = om.SHAPES[1][0][0]
    mod = DDPSigmoidLoss(B, fused_step=fused).to(dev)
    with torch.no_grad():
        mod.t_prime.fill_(ss.HOT[0])
        mod.bias.fill_(ss.HOT[1])
    o = om.Options()

    def reference(xi, xt, P):
        ri = operand_values(xi).cpu().requires_grad_(True)
        rt = operand_values(xt).cpu().requires_grad_(True)
        tp64 = torch.tensor(float(mod.t_prime), dtype=torch.float64, requires_grad=True)
        b64 = torch.tensor(float(mod.bias), dtype=torch.float64, requires_grad=True)
        ref = torch_loss(ri, rt, tp64, b64, torch.from_numpy(om.labels(P, o)[0][0]), batch=B)
        return ref, ri, rt, tp64, b64

    for k in range(MODULE_STEPS):
        tag = f"{'fused' if fused else 'split'} module step {k}"
        dtype = torch.bfloat16 if k % 2 == 0 else torch.float32
        P = om.planted(om.Cell(o, 1, 0, False, "fused", False, False, 128, 6, 2, 1, 900 + k))
        xi = torch.from_numpy(P.imgs[0][:B]).to(dtype).to(dev).requires_grad_(True)
        xt = torch.from_numpy(P.txts[0][:B]).to(dtype).to(dev).requires_grad_(True)
        metrics = k % 2 == 1
        got = mod(xi, xt, return_metrics=metrics)
        loss, met = got if metrics else (got, None)
        ref, ri, rt, tp64, b64 = reference(xi, xt, P)
        scale = 2.0 ** (k % 4 - 1)
        mod.zero_grad()
        (loss * scale).backward()
        (ref * scale).backward()
        tol = 4e-3 if dtype == torch.bfloat16 else om.TOL   # bf16 gradients: 2^-9 rounding
        _check(tag, "module loss", loss.detach(), ref.detach(), tol)
        _check(tag, "module dimg", xi.grad, ri.grad, tol)
        _check(tag, "module dtxt", xt.grad, rt.grad, tol)
        _check(tag, "module dt'", mod.t_prime.grad, tp64.grad, tol)
        _check(tag, "module dbias", mod.bias.grad, b64.grad, tol)
        if metrics:
            y = om.retrieval(P, o, 1)[0]
            assert np.array_equal(torch.stack([met["i2t_top1"], met["t2i_top1"]]).cpu().numpy(), y["top1"]), tag
        with torch.no_grad():   # an fp32 evaluation forward of other data at the current parameters
            Q = om.planted(om.Cell(o, 1, 0, False, "fused", False, False, 128, 6, 2, 1, 950 + k))
            ei = torch.from_numpy(Q.imgs[0][:B]).float().to(dev)
            et = torch.from_numpy(Q.txts[0][:B]).float().to(dev)
            ev = mod(ei, et)
            _check(tag, "module evaluation loss", ev, reference(ei, et, Q)[0].detach(), om.TOL)
            mod.t_prime -= LR * mod.t_prime.grad
            mod.bias -= LR * mod.bias.grad


@pytest.mark.parametrize("call", ["fwd_bwd", "forward", "fwd"])
def test_an_engine_refusal_disarms_the_requests(call):
    """SigmoidLossEngine refusing a step's arguments before the library sees them consumes the armed requests, as a
    refusal of the library does: the buffers keep their sentinels through the next step, which launches what a plain
    step launches and matches the oracle."""
    seq = ss.make("engine-refusal", 1, 0, [dict()], seed=17)
    st = seq.steps[0]
    P = om.planted(seq.cell(st))
    ref, ret, stand = _references(seq, st, P)
    eng = _engine(seq)
    try:
        held = {}
        _apply(eng, held, seq.options(st))
        armed = _arm(eng, om.Options(metrics=True, losses=True, topk=3))
        _, _, _, imgs, txts = P.view(st.opts)
        img, txt = _operand(imgs[0], False), _operand(txts[0], False)
        tp, b = _scal(st.tp), _scal(st.bias)
        with pytest.raises(RuntimeError):   # a text operand one row short
            if call == "fwd_bwd":
                eng.fwd_bwd(img, txt[1:].contiguous(), tp, b)
            elif call == "forward":
                eng.forward(img, txt[1:].contiguous(), tp, b, True)
            else:
                eng.fwd(img, txt[1:].contiguous(), tp, b)
        n0 = eng.launch_count
        req, total, teacher = _prepare(eng, held, seq, st, 0, P, ref, stand)
        out = _run(eng, seq, st, P)
        launches = eng.launch_count - n0
        _compare(seq, st, 0, out, req, ref, ret, total, P)
        assert _untouched(armed), f"{call}: the refused step's request buffers were written"
        assert launches == _fresh_launches(seq, st, 0, P, ref, stand), f"{call}: a request stayed armed"
    finally:
        eng.close()
