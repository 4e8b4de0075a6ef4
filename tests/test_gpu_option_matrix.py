"""The loss step's options in combination on the H100: every cell of tests/option_matrix.py against the composed float64
oracle, with the other ranks of W = 2 and 3 standing in through the loopback hooks (their text chunks, ids, weights,
groups, teacher texts, argmax keys, top-K column lists, per-sample partials and extra-image ids).

Per cell: loss, dimg, the own-chunk dtxt and the peer slots, dt' and dbias within 1e-3 (the suite's norm-and-max
measure); per-sample losses within 1e-3 per sample; top-1 rates and indices, top-K lists and recall exactly (planted
data: every logit is exact); weight-0 samples exactly 0 in dimg, the own chunk's dtxt and the per-sample losses; and the
next step, without metrics, top-K or per-sample losses, gives loss and gradients bit for bit. The peers' stand-in keys
hold the accumulator the loss kernel keys on: 2^8 <img, txt> for fp16(16 x) operands. For the panel cells, the
metrics, top-K lists and per-sample losses are the same bits under every cluster shape and stage count, with and without
row panels. The modules run with every non-distillation option at once."""
import numpy as np
import pytest
import torch

import option_matrix as om
from exclude_groups_oracle import operand_values, torch_loss
from test_gpu_exclude_groups import _rel
from test_gpu_sample_losses import _check as _check_per_sample

pytestmark = pytest.mark.gpu

RESULTS = {}   # cell name -> its outputs (one run per cell, shared by the family checks)


def _dev():
    return torch.device("cuda", 0)


def _scal(x):
    return torch.tensor([x], device=_dev(), dtype=torch.float32)


def _check(name, got, ref, tol=om.TOL):
    err = _rel(got, ref)
    assert err <= tol, f"{name}: relative error {err:.3e}"


def _operand(x, f16):
    """Planted values as the kernels' operands: bf16, or fp16 holding 16 x (INPUT_F16); both exact."""
    t = torch.from_numpy(np.ascontiguousarray(x))
    return ((t * 16).half() if f16 else t.to(torch.bfloat16)).to(_dev())


def _i64(x):
    return torch.from_numpy(np.ascontiguousarray(x, np.int64)).to(_dev())


def _f32(x):
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(_dev())


def _engine(cell, stages=None, cg=None, mcast=None, panels=None):
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi

    o = cell.opts
    cg, mcast = cell.cg if cg is None else cg, cell.mcast if mcast is None else mcast
    Bs, Rs, Ts = cell.shapes()
    r, W = cell.r, cell.W
    kw = dict(cta_group=cg, rank_world=(r, W), loopback=W > 1, batch_per_rank=Bs)
    if o.teacher:
        kw["teacher_dim"] = om.DT
    if Rs != Bs:
        kw.update(images_per_rank=Rs, texts_per_rank=Ts)
    elif Ts != Bs:
        kw["texts_per_rank"] = Ts
    eng = SigmoidLossEngine(Bs[r], om.D, _dev(), **kw)
    for on, opt, val in ((mcast != 1, _capi.SIGLIP_OPT_MCAST, mcast),
                         (True, _capi.SIGLIP_OPT_STAGES_LOSS, cell.stages if stages is None else stages),
                         (True, _capi.SIGLIP_OPT_GRAD_TILE_N, cell.tile_n),
                         (cell.bidir, _capi.SIGLIP_OPT_BIDIR, 1),
                         (o.ids, _capi.SIGLIP_OPT_SAMPLE_IDS, 1),
                         (o.xt_ids, _capi.SIGLIP_OPT_EXTRA_TEXT_IDS, 1),
                         (o.xi_ids, _capi.SIGLIP_OPT_EXTRA_IMAGE_IDS, 1),
                         (o.weights, _capi.SIGLIP_OPT_SAMPLE_WEIGHTS, 1),
                         (o.groups, _capi.SIGLIP_OPT_EXCLUDE_GROUPS, 1),
                         (o.teacher, _capi.SIGLIP_OPT_DISTILL, 1)):
        if on:
            eng.set_option(opt, val)
    if cell.panels if panels is None else panels:
        eng.set_sigma_budget(cell.budget_mib(cg * mcast) << 20)
        assert eng.sigma_panels()[1] > 1, f"{cell.name}: the budget does not split the rows"
    return eng


def _inputs(eng, cell, P):
    """The step's own inputs (ids, weights, groups, teacher), given before every step."""
    o, r = cell.opts, cell.r
    Bs, Rs, Ts, _, _ = P.view(o)
    if o.ids:
        eng.set_sample_ids(_i64(P.ids[r]))
        if o.xt_ids:
            eng.set_extra_text_ids(_i64(P.xt_ids[r][:Ts[r] - Bs[r]]))
        if o.xi_ids:
            eng.set_extra_image_ids(_i64(P.xi_ids[r][:Rs[r] - Bs[r]]))
    if o.weights:
        eng.set_sample_weights(_f32(P.iw[r][:Rs[r]]), _f32(P.tw[r][:Ts[r]]))
    if o.groups:
        eng.set_groups(_i64(P.ig[r][:Rs[r]]), _i64(P.tg[r][:Ts[r]]))
    if o.teacher:   # the engine records the pointers: the caller keeps the tensors until the step is enqueued
        teacher = (_operand(P.timgs[r], cell.f16), _operand(P.ttxts[r], cell.f16), _scal(om.TTP), _scal(om.TBIAS))
        eng.set_teacher(*teacher, om.LAM)
        return teacher
    return None


def _seed_peers(eng, cell, P, stand_ins):
    """What the other ranks publish: their text chunks and per-chunk inputs, and for the step's requests their keys,
    lists, partials and extra-image ids."""
    o, r = cell.opts, cell.r
    Bs, Rs, Ts, _, txts = P.view(o)
    for k in range(cell.W):
        eng.debug_set_text_chunk(k, _operand(txts[k], cell.f16))
        if o.teacher:
            eng.debug_set_teacher_text_chunk(k, _operand(P.ttxts[k], cell.f16))
        if k == r:
            continue
        if o.ids:
            eng.debug_set_chunk_ids(k, _i64(np.concatenate([P.ids[k], P.xt_ids[k][:Ts[k] - Bs[k]]]) if o.xt_ids
                                            else P.ids[k]))
        if o.weights:
            eng.debug_set_chunk_weights(k, _f32(P.tw[k][:Ts[k]]))
        if o.groups:
            eng.debug_set_chunk_groups(k, _i64(P.tg[k][:Ts[k]]))
    for p, d in stand_ins.items():
        if o.keys:
            eng.debug_set_peer_metric_keys(p, _i64(d["metric_keys"]))
        if o.topk > 1:
            eng.debug_set_peer_topk_keys(p, _i64(d["topk_keys"]))
        if o.losses:
            eng.debug_set_peer_sample_loss_partials(p, _i64(d["partials"]))
        if o.xi_ids and (o.keys or o.topk > 1) and Rs[p] > Bs[p]:
            eng.debug_set_peer_extra_image_ids(p, _i64(d["xi_ids"]))


def _step(eng, cell, P, requests=True):
    """One step of the cell's schedule; returns its outputs by name (peer slots as slot<k>)."""
    o = cell.opts
    Bs, Rs, Ts, imgs, txts = P.view(o)
    r, dev = cell.r, _dev()
    teacher = _inputs(eng, cell, P)  # noqa: F841
    out = {}
    if requests and o.metrics:
        out["top1"] = torch.full((2,), -1.0, device=dev)
        out["i2t"] = torch.full((eng.metric_images,), -7, dtype=torch.int64, device=dev)
        out["t2i"] = torch.full((eng.metric_texts,), -7, dtype=torch.int64, device=dev)
        eng.request_metrics(out["top1"], out["i2t"], out["t2i"])
    if requests and o.topk:
        k = o.topk
        out["recall"] = torch.full((2 * k,), -1.0, device=dev)
        out["i2t_k"] = torch.full((eng.metric_images, k), -7, dtype=torch.int64, device=dev)
        out["t2i_k"] = torch.full((eng.metric_texts, k), -7, dtype=torch.int64, device=dev)
        eng.request_topk(k, out["recall"], out["i2t_k"], out["t2i_k"])
    if requests and o.losses:
        out["image_loss"] = torch.full((eng.images,), -1.0, device=dev)
        out["text_loss"] = torch.full((eng.texts,), -1.0, device=dev)
        eng.request_sample_losses(out["image_loss"], out["text_loss"])
    img, txt = _operand(imgs[r], cell.f16), _operand(txts[r], cell.f16)
    tp, b = _scal(om.TP), _scal(om.BIAS)
    if cell.sched == "fused":
        out["loss"], out["dimg"], out["dtxt"], out["dtp"], out["db"] = eng.fwd_bwd(img, txt, tp, b)
    elif cell.sched == "split":
        out["loss"] = eng.forward(img, txt, tp, b, True)
        out["dimg"], out["dtxt"], out["dtp"], out["db"] = eng.backward(img, txt, tp, None)
    else:
        out["loss"] = eng.fwd(img, txt, tp, b)
    if cell.sched != "fwd":
        for k in range(cell.W):
            if k != r:
                out[f"slot{k}"] = eng.debug_get_slot(k)
    torch.cuda.synchronize()
    return {k: v.clone() for k, v in out.items()}


def _references(cell, P):
    o = cell.opts
    res = om.oracle(P, o)
    ret = om.retrieval(P, o, o.topk) if (o.keys or o.topk > 1 or cell.W > 1) else None
    return res, ret, om.peer_stand_ins(P, o, cell.r, res, ret, cell.f16)


def _compare(cell, P, out, res, ret):
    o, r, tag = cell.opts, cell.r, cell.name
    Bs, Rs, Ts, _, _ = P.view(o)
    x = res[r]
    _check(f"{tag} loss", out["loss"], x["loss"])
    if cell.sched != "fwd":
        _check(f"{tag} dimg", out["dimg"], x["dimg"])
        _check(f"{tag} dt_prime", out["dtp"], x["dt_prime"])
        _check(f"{tag} dbias", out["db"], x["dbias"])
        for k in range(cell.W):
            _check(f"{tag} contribution to chunk {k}", out["dtxt"] if k == r else out[f"slot{k}"], x["contrib"][k])
        if o.weights:
            zi, zt = P.iw[r][:Rs[r]] == 0, P.tw[r][:Ts[r]] == 0
            assert zi.any() and zt.any()
            assert (out["dimg"].cpu()[torch.from_numpy(zi)] == 0).all(), f"{tag}: a weight-0 image has a gradient"
            assert (out["dtxt"].cpu()[torch.from_numpy(zt)] == 0).all(), f"{tag}: a weight-0 text has a gradient"
    if o.losses:
        zi = P.iw[r][:Rs[r]] == 0 if o.weights else None
        zt = P.tw[r][:Ts[r]] == 0 if o.weights else None
        _check_per_sample(f"{tag} image_loss", out["image_loss"], x["image_loss"], zi)
        _check_per_sample(f"{tag} text_loss", out["text_loss"], x["text_loss"], zt)
    if o.metrics:
        y = ret[r]
        assert np.array_equal(out["top1"].cpu().numpy(), y["top1"]), f"{tag}: top-1 rates {out['top1']} vs {y['top1']}"
        assert np.array_equal(out["i2t"].cpu().numpy(), y["i2t_index"]), f"{tag}: i2t indices"
        assert np.array_equal(out["t2i"].cpu().numpy(), y["t2i_index"]), f"{tag}: t2i indices"
    if o.topk:
        y = ret[r]
        assert np.array_equal(out["i2t_k"].cpu().numpy(), y["i2t_topk"]), f"{tag}: i2t top-K lists"
        assert np.array_equal(out["t2i_k"].cpu().numpy(), y["t2i_topk"]), f"{tag}: t2i top-K lists"
        assert np.array_equal(out["recall"].cpu().numpy(), y["recall_f32"]), f"{tag}: recall"


DETACHED = ("top1", "i2t", "t2i", "recall", "i2t_k", "t2i_k", "image_loss", "text_loss")


def _run(cell, **variant):
    """Runs the cell (once per variant) and returns its outputs; the plain run is checked against the oracle and against
    a second step without requests (the same bits: the requests change no loss or gradient bit, and no step carries
    state into the next)."""
    key = (cell.name, tuple(sorted(variant.items())))
    if key in RESULTS:
        return RESULTS[key]
    P = om.planted(cell)
    res, ret, stand = _references(cell, P)
    eng = _engine(cell, **variant)
    try:
        if cell.W > 1:
            _seed_peers(eng, cell, P, stand)
        out = _step(eng, cell, P)
        if not variant:
            _compare(cell, P, out, res, ret)
            plain = _step(eng, cell, P, requests=False)
            for k, v in plain.items():
                assert torch.equal(v, out[k]), f"{cell.name}: {k} differs in a second step without requests"
    finally:
        eng.close()
    RESULTS[key] = {k: v for k, v in out.items() if k in DETACHED}
    return RESULTS[key]


@pytest.mark.parametrize("cell", om.TABLE, ids=lambda c: c.name)
def test_cell_matches_the_composed_oracle(cell):
    _run(cell)


PANEL_CELLS = [c for c in om.TABLE if c.panels and (c.opts.keys or c.opts.topk or c.opts.losses)]
VARIANTS = [dict(stages=st, cg=cg, mcast=mc) for st in (4, 6) for cg, mc in ((1, 1), (2, 1), (1, 2), (2, 2))]


@pytest.mark.parametrize("cell", PANEL_CELLS, ids=lambda c: c.name)
def test_detached_outputs_are_the_same_bits_across_configurations(cell):
    """Metrics, top-K lists and per-sample losses of a cell: the same bits under every stage count and cluster shape,
    in row panels and without them."""
    first = _run(cell)
    for v in VARIANTS + [dict(panels=False)]:
        got = _run(cell, **v)
        for k in first:
            assert torch.equal(got[k], first[k]), f"{cell.name} {v}: {k} differs"


# ---------------------------------------------------------------------------------------------------------------------
# the modules with every non-distillation option at once
# ---------------------------------------------------------------------------------------------------------------------
MODULE_CELL = om.Cell(om.Options(ids=True, xtexts=True, ximages=True, xt_ids=True, xi_ids=True, weights=True,
                                 groups=True, metrics=True, losses=True, topk=5),
                      1, 0, False, "fused", True, False, 128, 6, 2, 1, 200)


@pytest.mark.parametrize("kind", ["ddp", "siglip"])
@pytest.mark.parametrize("dtype,normalize", [(torch.bfloat16, False), (torch.float32, False), (torch.float32, True)])
def test_modules_with_every_option(kind, dtype, normalize):
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    cell = MODULE_CELL
    o = cell.opts
    P = om.planted(cell)
    Bs, Rs, Ts, imgs, txts = P.view(o)
    B, K, E, k = Bs[0], Ts[0] - Bs[0], Rs[0] - Bs[0], o.topk
    dev = _dev()
    scale = 3.0 if normalize else 1.0
    xi = (torch.from_numpy(imgs[0]) * scale).to(dtype).to(dev).requires_grad_(True)
    xt = (torch.from_numpy(txts[0]) * scale).to(dtype).to(dev).requires_grad_(True)
    kw = dict(multi_positive=True, extra_texts=K, extra_images=E, sample_weights=True, exclude_groups=True,
              sigma_budget_bytes=cell.budget_mib() << 20)
    args = dict(sample_ids=_i64(P.ids[0]), extra_text=xt[B:], extra_text_ids=_i64(P.xt_ids[0]), extra_image=xi[B:],
                extra_image_ids=_i64(P.xi_ids[0]), image_weights=_f32(P.iw[0]), text_weights=_f32(P.tw[0]),
                image_groups=_i64(P.ig[0]), text_groups=_i64(P.tg[0]), return_metrics=True, metrics_topk=k,
                return_sample_losses=True)
    if kind == "ddp":
        mod = DDPSigmoidLoss(B, normalize_inputs=normalize, **kw).to(dev)
        with torch.no_grad():
            mod.t_prime.fill_(om.TP)
            mod.bias.fill_(om.BIAS)
        eng = mod.engine_for(B, om.D, dev)
        loss, met, sl = mod(xi[:B], xt[:B], **args)
        params = (mod.t_prime, mod.bias)
    else:
        if normalize:
            pytest.skip("SigLipLoss takes normalised features")
        mod = SigLipLoss(**kw)
        tp = torch.tensor(om.TP, device=dev, requires_grad=True)
        bb = torch.tensor(om.BIAS, device=dev, requires_grad=True)
        loss, met, sl = mod(xi[:B], xt[:B], tp, bb, **args)
        eng = mod._cache.get(B, om.D, dev, 0)
        params = (tp, bb)
    assert eng.sigma_panels()[1] > 1
    loss.backward()
    # float64 autograd of torch_loss on the values the kernels consume, with the oracle's labels
    y = torch.from_numpy(om.labels(P, o)[0][0])
    ri = operand_values(xi).cpu().requires_grad_(True)
    rt = operand_values(xt).cpu().requires_grad_(True)
    tp64 = torch.tensor(om.TP, dtype=torch.float64, requires_grad=True)
    b64 = torch.tensor(om.BIAS, dtype=torch.float64, requires_grad=True)
    ref = torch_loss(ri, rt, tp64, b64, y, torch.from_numpy(P.iw[0]).double(), torch.from_numpy(P.tw[0]).double(),
                     normalize=normalize, batch=B)
    ref.backward()
    tol = 4e-3 if dtype == torch.bfloat16 else om.TOL   # bf16 gradients: 2^-9 rounding
    tag = f"{kind} {dtype} normalize={normalize}"
    _check(f"{tag} loss", loss.detach(), ref.detach(), tol)
    _check(f"{tag} dimg", xi.grad, ri.grad, tol)
    _check(f"{tag} dtxt", xt.grad, rt.grad, tol)
    _check(f"{tag} dt'", params[0].grad, tp64.grad, tol)
    _check(f"{tag} dbias", params[1].grad, b64.grad, tol)
    assert float(sl["image_loss"].double().sum()) == pytest.approx(loss.item() * B, rel=1e-4)
    assert (sl["image_loss"].cpu()[torch.from_numpy(P.iw[0] == 0)] == 0).all()
    if not normalize:   # exact operands: retrieval against the oracle
        ret = om.retrieval(P, o, k)[0]
        assert np.array_equal(met["i2t_topk"].cpu().numpy(), ret["i2t_topk"])
        assert np.array_equal(met["t2i_topk"].cpu().numpy(), ret["t2i_topk"])
        assert np.array_equal(torch.cat([met["i2t_recall"], met["t2i_recall"]]).cpu().numpy(), ret["recall_f32"])
        assert np.array_equal(torch.stack([met["i2t_top1"], met["t2i_top1"]]).cpu().numpy(), ret["top1"])
        res = om.oracle(P, o)[0]
        _check_per_sample(f"{tag} image_loss", sl["image_loss"], res["image_loss"], P.iw[0] == 0)
        _check_per_sample(f"{tag} text_loss", sl["text_loss"], res["text_loss"], P.tw[0] == 0)
