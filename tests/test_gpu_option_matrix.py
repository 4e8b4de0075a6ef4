"""The loss step's options in combination on the H100: every cell of tests/option_matrix.py against the composed float64
oracle, with the other ranks of W = 2 and 3 standing in through the loopback hooks (their text chunks, ids, label sets,
weights, groups, teacher texts, argmax keys, top-K column lists, per-sample partials and extra-image ids and sets).

Per cell: loss, dimg, the own-chunk dtxt and the peer slots, dt' and dbias within 1e-3 (the suite's norm-and-max
measure); per-sample losses within 1e-3 per sample plus the 2^-32 resolution of each fixed-point word they are summed
from; top-1 rates and indices, top-K lists and recall exactly (planted
data: every logit is exact); weight-0 samples exactly 0 in dimg, the own chunk's dtxt and the per-sample losses; and the
next step, without metrics, top-K or per-sample losses, gives loss and gradients bit for bit. The peers' stand-in keys
hold the accumulator the loss kernel keys on: 2^8 <img, txt> for fp16(16 x) operands. For the panel cells, the
metrics, top-K lists and per-sample losses are the same bits under every cluster shape and stage count, with and without
row panels (a teacher cell: under each cluster shape, its kernels running 4 stages whatever the request). The modules run
with every non-distillation option at once, with the focal terms and every other non-teacher option, and with a teacher
and every option but the focal terms, against float64 autograd.

Observed on one H100 80GB HBM3 (700 W power limit): 424 tests (333 cells, their panel families and 14 module cases) in
about 7 to 8.5 min of wall time; the largest relative errors, all within the 1e-3 tolerance: loss 6.3e-5, the cells' dimg
and dtxt (own chunk and peer slots) 4.5e-4, dt' 9.5e-5, dbias 2.8e-4, per-sample losses of 1e-6 and above 3.3e-4;
the modules' bf16 gradients 2.7e-3 (their tolerance: 4e-3). With the 328 cold cells (om.COLD, whose launches run the
series path), on the same card at 700 W: 753 tests in 8 min 21 s of wall time; the cold cells' largest relative errors:
loss 3.2e-7, dimg 4.2e-4, dtxt (own chunk and peer slots) 3.5e-4, dt' 5.9e-5, dbias 5.7e-5, per-sample losses of 1e-6
and above 3.0e-5."""
import dataclasses

import numpy as np
import pytest
import torch

import option_matrix as om
from exclude_groups_oracle import operand_values, torch_loss
from focal_oracle import torch_focal_loss
from test_gpu_exclude_groups import _rel

WORD = 2.0 ** -32   # the resolution of a per-sample-loss partial: a fixed-point word holds value * 2^32

pytestmark = pytest.mark.gpu

RESULTS = {}   # cell name -> its outputs (one run per cell, shared by the family checks)
OBSERVED = {}  # output kind -> the largest relative error seen (pytest -s prints them)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(OBSERVED):
        print(f"option matrix: largest relative error of {k}: {OBSERVED[k]:.3e}")


def _note(kind, err, tag=""):
    cold = tag.endswith("-cold") or "-cold " in tag or "-cold-" in tag
    multi = tag.endswith("-multi") or "-multi " in tag
    kind = ("multi-tile " if multi and cold else "") + ("cold cells: " if cold else "multi-tile cells: " if multi
                                                          else "") + kind
    OBSERVED[kind] = max(OBSERVED.get(kind, 0.0), err)


def _dev():
    return torch.device("cuda", 0)


def _scal(x):
    return torch.tensor([x], device=_dev(), dtype=torch.float32)


def _check(name, got, ref, tol=om.TOL):
    err = _rel(got, ref)
    _note("dtxt (own chunk and peer slots)" if "chunk" in name else name.rsplit(" ", 1)[1], err, name)
    assert err <= tol, f"{name}: relative error {err:.3e}"


def _check_sample_losses(tag, got, want, zero, words):
    """Per-sample losses within 1e-3 relative, plus one fixed-point step per partial word a sample's loss is summed
    from (words): the focal terms at gamma = 5 leave a well-classified sample a loss of 1e-10 .. 1e-7, where the
    words' absolute resolution, not the kernel's arithmetic, bounds the relative error. Weight-0 samples exactly 0."""
    g = got.double().cpu().numpy()
    w = np.asarray(want, np.float64)
    assert np.isfinite(g).all(), f"{tag}: non-finite values"
    if zero is not None:
        assert zero.any() and (g[zero] == 0).all(), f"{tag}: a weight-0 sample is not exactly 0"
    big = w >= 1e-6
    if big.any():
        _note(f"{tag.rsplit(' ', 1)[1]} (samples >= 1e-6)", float(np.max(np.abs(g - w)[big] / w[big])), tag)
    excess = np.abs(g - w) - (om.TOL * w + words * WORD)
    assert excess.max() <= 0, f"{tag}: sample {int(excess.argmax())} {g[excess.argmax()]:.6e} vs {w[excess.argmax()]:.6e}"


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
    kw = dict(cta_group=cg, rank_world=(r, W), loopback=W > 1, batch_per_rank=Bs, labels=o.labels)
    if o.teacher:   # a teacher with extras or with kModeDistillOpts's options: a distill-extras context
        kw.update(teacher_dim=om.DT, distill_options=om.distill_extras_context(cell))
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
                         (o.labels > 0, _capi.SIGLIP_OPT_LABEL_SETS, 1),
                         (o.focal is not None, _capi.SIGLIP_OPT_FOCAL, 1),
                         (o.weights, _capi.SIGLIP_OPT_SAMPLE_WEIGHTS, 1),
                         (o.groups, _capi.SIGLIP_OPT_EXCLUDE_GROUPS, 1),
                         (o.teacher, _capi.SIGLIP_OPT_DISTILL, 1)):
        if on:
            eng.set_option(opt, val)
    if o.focal is not None:
        eng.set_focal(*o.focal)
    if cell.panels if panels is None else panels:
        eng.set_sigma_budget(cell.budget_mib(cg * mcast) << 20)
        assert eng.sigma_panels()[1] > 1, f"{cell.name}: the budget does not split the rows"
    return eng


def _inputs(eng, cell, P):
    """The step's own inputs (ids, label sets, weights, groups, teacher), given before every step."""
    o, r = cell.opts, cell.r
    Bs, Rs, Ts, _, _ = P.view(o)
    if o.labels:   # extras without sets of their own: None, the empty sets
        isets, tsets = P.sets(o)
        eng.set_label_sets(_i64(isets[r][:Bs[r]]), _i64(tsets[r][Bs[r]:]) if o.xt_sets else None,
                           _i64(isets[r][Bs[r]:]) if o.xi_sets else None)
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
        timgs, ttxts = P.teacher(o)
        teacher = (_operand(timgs[r], cell.f16), _operand(ttxts[r], cell.f16), _scal(om.TTP), _scal(om.TBIAS))
        eng.set_teacher(*teacher, om.LAM)
        return teacher
    return None


def _seed_peers(eng, cell, P, stand_ins):
    """What the other ranks publish: their text chunks and per-chunk inputs, and for the step's requests their keys,
    lists, partials and extra-image ids or sets."""
    o, r = cell.opts, cell.r
    Bs, Rs, Ts, _, txts = P.view(o)
    ttxts = P.teacher(o)[1]
    for k in range(cell.W):
        eng.debug_set_text_chunk(k, _operand(txts[k], cell.f16))
        if o.teacher:
            eng.debug_set_teacher_text_chunk(k, _operand(ttxts[k], cell.f16))
        if k == r:
            continue
        if o.labels:
            eng.debug_set_chunk_label_sets(k, _i64(stand_ins[k]["tsets"]))
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
        if o.labels and (o.keys or o.topk > 1) and Rs[p] > Bs[p]:
            eng.debug_set_peer_extra_image_label_sets(p, _i64(d["xi_sets"]))


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
        # words: a row's partials of 128 columns per chunk and a column's of 16 rows (a row panel's window adds one per
        # chunk), and one word from each peer
        rows = sum((t + 127) // 128 + 1 for t in Ts)
        cols = (Rs[r] + 15) // 16 + 1 + cell.W - 1
        _check_sample_losses(f"{tag} image_loss", out["image_loss"], x["image_loss"], zi, rows)
        _check_sample_losses(f"{tag} text_loss", out["text_loss"], x["text_loss"], zt, cols)
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


def test_coverage_holds_with_the_device_cluster_counts():
    """The multi-tile families' coverage (test_option_matrix_cpu._multi_missing) derived again from this device's
    co-resident clusters of every loss-kernel instantiation: if a count differs from an H100 SXM's and a cluster no
    longer runs several tiles somewhere, this fails and names what is missing."""
    from distributed_sigmoid_loss_b200 import _capi
    from test_option_matrix_cpu import _multi_missing

    props = torch.cuda.get_device_properties(0)
    counts = {}
    for mode in om.MODES:
        for st in sorted({i[1] for i in om.instantiations(mode)}):
            for cs, shapes in om.CLUSTERS.items():
                got = {_capi.loss_max_active_clusters(mode, cg, mc, st) for cg, mc in shapes}
                assert len(got) == 1, f"{mode} {st} stages: cluster shapes of {cs} CTAs differ: {got}"
                counts[(mode, st, cs)] = got.pop()
                assert 1 <= counts[(mode, st, cs)] <= props.multi_processor_count // cs
    print(f"\n{props.name}, {props.multi_processor_count} SMs: co-resident clusters of the loss kernel "
          "(mode, stages, cluster size)")
    for k in sorted(counts):
        print(f"  {k}: {counts[k]}")
    with pytest.raises(_capi.SiglipError):   # mode 1 is the gradient kernel
        _capi.check(-_capi.lib().siglip_debug_loss_max_active_clusters(0, 1, 1, 1, 6))
    for name in ("MULTI", "MULTI_COLD"):
        missing = _multi_missing(getattr(om, name), counts, props.multi_processor_count)
        assert not missing, f"{name} with this device's cluster counts: " + "; ".join(missing)


@pytest.mark.parametrize("cell", om.TABLE + om.COLD + om.MULTI + om.MULTI_COLD, ids=lambda c: c.name)
def test_cell_matches_the_composed_oracle(cell):
    _run(cell)


PANEL_CELLS = [c for c in om.TABLE if c.panels and (c.opts.keys or c.opts.topk or c.opts.losses)]
SHAPES = ((1, 1), (2, 1), (1, 2), (2, 2))
VARIANTS = [dict(stages=st, cg=cg, mcast=mc) for st in (4, 6) for cg, mc in SHAPES]


@pytest.mark.parametrize("cell", PANEL_CELLS, ids=lambda c: c.name)
def test_detached_outputs_are_the_same_bits_across_configurations(cell):
    """Metrics, top-K lists and per-sample losses of a cell: the same bits under every stage count and cluster shape,
    in row panels and without them (a teacher's kernels run 4 stages whatever the request: its cluster shapes only)."""
    first = _run(cell)
    variants = [v for v in VARIANTS if not cell.opts.teacher or v["stages"] == om.DISTILL_STAGES]
    for v in variants + [dict(panels=False)]:
        got = _run(cell, **v)
        for k in first:
            assert torch.equal(got[k], first[k]), f"{cell.name} {v}: {k} differs"


# ---------------------------------------------------------------------------------------------------------------------
# the modules with every non-distillation option at once, with the focal terms and every other non-teacher option (label
# sets instead of ids), and with a teacher and every option but the focal terms
# ---------------------------------------------------------------------------------------------------------------------
MODULE_CELL = om.Cell(om.Options(ids=True, xtexts=True, ximages=True, xt_ids=True, xi_ids=True, weights=True,
                                 groups=True, metrics=True, losses=True, topk=5),
                      1, 0, False, "fused", True, False, 128, 6, 2, 1, 200)
FOCAL_MODULE_CELL = om.Cell(om.Options(xtexts=True, ximages=True, labels=3, xt_sets=True, xi_sets=True, weights=True,
                                       groups=True, focal=(2.0, 0.25), metrics=True, losses=True, topk=5),
                            1, 0, False, "fused", True, False, 128, 6, 2, 1, 201)
TEACHER_MODULE_CELL = om.Cell(dataclasses.replace(MODULE_CELL.opts, teacher=True),
                              1, 0, False, "fused", True, False, 128, 6, 2, 1, 202)


def _module_case(cell, kind, dtype, normalize):
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    o = cell.opts
    P = om.planted(cell)
    Bs, Rs, Ts, imgs, txts = P.view(o)
    B, K, E, k = Bs[0], Ts[0] - Bs[0], Rs[0] - Bs[0], o.topk
    dev = _dev()
    scale = 3.0 if normalize else 1.0
    xi = (torch.from_numpy(imgs[0]) * scale).to(dtype).to(dev).requires_grad_(True)
    xt = (torch.from_numpy(txts[0]) * scale).to(dtype).to(dev).requires_grad_(True)
    kw = dict(extra_texts=K, extra_images=E, sample_weights=True, exclude_groups=True,
              sigma_budget_bytes=cell.budget_mib() << 20)
    args = dict(extra_text=xt[B:], extra_image=xi[B:], image_weights=_f32(P.iw[0]), text_weights=_f32(P.tw[0]),
                image_groups=_i64(P.ig[0]), text_groups=_i64(P.tg[0]), return_metrics=True, metrics_topk=k,
                return_sample_losses=True)
    if o.labels:
        isets, tsets = P.sets(o)
        kw["multi_label"] = o.labels
        args.update(sample_labels=_i64(isets[0][:B]), extra_text_labels=_i64(tsets[0][B:]),
                    extra_image_labels=_i64(isets[0][B:]))
    else:
        kw["multi_positive"] = True
        args.update(sample_ids=_i64(P.ids[0]), extra_text_ids=_i64(P.xt_ids[0]), extra_image_ids=_i64(P.xi_ids[0]))
    if o.focal is not None:
        kw.update(focal_gamma=o.focal[0], focal_alpha=o.focal[1])
    teacher = None
    if o.teacher:
        kw.update(distill=om.LAM, distill_options=True)
        timgs, ttxts = P.teacher(o)
        timg, ttxt = (torch.from_numpy(x[0]).to(dtype).to(dev) for x in (timgs, ttxts))
        args.update(teacher_image=timg[:B], teacher_text=ttxt[:B], teacher_extra_text=ttxt[B:],
                    teacher_extra_image=timg[B:])
        tscal = (torch.tensor(om.TTP, device=dev), torch.tensor(om.TBIAS, device=dev))
        teacher = (operand_values(timg).cpu(), operand_values(ttxt).cpu(), om.TTP, om.TBIAS, om.LAM)
    if kind == "ddp":
        if o.teacher:
            args.update(teacher_t_prime=tscal[0], teacher_bias=tscal[1])
        mod = DDPSigmoidLoss(B, normalize_inputs=normalize, **kw).to(dev)
        with torch.no_grad():
            mod.t_prime.fill_(om.TP)
            mod.bias.fill_(om.BIAS)
        eng = mod.engine_for(B, om.D, dev, om.DT if o.teacher else 0)
        loss, met, sl = mod(xi[:B], xt[:B], **args)
        params = (mod.t_prime, mod.bias)
    else:
        if normalize:
            pytest.skip("SigLipLoss takes normalised features")
        if o.teacher:
            args.update(teacher_logit_scale=tscal[0], teacher_logit_bias=tscal[1])
        mod = SigLipLoss(**kw)
        tp = torch.tensor(om.TP, device=dev, requires_grad=True)
        bb = torch.tensor(om.BIAS, device=dev, requires_grad=True)
        loss, met, sl = mod(xi[:B], xt[:B], tp, bb, **args)
        eng = mod._cache.get(B, om.D, dev, om.DT if o.teacher else 0)
        params = (tp, bb)
    assert eng.sigma_panels()[1] > 1
    loss.backward()
    # float64 autograd of the restatement on the values the kernels consume, with the oracle's labels
    y = torch.from_numpy(om.labels(P, o)[0][0])
    ri = operand_values(xi).cpu().requires_grad_(True)
    rt = operand_values(xt).cpu().requires_grad_(True)
    tp64 = torch.tensor(om.TP, dtype=torch.float64, requires_grad=True)
    b64 = torch.tensor(om.BIAS, dtype=torch.float64, requires_grad=True)
    iw, tw = torch.from_numpy(P.iw[0]).double(), torch.from_numpy(P.tw[0]).double()
    if o.focal is not None:
        ref = torch_focal_loss(ri, rt, tp64, b64, y, o.focal[0], o.focal[1], iw, tw, normalize=normalize, batch=B)
    else:
        ref = torch_loss(ri, rt, tp64, b64, y, iw, tw, normalize=normalize, batch=B, teacher=teacher)
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
        _check_sample_losses(f"{tag} image_loss", sl["image_loss"], res["image_loss"], P.iw[0] == 0,
                             (Ts[0] + 127) // 128 + 1)
        _check_sample_losses(f"{tag} text_loss", sl["text_loss"], res["text_loss"], P.tw[0] == 0,
                             (Rs[0] + 15) // 16 + 1)


MODULE_CASES = [("ddp", torch.bfloat16, False), ("ddp", torch.float32, False), ("ddp", torch.float32, True),
                ("siglip", torch.bfloat16, False), ("siglip", torch.float32, False)]


@pytest.mark.parametrize("kind", ["ddp", "siglip"])
@pytest.mark.parametrize("dtype,normalize", [(torch.bfloat16, False), (torch.float32, False), (torch.float32, True)])
def test_modules_with_every_option(kind, dtype, normalize):
    _module_case(MODULE_CELL, kind, dtype, normalize)


@pytest.mark.parametrize("kind,dtype,normalize", MODULE_CASES)
def test_modules_with_focal_and_every_other_option(kind, dtype, normalize):
    """focal_gamma / focal_alpha with label sets (extras with sets of their own), weights, groups, top-K and per-sample
    losses in row panels, against float64 autograd of focal_oracle.torch_focal_loss."""
    _module_case(FOCAL_MODULE_CELL, kind, dtype, normalize)


@pytest.mark.parametrize("kind,dtype,normalize", MODULE_CASES)
def test_modules_with_a_teacher_and_every_option_but_focal(kind, dtype, normalize):
    """distill=lambda, distill_options=True with ids, extras with ids and their teacher rows, weights, groups, top-K and
    per-sample losses in row panels, against float64 autograd of exclude_groups_oracle.torch_loss with the teacher."""
    _module_case(TEACHER_MODULE_CELL, kind, dtype, normalize)
