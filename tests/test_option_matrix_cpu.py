"""The option matrix (tests/option_matrix.py) on the CPU: the composed oracle against float64 autograd with every
non-distillation option on, with the focal terms and every other non-teacher option, and with a teacher and every option
but the focal terms; its reduction to the single-feature oracles; every cell's sensitivity to each option it turns on;
the table's coverage of the loss kernel's instantiations and runtime branches; the table's modes against the loss modes
launch_gemm dispatches to; and the exactness of the planted logits."""
import dataclasses
import math
import pathlib
import re

import numpy as np
import pytest
import torch

import option_matrix as om
from distill_oracle import closed_form_distill
from distill_options_oracle import closed_form_distill_options
from exclude_groups_oracle import closed_form_groups, group_labels, torch_loss, torch_terms
from extra_images_oracle import closed_form_extras, label_blocks, retrieval_metrics_extras
from focal_oracle import closed_form_focal, torch_focal_terms
from label_sets_oracle import closed_form_sets
from retrieval_metrics_oracle import retrieval_metrics
from sample_losses_oracle import sample_losses
from sample_weights_oracle import closed_form_weighted

ALL = om.Options(ids=True, xtexts=True, ximages=True, xt_ids=True, xi_ids=True, weights=True, groups=True,
                 metrics=True, losses=True, topk=5)


def _cell(W, panels=False, seed=0):
    return om.Cell(ALL, W, W - 1, False, "fused", panels, False, 128, 6, 2, 1, seed)


# ---------------------------------------------------------------------------------------------------------------------
# the oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W", [1, 2, 3])
def test_every_option_at_once_matches_autograd(W):
    """Per rank: float64 autograd of torch_loss over the whole text set gives loss, dimg, dt', dbias and the pair terms'
    row / column sums; the sum of every rank's loss gives each chunk's text gradient (dtxt_c = sum_r contrib_c)."""
    cell = _cell(W, seed=W)
    P = om.planted(cell)
    res = om.oracle(P, ALL)
    Bs, Rs, Ts, imgs, txts = P.view(ALL)
    lab = om.labels(P, ALL)
    assert any((y == 0).any() for row in lab for y in row) and any((y > 0).any() for row in lab for y in row)
    tchunks = [torch.tensor(x, dtype=torch.float64, requires_grad=True) for x in txts]
    tw = torch.from_numpy(np.concatenate(P.tw).astype(np.float64))
    total = 0.0
    for r in range(W):
        img = torch.tensor(imgs[r], dtype=torch.float64, requires_grad=True)
        tp = torch.tensor(om.TP, dtype=torch.float64, requires_grad=True)
        b = torch.tensor(om.BIAS, dtype=torch.float64, requires_grad=True)
        y = torch.from_numpy(np.concatenate(lab[r], axis=1))
        iw = torch.from_numpy(P.iw[r].astype(np.float64))
        txt = torch.cat(tchunks)
        loss = torch_loss(img, txt, tp, b, y, iw, tw, batch=Bs[r])
        gi, gt, gb = torch.autograd.grad(loss, [img, tp, b], retain_graph=True)
        x = res[r]
        assert om.rel(x["loss"], loss.item()) < 1e-12
        assert om.rel(x["dimg"], gi.numpy()) < 1e-12
        assert om.rel(x["dt_prime"], float(gt)) < 1e-12 and om.rel(x["dbias"], float(gb)) < 1e-12
        terms = torch_terms(img, txt, tp, b, y, iw, tw).detach().numpy()
        assert om.rel(x["image_loss"], terms.sum(axis=1)) < 1e-12
        lo = np.cumsum([0] + list(Ts))
        for c in range(W):
            assert om.rel(x["text_part"][c], terms[:, lo[c]:lo[c + 1]].sum(axis=0)) < 1e-12
        total = total + loss
    grads = torch.autograd.grad(total, tchunks)
    for c in range(W):
        assert om.rel(sum(x["contrib"][c] for x in res), grads[c].numpy()) < 1e-12
        assert om.rel(res[c]["text_loss"], sum(x["text_part"][c] for x in res)) == 0


FOCAL_ALL = om.Options(xtexts=True, ximages=True, labels=3, xt_sets=True, xi_sets=True, weights=True, groups=True,
                       focal=(2.0, 0.25), metrics=True, losses=True, topk=5)


def _terms_against_autograd(o, W, seed, terms_of):
    """The composed oracle of every rank against float64 autograd of terms_of(r, img, txt, t', bias, y) ([R_r, sum T]
    pair terms, the loss their sum / B_r): loss, dimg, dt', dbias, the per-sample row / column sums and, summed over the
    ranks, every chunk's text gradient."""
    cell = om.Cell(o, W, W - 1, False, "fused", False, False, 128, 6, 2, 1, seed)
    P = om.planted(cell)
    res = om.oracle(P, o)
    Bs, Rs, Ts, imgs, txts = P.view(o)
    lab = om.labels(P, o)
    assert any((y == 0).any() for row in lab for y in row) and any((y > 0).any() for row in lab for y in row)
    tchunks = [torch.tensor(x, dtype=torch.float64, requires_grad=True) for x in txts]
    total = 0.0
    lo = np.cumsum([0] + list(Ts))
    for r in range(W):
        img = torch.tensor(imgs[r], dtype=torch.float64, requires_grad=True)
        tp = torch.tensor(om.TP, dtype=torch.float64, requires_grad=True)
        b = torch.tensor(om.BIAS, dtype=torch.float64, requires_grad=True)
        y = torch.from_numpy(np.concatenate(lab[r], axis=1))
        terms = terms_of(r, img, torch.cat(tchunks), tp, b, y)
        loss = terms.sum() / Bs[r]
        gi, gt, gb = torch.autograd.grad(loss, [img, tp, b], retain_graph=True)
        x = res[r]
        assert om.rel(x["loss"], loss.item()) < 1e-12
        assert om.rel(x["dimg"], gi.numpy()) < 1e-12
        assert om.rel(x["dt_prime"], float(gt)) < 1e-12 and om.rel(x["dbias"], float(gb)) < 1e-12
        t = terms.detach().numpy()
        assert om.rel(x["image_loss"], t.sum(axis=1)) < 1e-12
        for c in range(W):
            assert om.rel(x["text_part"][c], t[:, lo[c]:lo[c + 1]].sum(axis=0)) < 1e-12
        total = total + loss
    grads = torch.autograd.grad(total, tchunks)
    for c in range(W):
        assert om.rel(sum(x["contrib"][c] for x in res), grads[c].numpy()) < 1e-12
    return P


@pytest.mark.parametrize("W", [1, 2, 3])
def test_focal_with_every_other_option_matches_autograd(W):
    """Label sets (extras with sets of their own), weights, groups and the focal terms at once, against float64
    autograd of focal_oracle.torch_focal_terms."""
    o = FOCAL_ALL
    P = om.planted(om.Cell(o, W, W - 1, False, "fused", False, False, 128, 6, 2, 1, 20 + W))
    Bs, Rs, Ts, _, _ = P.view(o)
    tw = torch.from_numpy(np.concatenate([x[:n] for x, n in zip(P.tw, Ts)]).astype(np.float64))

    def terms_of(r, img, txt, tp, b, y):
        iw = torch.from_numpy(P.iw[r][:Rs[r]].astype(np.float64))
        return torch_focal_terms(img, txt, tp, b, y, o.focal[0], o.focal[1], iw, tw)

    _terms_against_autograd(o, W, 20 + W, terms_of)


@pytest.mark.parametrize("W", [1, 2, 3])
@pytest.mark.parametrize("source", ["ids", "sets"])
def test_teacher_with_every_option_but_focal_matches_autograd(W, source):
    """A teacher with extras (with ids or sets of their own), weights, groups, per-sample losses and top-K at once,
    against float64 autograd of exclude_groups_oracle.torch_terms with the teacher (rows for every image and text)."""
    ids = source == "ids"
    o = om.Options(ids=ids, xtexts=True, ximages=True, xt_ids=ids, xi_ids=ids, labels=0 if ids else 2,
                   xt_sets=not ids, xi_sets=not ids, weights=True, groups=True, teacher=True, metrics=True,
                   losses=True, topk=5)
    assert om.mode_of(o) == "distill_opts"
    seed = 30 + W + 3 * ids
    P = om.planted(om.Cell(o, W, W - 1, False, "fused", False, False, 128, 6, 2, 1, seed))
    Bs, Rs, Ts, _, _ = P.view(o)
    timgs, ttxts = P.teacher(o)
    assert [len(x) for x in timgs] == list(Rs) and [len(x) for x in ttxts] == list(Ts)
    tw = torch.from_numpy(np.concatenate([x[:n] for x, n in zip(P.tw, Ts)]).astype(np.float64))
    ttxt = torch.from_numpy(np.concatenate(ttxts))

    def terms_of(r, img, txt, tp, b, y):
        iw = torch.from_numpy(P.iw[r][:Rs[r]].astype(np.float64))
        return torch_terms(img, txt, tp, b, y, iw, tw,
                           teacher=(torch.from_numpy(timgs[r]), ttxt, om.TTP, om.TBIAS, om.LAM))

    _terms_against_autograd(o, W, seed, terms_of)


def _same(a, b, tag):
    assert len(a) == len(b)
    for ra, rb in zip(a, b):
        for k in ("loss", "dimg", "dt_prime", "dbias"):
            assert np.array_equal(np.asarray(ra[k]), np.asarray(rb[k])), f"{tag}: {k}"
        for x, y in zip(ra["contrib"], rb["contrib"], strict=True):
            assert np.array_equal(x, y), f"{tag}: contrib"


def test_reduces_to_the_single_feature_oracles():
    """With options off the composed oracle gives what the single-feature oracles give, bit for bit."""
    P = om.planted(_cell(3, seed=7))
    f = P.view
    # plain, ids, weights, hard negatives, extra texts / images with ids: closed_form_extras / closed_form_weighted
    for o in (om.Options(), om.Options(ids=True), om.Options(weights=True), om.Options(xtexts=True),
              om.Options(ids=True, xtexts=True, xt_ids=True, ximages=True, xi_ids=True, weights=True),
              om.Options(ximages=True, xtexts=True)):
        Bs, Rs, Ts, imgs, txts = f(o)
        got = om.oracle(P, o)
        iw = [x[:n].astype(np.float64) for x, n in zip(P.iw, Rs)] if o.weights else None
        tw = [x[:n].astype(np.float64) for x, n in zip(P.tw, Ts)] if o.weights else None
        _same(got, closed_form_extras(imgs, txts, Bs, om.TP, om.BIAS, om.labels(P, o), iw, tw), f"extras {o}")
        want = sample_losses(imgs, txts, Bs, om.TP, om.BIAS, om.labels(P, o), iw, tw)
        for r in range(3):
            assert np.array_equal(got[r]["image_loss"], want[r]["image_loss"])
            assert np.allclose(got[r]["text_loss"], want[r]["text_loss"], rtol=1e-14, atol=0)
        if not (o.xtexts or o.ximages):
            _same(got, closed_form_weighted(imgs, txts, om.TP, om.BIAS, iw, tw, om.labels(P, o)), f"weighted {o}")
    # a teacher without extras: closed_form_distill
    o = om.Options(ids=True, weights=True, teacher=True)
    Bs, Rs, Ts, imgs, txts = f(o)
    _same(om.oracle(P, o), closed_form_distill(imgs, txts, om.TP, om.BIAS, *P.teacher(o), om.TTP, om.TBIAS, om.LAM,
                                               [x[:b] for x, b in zip(P.iw, Bs)], [x[:b] for x, b in zip(P.tw, Bs)],
                                               om.labels(P, o)), "distill")
    # a teacher with extras, ids and groups: closed_form_distill_options on labels built here (divided by B_r)
    o = om.Options(ids=True, xtexts=True, xt_ids=True, ximages=True, weights=True, groups=True, teacher=True)
    Bs, Rs, Ts, imgs, txts = f(o)
    iw, tw = [x[:n] for x, n in zip(P.iw, Rs)], [x[:n] for x, n in zip(P.tw, Ts)]
    lab = group_labels(label_blocks(Bs, Rs, Ts, P.ids, P.xt_ids), [x[:n] for x, n in zip(P.ig, Rs)],
                       [x[:n] for x, n in zip(P.tg, Ts)])
    want = closed_form_distill_options(imgs, txts, om.TP, om.BIAS, [x[:n] for x, n in zip(P.timgs, Rs)],
                                       [x[:n] for x, n in zip(P.ttxts, Ts)], om.TTP, om.TBIAS, om.LAM, lab, Bs, iw, tw)
    _same(om.oracle(P, o), want, "distill options")
    # label sets with extras that carry sets, hard-negative images (empty sets), weights and groups: closed_form_sets
    o = om.Options(labels=3, xtexts=True, xt_sets=True, ximages=True, weights=True, groups=True)
    Bs, Rs, Ts, imgs, txts = f(o)
    iw, tw = [x[:n] for x, n in zip(P.iw, Rs)], [x[:n] for x, n in zip(P.tw, Ts)]
    isets, tsets = P.sets(o)
    for si, st, b in zip(isets, tsets, Bs):
        assert (si[b:] == -1).all() and (st[b:] >= 0).any(axis=1).all() and np.array_equal(si[:b], st[:b])
    got = om.oracle(P, o)
    _same(got, closed_form_sets(imgs, txts, om.TP, om.BIAS, isets, tsets, Bs, iw, tw,
                                [x[:n] for x, n in zip(P.ig, Rs)], [x[:n] for x, n in zip(P.tg, Ts)]), "label sets")
    # the focal terms on the same labels: closed_form_focal; gamma 0 without alpha: the SigLIP terms
    for gamma, alpha in om.FOCALS + ((0.0, None),):
        of = dataclasses.replace(o, focal=(gamma, alpha))
        _same(om.oracle(P, of), closed_form_focal(imgs, txts, om.TP, om.BIAS, om.labels(P, o), gamma, alpha, Bs, iw,
                                                   tw), f"focal {gamma} {alpha}")
    for a, b in zip(om.oracle(P, dataclasses.replace(o, focal=(0.0, None))), got):
        for k in ("loss", "dimg", "dt_prime", "dbias", "image_loss", "text_loss"):
            assert om.rel(a[k], b[k]) < 1e-13, k
    # M = 1 sets hold the id alone: the sample ids' labels
    for a, b in zip(om.labels(P, om.Options(labels=1)), om.labels(P, om.Options(ids=True))):
        for ya, yb in zip(a, b):
            assert np.array_equal(ya, yb)
    # retrieval: the top-1 oracles
    for o in (om.Options(), om.Options(ids=True)):
        _, _, _, imgs, txts = f(o)
        ret = om.retrieval(P, o, 1)
        want = retrieval_metrics(imgs, txts, P.ids if o.ids else None)
        for r in range(3):
            assert np.array_equal(ret[r]["i2t_index"], want[r]["i2t_index"])
            assert np.array_equal(ret[r]["t2i_index"], want[r]["t2i_index"])
            assert ret[r]["top1"][0] == np.float32(want[r]["i2t_top1"]) or \
                abs(ret[r]["top1"][0] - want[r]["i2t_top1"]) < 1e-6
    o = om.Options(ids=True, xtexts=True, xt_ids=True, ximages=True, xi_ids=True)
    Bs, Rs, Ts, imgs, txts = f(o)
    ret = om.retrieval(P, o, 3)
    want = retrieval_metrics_extras(imgs, txts, Bs, P.ids, P.xt_ids, P.xi_ids)
    for r in range(3):
        assert np.array_equal(ret[r]["i2t_index"], want[r]["i2t_index"])
        assert np.array_equal(ret[r]["t2i_index"], want[r]["t2i_index"])
        assert abs(ret[r]["top1"][1] - want[r]["t2i_top1"]) < 1e-6


# ---------------------------------------------------------------------------------------------------------------------
# every cell: each option it turns on changes what it checks
# ---------------------------------------------------------------------------------------------------------------------
def _outputs(cell, res, r):
    """The loss-side outputs the GPU test compares for the cell, as arrays."""
    x = res[r]
    out = {"loss": x["loss"]}
    if cell.sched != "fwd":
        out.update(dimg=x["dimg"], dt_prime=x["dt_prime"], dbias=x["dbias"],
                   **{f"contrib{c}": v for c, v in enumerate(x["contrib"])})
    if cell.opts.losses:
        out.update(image_loss=x["image_loss"], text_loss=x["text_loss"])
    return out


def _cut(a, b):
    """a and b over their common leading rows (an option that removes extras removes rows)."""
    a, b = np.atleast_1d(np.asarray(a)), np.atleast_1d(np.asarray(b))
    n = min(len(a), len(b))
    return a[:n], b[:n]


@pytest.mark.parametrize("cell", om.TABLE, ids=lambda c: c.name)
def test_every_option_of_a_cell_matters(cell):
    P = om.planted(cell)
    o = cell.opts
    full = _outputs(cell, om.oracle(P, o), cell.r)
    assert o.removals() or not (o.ids or o.labels or o.weights or o.groups or o.focal or o.teacher or o.xtexts or
                                o.ximages)
    for what, less in o.removals().items():
        part = _outputs(cell, om.oracle(P, less), cell.r)
        moved = max(om.rel(*_cut(part[k], full[k])[::-1]) for k in full)
        assert moved > 20 * om.TOL, f"{cell.name}: removing {what} moves its outputs by {moved:.2e} only"


# ---------------------------------------------------------------------------------------------------------------------
# coverage, derived from the table
# ---------------------------------------------------------------------------------------------------------------------
def _branch(mode, rt, fine):
    """A launch's runtime options as the coverage counts them. fine=False counts the iota ids of a positional step with
    extras of both kinds as ids (the branch they take), and under label sets as the sets they are folded into (the
    label-set pre-pass; kModeLabels has no ids option); fine=True keeps them apart, and keeps a teacher step in a
    distill-extras context apart from one in a distillation context (the workspace layout the kernel reads)."""
    if fine:
        return rt
    d = dict(rt)
    d.pop("extras_ctx", None)
    if mode == "labels":
        del d["ids"]
    elif d.get("sets") and d["ids"] == "iota":
        d["ids"] = False
    return tuple((k, bool(v)) for k, v in sorted(d.items()))


def _coverage(table, fine=False):
    """(instantiations, runtime combinations, mode-axis pairings) the table runs (iota ids as _branch counts them)."""
    inst, combos, pairs = set(), set(), set()
    for cell in table:
        for i, rt in om.route(cell):
            inst.add(tuple((v if fine else bool(v)) if k == 3 else v for k, v in enumerate(i)))
            combos.add((i[0], _branch(i[0], rt, fine)))
        for axis in om.axis_values(cell.mode):
            pairs.add((cell.mode, axis, om.axis_of(cell, axis)))
    return inst, combos, pairs


def _required():
    inst = set().union(*(om.instantiations(m) for m in om.MODES))
    combos = {(m, tuple(sorted(f.items()))) for m in om.MODES if m != "loss" for f in om.runtime_combos(m)}
    combos |= {("loss", ())}
    pairs = {(m, a, v) for m in om.MODES for a, vals in om.axis_values(m).items() for v in vals}
    return inst, combos, pairs


def test_coverage_of_instantiations_runtime_branches_and_axes():
    inst, combos, pairs = _coverage(om.TABLE)
    need_i, need_c, need_p = _required()
    counts = {m: len([i for i in need_i if i[0] == m]) for m in om.MODES}
    assert counts == dict(loss=48, sample_loss=6, topk=6, groups=6, labels=6, focal=6, distill=3, distill_opts=3)
    assert sum(counts.values()) == 84
    assert {m: len([c for c in need_c if c[0] == m]) for m in om.MODES if m != "loss"} == \
        dict(sample_loss=8, topk=16, groups=32, labels=32, focal=96, distill=8, distill_opts=88)
    assert need_i <= inst, f"instantiations never run: {sorted(need_i - inst)}"
    assert need_c <= combos, f"runtime combinations never run: {sorted(need_c - combos)}"
    assert need_p <= pairs, f"modes never paired with: {sorted(need_p - pairs)}"


# the loss modes of csrc/siglip_kernels.cu by the matrix's names; kModeOut is the gradient kernel
KERNEL_MODES = {"kModeLoss": "loss", "kModeSampleLoss": "sample_loss", "kModeTopK": "topk", "kModeGroups": "groups",
                "kModeLabels": "labels", "kModeFocal": "focal", "kModeDistill": "distill",
                "kModeDistillOpts": "distill_opts", "kModeOut": None}


def _dispatched_modes():
    """Every kMode... that launch_gemm and launch_distill_opts launch a kernel of (launch_impl<kMode...> or
    SIGLIP_LAUNCH_STAGES(kMode...))."""
    src = (pathlib.Path(__file__).resolve().parents[1] / "distributed_sigmoid_loss_b200" / "csrc" /
           "siglip_kernels.cu").read_text()
    found = set()
    for fn in ("launch_gemm", "launch_distill_opts"):
        m = re.search(r"^(?:static )?int " + fn + r"\([^;{]*\{(.*?)^\}", src, re.M | re.S)
        assert m, f"no definition of {fn}"
        found |= set(re.findall(r"(?:launch_impl<|SIGLIP_LAUNCH_STAGES\()(kMode\w+)", m.group(1)))
    return found


def test_the_matrix_has_every_loss_mode_launch_gemm_dispatches_to():
    """A loss mode added to launch_gemm without a row in the matrix (MODES, route, runtime_options) fails here."""
    found = _dispatched_modes()
    assert found <= set(KERNEL_MODES), f"loss modes the option matrix does not know: {sorted(found - set(KERNEL_MODES))}"
    assert {KERNEL_MODES[k] for k in found} - {None} == set(om.MODES)
    assert {c.mode for c in om.TABLE} == set(om.MODES)


def test_no_cell_is_redundant():
    """Each cell is the only one that runs some instantiation, runtime combination or pairing (iota ids apart from
    sample ids): removing a cell from the table loses coverage."""
    full = _coverage(om.TABLE, fine=True)
    for k, cell in enumerate(om.TABLE):
        rest = _coverage(om.TABLE[:k] + om.TABLE[k + 1:], fine=True)
        assert any(not (n <= h) for n, h in zip(full, rest)), f"{cell.name} covers nothing no other cell covers"


def test_table_respects_the_refusals():
    for cell in om.TABLE:
        o = cell.opts
        assert o.valid(), cell.name
        assert not (cell.panels and cell.sched == "split"), cell.name
        assert not (cell.bidir and cell.W == 1), cell.name
        assert 0 <= cell.r < cell.W and cell.cluster in om.CLUSTERS and cell.stages in (4, 6), cell.name
        if cell.panels:
            assert cell.budget_mib() > 0
    assert len({c.name for c in om.TABLE}) == len(om.TABLE)
    assert not om.Options(xt_ids=True, xtexts=True).valid() and not om.Options(xt_sets=True, xtexts=True).valid()
    assert not om.Options(ids=True, labels=2).valid() and not om.Options(teacher=True, focal=(2.0, None)).valid()
    assert om.Options(teacher=True, xtexts=True, ximages=True, groups=True, labels=2, losses=True, topk=5).valid()


# ---------------------------------------------------------------------------------------------------------------------
# exactness of the planted data
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W,panels", [(1, False), (3, False), (2, True)])
def test_planted_operands_and_logits_are_exact(W, panels):
    P = om.planted(_cell(W, panels, seed=11))
    I, T = np.concatenate(P.imgs), np.concatenate(P.txts)
    for x in (I, T, np.concatenate(P.timgs), np.concatenate(P.ttxts)):
        t = torch.from_numpy(x)
        assert torch.equal(t.to(torch.bfloat16).double(), t)
        assert torch.equal((t * 16).half().double() / 16, t)
    S64 = I @ T.T
    S32 = torch.from_numpy(I).float() @ torch.from_numpy(T).float().T
    assert np.array_equal(S32.double().numpy(), S64)
    # (16 x)(16 y) in fp32 over D, then 1 / 256: what the fp16 operand path accumulates
    S16 = (torch.from_numpy(I * 16).float() @ torch.from_numpy(T * 16).float().T) / 256.0
    assert np.array_equal(S16.double().numpy(), S64)
    TI, TT = np.concatenate(P.timgs), np.concatenate(P.ttxts)
    assert np.array_equal((torch.from_numpy(TI).float() @ torch.from_numpy(TT).float().T).double().numpy(), TI @ TT.T)
    # the weights are fp32 values, and the negatives carry weight: sigma(z) of a same-group negative is not small
    assert all(w.dtype == np.float32 for w in P.iw + P.tw)
    lab = om.labels(P, dataclasses.replace(ALL, groups=False))[0][0]
    z = math.exp(om.TP) * (P.imgs[0] @ P.txts[0].T) + om.BIAS
    same = P.ig[0][:, None] == P.tg[0][None, :]
    assert (1 / (1 + np.exp(-z[(lab < 0) & same]))).mean() > 0.1
