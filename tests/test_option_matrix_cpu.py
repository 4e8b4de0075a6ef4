"""The option matrix (tests/option_matrix.py) on the CPU: the composed oracle against float64 autograd with every
non-distillation option on, with the focal terms and every other non-teacher option, and with a teacher and every option
but the focal terms; its reduction to the single-feature oracles; every cell's sensitivity to each option it turns on;
the table's coverage of the loss kernel's instantiations and runtime branches; the table's modes against the loss modes
launch_gemm dispatches to; the exactness of the planted logits; and the series path: the slab model of
tests/slab_paths.py, the cold family's coverage of every instantiation and runtime combination in series slabs, and
each cold cell's sensitivity to a bug local to its series slabs; the loss kernel's tile schedule (tests/tile_schedule.py),
the multi-tile families' coverage of the state a CTA carries from one tile into the next, and each family's
sensitivity to a leak of that state."""
import dataclasses
import functools
import math
import pathlib
import re

import numpy as np
import pytest
import torch

import option_matrix as om
import slab_paths as sp
import tile_schedule as ts
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


# ---------------------------------------------------------------------------------------------------------------------
# the series path: the slab model (tests/slab_paths.py) and the cold family
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _slabs(cell):
    return om.cell_slabs(cell, om.planted(cell))


def _student_series(cell, m):
    """The slabs of a launch whose student takes the series path (any class in the teacher modes)."""
    return m.series if cell.opts.teacher else m.series & (m.cls == sp.FREE)


def test_slab_classes_hold_exactly_the_special_elements():
    """The model's classes against the kernel's geometry (test_protocol_model's slab-class test on the 16 x 32 slabs):
    every element past the matrix lies in an edge slab and only edge slabs hold one; every own positional positive lies
    in a diag slab, which only a diagonal 128 x 128 tile holds; positives and excluded pairs never lie in a free slab."""
    g = np.random.default_rng(3)
    for M, N in [(300, 337), (128, 128), (136, 200), (520, 600), (40, 24), (257, 129)]:
        for own in (False, True):
            y = np.where(g.random((M, N)) < 0.002, 1, np.where(g.random((M, N)) < 0.002, 0, -1))
            cls = sp.classes(M, N, own, y)
            nb, nc = cls.shape
            assert (nb, nc) == (-(-M // 16), -(-N // 32))
            for b in range(nb):
                for c in range(nc):
                    masked = b * 16 + 16 > M or c * 32 + 32 > N
                    assert (cls[b, c] == sp.EDGE) == masked
                    on_diag = own and any(b * 16 + i == c * 32 + j for i in range(16) for j in range(32)
                                          if b * 16 + i < M and c * 32 + j < N)
                    if on_diag and not masked:
                        assert cls[b, c] == sp.DIAG and (b * 16) // 128 == (c * 32) // 128
                    if cls[b, c] == sp.DIAG:
                        assert on_diag
                    blk = y[b * 16:b * 16 + 16, c * 32:c * 32 + 32]
                    if (blk >= 0).any():
                        assert cls[b, c] != sp.FREE


def test_slab_votes_are_the_kernels_fp32_votes():
    """fmaf(max s, t_eff, bias) in fp32 with t_eff = expf(t') (bf16) or expf(t') / 256 on 256 s (fp16(16 x)): the same
    value; a slab's elements past the matrix read s = 0 (z = bias); the series path iff the vote is below kFastZ."""
    s = np.full((20, 40), 23 / 64.0)
    s[3, 5] = 24 / 64.0
    m = sp.slab_map(s, -np.ones_like(s), False, om.TP, om.BIAS)
    assert m.z[0, 0] == np.float32(np.float32(5.0) * np.float32(24 / 64.0) + np.float32(-6.0))
    assert m.z[0, 0] > sp.FAST_Z and m.z[0, 1] < sp.FAST_Z and m.z[0, 1] == np.float32(5 * 23 / 64 - 6)
    assert np.array_equal(m.z, sp.slab_map(s, -np.ones_like(s), False, om.TP, om.BIAS, f16=True).z)
    assert m.cls[1, 0] == sp.EDGE and m.cls[0, 1] == sp.EDGE and m.cls[0, 0] == sp.FREE
    t = sp.slab_map(-np.ones((20, 40)), -np.ones((20, 40)), False, om.TP, om.BIAS)
    assert t.z[1, 1] == np.float32(om.BIAS) and t.z[0, 0] == np.float32(-11.0)
    assert list(m.student_path(False)[0]) == ["general", "general"] and list(t.student_path(True)[0]) == ["series"] * 2


def test_slab_fast_fraction_of_the_trained_regime_is_the_models():
    """trained_regime.slab_fast_fraction counts the free slabs of slab_paths, the same as a direct float64 count."""
    from trained_regime import REGIMES, make_batch, pair_terms, slab_fast_fraction

    R = REGIMES["trained"]
    imgs, texts, _, _ = make_batch(R, (160, 96), (40, 0), 64, 5, "hn")
    fast = total = 0
    for r, row in enumerate(pair_terms(imgs, texts, R.t_prime, R.bias)):
        for c, x in enumerate(row):
            z = math.exp(R.t_prime) * x["s"] + R.bias
            M, N = z.shape
            for b in range(0, M - 15, 16):
                for c0 in range(0, N - 31, 32):
                    if r == c and b < c0 + 32 and c0 < b + 16 or (x["y"][b:b + 16, c0:c0 + 32] > 0).any():
                        continue
                    total += 1
                    fast += z[b:b + 16, c0:c0 + 32].max() < -4.2
    assert slab_fast_fraction(imgs, texts, R.t_prime, R.bias) == (fast / total, total)
    assert 0 < fast < total


def test_row_panel_windows_tile_the_step():
    """slab_paths.windows restates run_fwd_bwd's loss launches: every element of every chunk is scored once, the own
    chunk's positional diagonal only in launches that carry own_chunk, and a window's origin is a multiple of 128."""
    for cell in [c for c in om.TABLE + om.COLD if c.panels][:12] + om.COLD[:6]:
        Bs, Rs, Ts = cell.shapes()
        r = cell.r
        for c in range(cell.W):
            seen = np.zeros((Rs[r], Ts[c]), int)
            diag = np.zeros(Rs[r], bool)
            for r0, rows, c0, cols, own in sp.windows(Rs[r], Bs[r], Ts[c], c == r, om.own_pos_ids(cell),
                                                      cell.panel_rows()):
                assert r0 % 128 == 0 and c0 % 128 == 0
                seen[r0:r0 + rows, c0:c0 + cols] += 1
                if own:
                    i = np.arange(r0, r0 + rows)
                    diag[i[(i >= c0) & (i < c0 + cols)]] = True
            assert (seen == 1).all(), cell.name
            assert diag[:Bs[r]].all() == (c == r and not om.own_pos_ids(cell)), cell.name
        assert cell.panel_rows() < Rs[r] if cell.panels else cell.panel_rows() == Rs[r]


def test_warm_cells_run_no_series_slab():
    """The planted data of the table's cells (t = 5, bias = -6, group centres and duplicate ids) never votes the
    student's series path: what the cold family is for. (The teacher's vote does go either way there.)"""
    series = {}
    for cell in om.TABLE:
        for _, m in _slabs(cell):
            series[cell.mode] = series.get(cell.mode, 0) + int((m.series & (m.cls == sp.FREE)).sum())
    assert series == {m: 0 for m in om.MODES}, series


def _cold_items(cell):
    """What a cold cell covers, each only where its launches run series slabs and general slabs off the diagonal:
    its instantiations and runtime combinations (iota ids and a teacher's context apart: the coverage's fine items),
    the student x teacher vote pairs of its free slabs, and its schedule, row panels, INPUT_F16 and peer chunks."""
    out = set()
    by_route = {}
    for rt, m in _slabs(cell):
        free = m.cls == sp.FREE
        a = by_route.setdefault(rt, np.zeros(2, int))
        a += [int(_student_series(cell, m).sum()), int((free & ~m.series).sum())]
        if cell.opts.teacher:
            for sv in (False, True):
                for tv in (False, True):
                    if (free & (m.series == sv) & (m.tseries == tv)).any():
                        out.add(("votes", cell.mode, sv, tv))
        if m.chunk != cell.r and _student_series(cell, m).any() and (free & ~m.series).any():
            out.add(("peer chunk", cell.W))
    for (inst, rt), (n_series, n_general) in by_route.items():
        if n_series and n_general:
            out.add(("instantiation", inst))
            out.add(("branch", inst[0], rt))
            out.update([("sched", cell.sched), ("panels", cell.panels), ("f16", cell.f16)])
    return out


def test_cold_cells_cover_every_instantiation_and_branch_in_series_slabs():
    """Every loss-kernel instantiation and every runtime combination runs in a cold cell whose launches of it hold
    series slabs and general slabs off the diagonal; the teacher modes run every student x teacher vote pair in free
    slabs; the cold cells run each schedule, row panels, INPUT_F16 and peer chunks at W = 2 and 3 that way; every vote
    is at least slab_paths.MARGIN from kFastZ, and some series slabs have their max z just below it, some general slabs
    just above. pytest -s prints how many cold-cell slabs take each path, per mode."""
    items = set().union(*(_cold_items(c) for c in om.COLD))
    inst = {x[1] for x in items if x[0] == "instantiation"}
    inst = {tuple(bool(v) if k == 3 else v for k, v in enumerate(i)) for i in inst}
    combos = {(x[1], _branch(x[1], x[2], False)) for x in items if x[0] == "branch"}
    need_i, need_c, _ = _required()
    assert need_i <= inst, f"instantiations without series slabs: {sorted(need_i - inst)}"
    assert need_c <= combos, f"runtime combinations without series slabs: {sorted(need_c - combos)}"
    for mode in ("distill", "distill_opts"):
        for sv in (False, True):
            for tv in (False, True):
                assert ("votes", mode, sv, tv) in items, (mode, sv, tv)
    for x in [("sched", s) for s in om.SCHEDS] + [("panels", True), ("f16", True), ("peer chunk", 2),
                                                   ("peer chunk", 3)]:
        assert x in items, x
    counts, near = {}, [0, 0]
    for cell in om.COLD:
        for _, m in _slabs(cell):
            assert m.min_margin(cell.opts.teacher) >= sp.MARGIN, cell.name
            ser = _student_series(cell, m)
            gen = (m.cls == sp.FREE) & ~m.series
            near[0] += int((ser & (m.z > sp.FAST_Z - 0.01)).sum())
            near[1] += int((gen & (m.z < sp.FAST_Z + 0.1)).sum())
            c = counts.setdefault(cell.mode, {k: 0 for k in ("series", "general off the diagonal") + sp.CLASSES[:-1]})
            c["series"] += int(ser.sum())
            c["general off the diagonal"] += int(gen.sum())
            for k in sp.CLASSES[:-1]:
                c[k] += int((m.cls == k).sum())
    assert near[0] > 0 and near[1] > 0, near
    for mode, c in counts.items():
        print(f"cold cells, {mode}: " + ", ".join(f"{k} {v}" for k, v in c.items()))


def test_no_cold_cell_is_redundant():
    """Each cold cell is the only one that covers some item of _cold_items (iota ids apart from sample ids, a teacher's
    context apart): removing one from the family loses series-path coverage."""
    per = [_cold_items(c) for c in om.COLD]
    for k, cell in enumerate(om.COLD):
        rest = set().union(*(per[:k] + per[k + 1:]))
        assert per[k] - rest, f"{cell.name} covers nothing no other cold cell covers"


def _series_variants(cell):
    """The variants of the sensitivity test: the step with one thing done wrong in its series slabs only. 'series terms':
    the slabs' terms dropped; 'row weight' / 'column weight': a unit image / text weight; 'row sums' / 'column sums': the
    slabs' terms left out of the per-sample losses; 'gamma' / 'alpha': the focal terms without gamma / alpha; 'target':
    the teacher's soft target q replaced by the hard label; 'INPUT_F16 scale': t_eff off by 2^1."""
    o = cell.opts
    out = ["series terms"]
    out += ["row weight", "column weight"] if o.weights else []
    out += ["row sums", "column sums"] if o.losses else []
    out += ["gamma"] + (["alpha"] if o.focal[1] is not None else []) if o.focal else []
    out += ["target"] if o.teacher else []
    out += ["INPUT_F16 scale"] if cell.f16 else []
    return out


def _rank_outputs(cell, P, S, res):
    """Rank r's checked outputs by float64 autograd of its pair terms over the whole text set, with a variant applied to
    the elements in S ([R_r, sum T] bool): a function of the variant (None: the step as it is) giving loss, dimg, dt',
    dbias, contrib<c>, image_loss and text_loss (every rank's column sums of the own chunk: the other ranks' parts from
    the oracle's res)."""
    o, r = cell.opts, cell.r
    Bs, Rs, Ts, imgs, txts = P.view(o)
    T64 = functools.partial(torch.tensor, dtype=torch.float64)
    F = torch.nn.functional
    y = torch.from_numpy(np.concatenate(om.labels(P, o)[r], axis=1))
    txt = np.concatenate(txts)
    s0 = imgs[r] @ txt.T
    one = torch.ones(1, dtype=torch.float64)
    iw = T64(P.iw[r][:Rs[r]]) if o.weights else one
    tw = T64(np.concatenate([x[:n] for x, n in zip(P.tw, Ts)])) if o.weights else one
    p = None
    if o.teacher:
        timgs, ttxts = P.teacher(o)
        p = torch.sigmoid(math.exp(om.TTP) * T64(timgs[r] @ np.concatenate(ttxts).T) + om.TBIAS)
    Sm = torch.from_numpy(S)
    lo = np.cumsum([0] + list(Ts))
    gamma, alpha = o.focal if o.focal else (0.0, None)

    def evaluate(variant=None):
        s = T64(s0, requires_grad=True)
        tp, b = T64(om.TP, requires_grad=True), T64(om.BIAS, requires_grad=True)

        def terms(tp_=tp, iw_=iw, tw_=tw, gamma=gamma, alpha=alpha, teacher=o.teacher):
            z = torch.exp(tp_) * s + b
            w = y.abs() * iw_[:, None] * tw_[None, :]
            if o.focal is not None:
                m = torch.where(y > 0, -z, z)
                a = 1.0 if alpha is None else torch.where(y > 0, alpha, 1.0 - alpha).to(z.dtype)
                return w * a * torch.exp(-gamma * F.softplus(-m)) * F.softplus(m)
            if teacher:
                return w * (F.softplus(z) - ((1.0 - om.LAM) * (y > 0).double() + om.LAM * p) * z)
            return w * F.softplus(-torch.where(y == 0, -torch.ones_like(y), y) * z)

        full = terms()
        wrong = {"series terms": lambda: torch.zeros_like(full), "row weight": lambda: terms(iw_=one),
                 "column weight": lambda: terms(tw_=one), "gamma": lambda: terms(gamma=0.0),
                 "alpha": lambda: terms(alpha=None), "target": lambda: terms(teacher=False),
                 "INPUT_F16 scale": lambda: terms(tp_=tp + math.log(2.0))}
        summed = torch.where(Sm, wrong[variant](), full) if variant in wrong else full
        loss = summed.sum() / Bs[r]
        gs, gt, gb = torch.autograd.grad(loss, [s, tp, b])
        gs = gs.numpy()
        out = {"loss": loss.item(), "dimg": gs @ txt, "dt_prime": float(gt), "dbias": float(gb)}
        out.update({f"contrib{c}": gs[:, lo[c]:lo[c + 1]].T @ imgs[r] for c in range(cell.W)})
        t = summed.detach()   # the per-sample sums add the same terms (lrow / lcol)
        rows = torch.where(Sm, 0.0, t) if variant == "row sums" else t
        cols = torch.where(Sm, 0.0, t) if variant == "column sums" else t
        out["image_loss"] = rows.sum(axis=1).numpy()
        out["text_loss"] = res[r]["text_loss"] - res[r]["text_part"][r] + cols[:, lo[r]:lo[r + 1]].sum(axis=0).numpy()
        return out

    return evaluate


def _moved(cell, key, a, b):
    """How far a variant moves an output, in units of what the GPU test allows: the norm-and-max error over 1e-3; for
    the per-sample losses the largest per-sample error past the fixed-point words' resolution, over 1e-3 relative."""
    if key not in ("image_loss", "text_loss"):
        return om.rel(a, b) / om.TOL
    Bs, Rs, Ts = cell.shapes()
    words = sum((t + 127) // 128 + 1 for t in Ts) if key == "image_loss" else (Rs[cell.r] + 15) // 16 + cell.W
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max((np.abs(a - b) - words * 2.0 ** -32) / (om.TOL * np.abs(b) + 1e-300)))


@pytest.mark.parametrize("cell", om.COLD, ids=lambda c: c.name)
def test_a_series_path_bug_moves_what_the_cell_checks(cell):
    """For each thing the series path computes in the cell (its terms, each weight, each per-sample sum, the focal
    gamma and alpha, a teacher's target, the INPUT_F16 scale), the step with that done wrong in its series slabs only
    moves an output the GPU test checks by more than 20x its tolerance. The restatement here is the composed oracle
    (the same outputs to 1e-10), so a bug local to the series path of any instantiation fails the GPU test. One
    exception: a teacher cell that checks its loss alone sees the INPUT_F16 scale off by 2 at 8x its tolerance or more
    only (its soft targets' -q z terms move little), which the cells with gradients cover; and a text's loss holds the
    terms of every rank, so at W > 1 a column-sum bug of this rank's series slabs moves it by 10x or more."""
    P = om.planted(cell)
    Bs, Rs, Ts, _, _ = P.view(cell.opts)
    S = [np.zeros((Rs[cell.r], t), bool) for t in Ts]
    for _, m in _slabs(cell):
        S[m.chunk][m.r0:m.r0 + m.rows, m.c0:m.c0 + m.cols] |= m.elements(_student_series(cell, m))
    S = np.concatenate(S, axis=1)
    assert S.any()
    res = om.oracle(P, cell.opts)
    checked = list(_outputs(cell, res, cell.r))
    evaluate = _rank_outputs(cell, P, S, res)
    full = evaluate()
    for k in ("loss", "dimg", "dt_prime", "dbias", "image_loss", "text_loss"):
        assert om.rel(full[k], res[cell.r][k]) < 1e-10, k
    weak = []
    for v in _series_variants(cell):
        got = evaluate(v)
        moved = max(_moved(cell, k, got[k], full[k]) for k in checked)
        if moved <= (10 if v == "column sums" and cell.W > 1 else 20):
            weak.append(f"{v}: {moved:.1f}x")
    if cell.opts.teacher and cell.sched == "fwd":
        weak = [w for w in weak if not w.startswith("INPUT_F16")]
    assert not weak, f"{cell.name}: a series-path bug moves its checked outputs by {weak} of the tolerance only"


# ---------------------------------------------------------------------------------------------------------------------
# several tiles per CTA: the tile schedule (tests/tile_schedule.py) and the multi-tile family
# ---------------------------------------------------------------------------------------------------------------------
def test_tile_schedule_by_hand():
    """Schedules worked out by hand from launch_impl and decode_tile."""
    # 300 x 640 at cluster size 1 on 4 clusters, 3 k-blocks, 4 stages: 3 x 5 tiles in row-panel order
    L = ts.launch(300, 640, 1, 4, 3, 4)
    assert (L.clusters, L.tiles_m, L.tiles_n) == (4, 3, 5)
    assert L.per_cluster[0] == [ts.Tile(0, 0, 0, 0), ts.Tile(0, 4, 3, 0), ts.Tile(1, 3, 2, 1), ts.Tile(2, 2, 1, 0)]
    assert [(t.mrow, t.n_blk) for t in L.per_cluster[3]] == [(0, 3), (1, 2), (2, 1)]
    assert L.ragged() and L.max_tiles() == 4 and L.keeps_row_block() and L.changes_row_block()
    assert L.mid_ring() and L.phase_one()
    # 6 stages: the third tile starts at stage 0 again, on phase 1
    assert [(t.stage, t.phase) for t in ts.launch(300, 640, 1, 6, 3, 4).per_cluster[0]] == [(0, 0), (3, 0), (0, 1),
                                                                                           (3, 1)]
    # a teacher tile of 2 + 3 k-blocks on 4 stages: the second tile starts at stage 1, phase 1
    assert ts.num_kb(om.D, om.DT) == 5 and ts.num_kb(om.D) == 3
    assert [(t.stage, t.phase) for t in ts.launch(128, 256, 1, 4, 5, 1).per_cluster[0]] == [(0, 0), (1, 1)]
    # cluster size 2, 300 rows: row blocks 0 and 1, then 2 (rows 256..299) and 3, a phantom past row 300
    L = ts.launch(300, 256, 2, 6, 3, 66)
    assert (L.clusters, L.tiles_m, L.tiles_n) == (4, 2, 2) and L.max_tiles() == 1 and not L.ragged()
    assert L.cta_tiles(2, 0) == [(2, 0, 0, 0, False)] and L.cta_tiles(2, 1) == [(3, 0, 0, 0, True)]
    # on 3 clusters: cluster 0 runs tiles 0 and 3; its second CTA scores block 1, then the phantom block 3
    L = ts.launch(300, 256, 2, 6, 3, 3)
    assert L.cta_tiles(0, 1) == [(1, 0, 0, 0, False), (3, 1, 3, 0, True)]
    assert L.phantom_after_real() and not L.phantom_then_more() and not L.phantom_before_real()
    # the grid of the step's widest chunk: 8 clusters for a one-tile chunk, 7 of them without a tile
    L = ts.launch(128, 128, 1, 6, 3, 132, grid_n=1000)
    assert L.clusters == 8 and [len(x) for x in L.per_cluster] == [1] + [0] * 7
    # at most num_sms / cluster size clusters, whatever the co-resident count says
    assert ts.launch(4096, 4096, 4, 6, 3, 40).clusters == 33


@pytest.mark.parametrize("rows,cols,cs", [(520, 17520, 1), (520, 17520, 2), (520, 17520, 4), (2100, 300, 4),
                                          (1000, 5000, 2)])
def test_a_phantom_block_is_never_followed_by_a_real_one(rows, cols, cs):
    """The last row panel is the last in the tile order, so a CTA that scores a phantom block scores only phantom blocks
    after it; what a phantom hands on is the ring position, to its own later phantoms and to its siblings' real tiles."""
    L = ts.launch(rows, cols, cs, 4, 3, ts.H100_CLUSTERS[cs])
    assert not L.phantom_before_real()
    for c in range(L.clusters):
        for k in range(cs):
            ph = [x[4] for x in L.cta_tiles(c, k)]
            assert ph == sorted(ph)


def _multi_missing(families, clusters=None, num_sms=ts.NUM_SMS):
    """What the families' launches do not reach of the tile schedule (om.multi_items), one line per kind, naming the
    instantiations, modes and cluster sizes left out."""
    items = set().union(*(om.multi_items(c, clusters, num_sms) for c in families))
    need_i, _, _ = _required()
    need_i = {tuple(bool(v) if k >= 3 else v for k, v in enumerate(i)) for i in need_i}
    missing = []
    for what, text in (("waves", "no cluster runs 3 tiles or more in a ragged last wave"),
                       ("keep", "no cluster's consecutive tiles keep the row block"),
                       ("change", "no cluster's consecutive tiles change the row block"),
                       ("stage", "no tile starts mid-ring"), ("phase", "no tile starts at phase 1")):
        lost = sorted(i for i in need_i if (what, i) not in items)
        if lost:
            missing.append(f"{text}: {lost}")
    lost = [cs for cs in (2, 4) if ("phantom", cs) not in items]
    if lost:
        missing.append(f"no CTA scores a real block then a phantom, in a cluster that goes on, at cluster size {lost}")
    need_o = {("option", m, o) for m in om.MODES for o in (["ids", "metrics", "weights"] if m == "loss" else
                                                            om.runtime_options(m))}
    need_o |= {("option", m, "ids=iota") for m in om.MODES if "ids" in om.runtime_options(m)}
    need_o |= {("option", m, "extras_ctx") for m in ("distill", "distill_opts")}
    lost = sorted(need_o - items)
    if lost:
        missing.append(f"runtime options never on in a multi-wave launch: {[x[1:] for x in lost]}")
    if ("grid_n",) not in items:
        missing.append("no cell at W > 1 whose chunks give a cluster different tile counts")
    return missing


@pytest.mark.parametrize("family", ["MULTI", "MULTI_COLD"])
def test_multi_tile_family_reaches_the_cross_tile_state(family):
    """With an H100 SXM's co-resident clusters (132, 66, 30), every loss-kernel instantiation runs, in a cell of the
    family, a launch where some cluster scores 3 tiles or more and the last wave is ragged; consecutive tiles that keep
    and that change the row block; a tile that starts mid-ring and one at phase 1. At cluster sizes 2 and 4 a CTA scores
    a real block and then a phantom; every runtime option of every mode (iota ids and a teacher's extras context
    included) is on in a multi-wave launch; and a cell at W = 2 has chunks that give a cluster different tile counts."""
    missing = _multi_missing(getattr(om, family))
    assert not missing, f"{family}: " + "; ".join(missing)


def test_the_other_families_do_not_reach_it():
    """The option matrix and the cold family never give a cluster a second tile: the multi-tile family is what does."""
    for c in om.TABLE + om.COLD:
        assert all(L.max_tiles() <= 1 for _, _, _, L in om.cell_launches(c)), c.name
    assert len(_multi_missing(om.TABLE + om.COLD)) >= 6


def test_no_multi_cell_is_redundant():
    """Each cell of a family is the only one that reaches some item of om.multi_items, and the family does not repeat a
    cell of the option matrix or the cold family."""
    for fam in (om.MULTI, om.MULTI_COLD):
        per = [om.multi_items(c) for c in fam]
        for k, cell in enumerate(fam):
            rest = set().union(*(per[:k] + per[k + 1:]))
            assert per[k] - rest, f"{cell.name} reaches nothing no other cell of its family reaches"
    names = [c.name for c in om.TABLE + om.COLD + om.MULTI + om.MULTI_COLD]
    assert len(set(names)) == len(names)
    for c in om.MULTI + om.MULTI_COLD:
        assert c.opts.valid() and not c.panels and not (c.bidir and c.W == 1) and 0 <= c.r < c.W, c.name


# ---------------------------------------------------------------------------------------------------------------------
# a cross-tile leak moves what a multi-tile cell checks
# ---------------------------------------------------------------------------------------------------------------------
def _later_tiles(cell):
    """(chunk, launch window, ordinal, previous (m_blk, n_blk), (m_blk, n_blk)) of every real tile after a CTA's first
    in rank r's launches, global rows and the chunk's columns: what the CTA scored before it, and what it scores."""
    out = []
    for _, chunk, (r0, rows, c0, cols, own), L in om.cell_launches(cell):
        for cl in range(L.clusters):
            for k in range(L.cs):
                t = L.cta_tiles(cl, k)
                for j in range(1, len(t)):
                    if not t[j][4]:
                        out.append((chunk, (r0, rows, c0, cols), j, t[j - 1][:2], t[j][:2], L))
    return out


def _block(win, m, n, lo):
    """Rows and global columns (lo: the chunks' offsets) of tile (m, n) of a launch window, clipped to the window."""
    r0, rows, c0, cols = win
    return (np.arange(m * 128, min(m * 128 + 128, rows)) + r0,
            np.arange(n * 128, min(n * 128 + 128, cols)) + c0)


def _leak_eval(cell, P, res):
    """Rank r's checked outputs by float64 autograd of its pair terms, from the labels y [R_r, sum T], element weights
    w, logits s and the teacher's p: a function of (y, w, s, p) overrides (None: the step's own)."""
    o, r = cell.opts, cell.r
    Bs, Rs, Ts, imgs, txts = P.view(o)
    F = torch.nn.functional
    txt = np.concatenate(txts)
    y0 = np.concatenate(om.labels(P, o)[r], axis=1)
    iw = P.iw[r][:Rs[r]].astype(np.float64) if o.weights else np.ones(Rs[r])
    tw = np.concatenate([x[:n] for x, n in zip(P.tw, Ts)]).astype(np.float64) if o.weights else np.ones(len(txt))
    w0 = iw[:, None] * tw[None, :]
    s0 = imgs[r] @ txt.T
    ts0 = None
    if o.teacher:
        timgs, ttxts = P.teacher(o)
        ts0 = timgs[r] @ np.concatenate(ttxts).T
    lo = np.cumsum([0] + list(Ts))
    gamma, alpha = o.focal if o.focal else (0.0, None)

    def evaluate(y=None, w=None, s=None, ts_=None, row_extra=None):
        y = torch.from_numpy(y0 if y is None else y)
        s = torch.tensor(s0 if s is None else s, dtype=torch.float64, requires_grad=True)
        tp = torch.tensor(om.TP, dtype=torch.float64, requires_grad=True)
        b = torch.tensor(om.BIAS, dtype=torch.float64, requires_grad=True)
        z = torch.exp(tp) * s + b
        wt = y.abs() * torch.from_numpy(w0 if w is None else w)
        if o.focal is not None:
            m = torch.where(y > 0, -z, z)
            a = 1.0 if alpha is None else torch.where(y > 0, alpha, 1.0 - alpha).to(z.dtype)
            terms = wt * a * torch.exp(-gamma * F.softplus(-m)) * F.softplus(m)
        elif o.teacher:
            p = torch.sigmoid(math.exp(om.TTP) * torch.from_numpy(ts0 if ts_ is None else ts_) + om.TBIAS)
            terms = wt * (F.softplus(z) - ((1.0 - om.LAM) * (y > 0).double() + om.LAM * p) * z)
        else:
            terms = wt * F.softplus(-torch.where(y == 0, -torch.ones_like(y), y) * z)
        loss = terms.sum() / Bs[r]
        gs, gt, gb = torch.autograd.grad(loss, [s, tp, b])
        gs = gs.numpy()
        out = {"loss": loss.item(), "dimg": gs @ txt, "dt_prime": float(gt), "dbias": float(gb)}
        out.update({f"contrib{c}": gs[:, lo[c]:lo[c + 1]].T @ imgs[r] for c in range(cell.W)})
        t = terms.detach().numpy()
        out["image_loss"] = t.sum(axis=1) + (0 if row_extra is None else row_extra)
        out["text_loss"] = res[r]["text_loss"] - res[r]["text_part"][r] + t[:, lo[r]:lo[r + 1]].sum(axis=0)
        return out, t

    return evaluate, y0, w0, s0, ts0, lo


def _row_swap(cell, lo, y0):
    """(rows, columns, previous rows) of every later tile whose row block differs from the CTA's previous one."""
    out = []
    for chunk, win, j, prev, cur, L in _later_tiles(cell):
        if prev[0] != cur[0]:
            rows, cols = _block(win, *cur, 0)
            prow = np.arange(len(rows)) + prev[0] * 128 + win[0]
            out.append((rows, cols + lo[chunk], prow))
    return out


def _leak_applies(cell, leak):
    """The cell has what the leak touches: row-side labels (ids, sets, groups, iota ids), weights, per-sample losses,
    a teacher."""
    o = cell.opts
    return {"row labels": o.ids or o.labels or o.groups or om.own_pos_ids(cell), "row weights": o.weights,
            "row partials": o.losses, "student k-block": True, "teacher k-block": o.teacher}[leak]


def _leak_moves(cell, leak):
    """How far the leak moves the cell's checked outputs, in units of the tolerance (_moved)."""
    o = cell.opts
    P = om.planted(cell)
    res = om.oracle(P, o)
    evaluate, y0, w0, s0, ts0, lo = _leak_eval(cell, P, res)
    checked = list(_outputs(cell, res, cell.r))
    full, terms = evaluate()
    for k in ("loss", "dimg", "dt_prime", "dbias", "image_loss", "text_loss"):
        assert om.rel(full[k], res[cell.r][k]) < 1e-10, k
    Bs, Rs, Ts = cell.shapes()
    own = np.zeros_like(y0, bool)   # the own chunk's positional positives: geometry, not a row-side value
    if not om.own_pos_ids(cell):
        i = np.arange(Bs[cell.r])
        own[i, lo[cell.r] + i] = True
    if leak == "row labels":   # ids, sets and groups of the previous row block
        y = y0.copy()
        for rows, cols, prow in _row_swap(cell, lo, y0):
            y[np.ix_(rows, cols)] = np.where(own[np.ix_(rows, cols)], y0[np.ix_(rows, cols)], y0[np.ix_(prow, cols)])
        got, _ = evaluate(y=y)
    elif leak == "row weights":
        w = w0.copy()
        for rows, cols, prow in _row_swap(cell, lo, y0):
            w[np.ix_(rows, cols)] = w0[np.ix_(prow, cols)]
        got, _ = evaluate(w=w)
    elif leak == "row partials":   # a tile's row sums start from the previous tile's
        extra = np.zeros(Rs[cell.r])
        for chunk, win, j, prev, cur, L in _later_tiles(cell):
            rows, cols = _block(win, *cur, 0)
            prows, pcols = _block(win, *prev, 0)
            part = np.zeros(len(rows))
            if prev[0] * 128 + win[0] < win[0] + win[1]:
                n = min(len(rows), len(prows))
                part[:n] = terms[np.ix_(prows[:n], pcols + lo[chunk])].sum(axis=1)
            extra[rows] += part
        got, _ = evaluate(row_extra=extra)
    else:   # a stale k-block: the first k-block of the student's (or the teacher's) pass in one later tile
        return _stale_kblock(cell, P, evaluate, checked, full, s0, ts0, lo, leak == "teacher k-block")
    return max(_moved(cell, k, got[k], full[k]) for k in checked)


def _stale_kblock(cell, P, evaluate, checked, full, s0, ts0, lo, teacher):
    """The largest move over a few later tiles (those with the most positives) of reading, in place of the pass's first
    k-block, what the same stage held one ring lap before (tile_schedule: ring position j kb - stages)."""
    o, r = cell.opts, cell.r
    Bs, Rs, Ts, imgs, txts = P.view(o)
    timgs, ttxts = P.teacher(o) if o.teacher else (None, None)
    kbt = ts.num_kb(om.DT) if o.teacher else 0
    y = np.concatenate(om.labels(P, o)[r], axis=1)
    # a later tile whose pass starts at least one ring lap in: its stage then holds an earlier k-block of the CTA
    cands = [x for x in _later_tiles(cell) if x[2] * x[5].num_kb + (0 if teacher else kbt) >= x[5].stages]
    cands.sort(key=lambda x: -int((y[np.ix_(*_block(x[1], *x[4], lo[x[0]]))] > 0).sum()))
    best = 0.0
    for chunk, win, j, prev, cur, L in cands[:3]:
        g = j * L.num_kb + (0 if teacher else kbt)
        gp = g - L.stages
        assert gp >= 0
        jp, kp = gp // L.num_kb, gp % L.num_kb
        cl = next(c for c in range(L.clusters) for k in range(L.cs)
                  if len(L.cta_tiles(c, k)) > j and L.cta_tiles(c, k)[j][:2] == cur and L.cta_tiles(c, k)[j - 1][:2] == prev)
        crank = next(k for k in range(L.cs) if L.cta_tiles(cl, k)[j][:2] == cur)
        src = L.cta_tiles(cl, crank)[jp][:2]

        def operands(tile, k, as_teacher):
            rows = np.arange(tile[0] * 128, tile[0] * 128 + 128) + win[0]
            cols = np.arange(tile[1] * 128, tile[1] * 128 + 128) + win[2]
            A = (timgs[r] if as_teacher else imgs[r])
            B = (ttxts[chunk] if as_teacher else txts[chunk])
            a, bm = np.zeros((128, 64)), np.zeros((128, 64))
            rr, cc = rows[rows < win[0] + win[1]], cols[cols < win[2] + win[3]]
            ks = slice(k * 64, k * 64 + 64)
            a[:len(rr), :A[:, ks].shape[1]] = A[rr, ks]
            bm[:len(cc), :B[:, ks].shape[1]] = B[cc, ks]
            return a @ bm.T, len(rr), len(cc)

        cur_prod, nr, nc = operands(cur, 0, teacher)
        src_prod, _, _ = operands(src, kp if kp < kbt else kp - kbt, kp < kbt)
        rows, cols = _block(win, *cur, lo[chunk])
        delta = (src_prod - cur_prod)[:nr, :nc]
        if teacher:
            t2 = ts0.copy()
            t2[np.ix_(rows, cols)] += delta
            got, _ = evaluate(ts_=t2)
        else:
            s2 = s0.copy()
            s2[np.ix_(rows, cols)] += delta
            got, _ = evaluate(s=s2)
        best = max(best, max(_moved(cell, k, got[k], full[k]) for k in checked))
    return best


LEAKS = ("row labels", "row weights", "row partials", "student k-block", "teacher k-block")


@pytest.mark.parametrize("leak", LEAKS)
@pytest.mark.parametrize("mode", om.MODES)
def test_a_cross_tile_leak_moves_what_a_multi_tile_cell_checks(mode, leak):
    """For each leak from one tile of a CTA into its next that the tile schedule allows, some multi-tile cell of each
    mode the leak applies to moves an output the GPU test checks by more than 20x its tolerance: a tile that labels its
    rows with the previous row block's ids, sets and groups (the own positional positives stay: geometry), or weights
    them with its weights; per-sample row sums that start from the previous tile's; and one k-block of one tile (the
    student's first, or the teacher's) that reads what its stage held one ring lap before."""
    cells = sorted([c for c in om.MULTI if c.mode == mode and _leak_applies(c, leak)], key=lambda c: c.W)
    if not cells:
        pytest.skip(f"no {mode} cell has what the leak touches")
    moved = {}
    for cell in cells[:3]:
        moved[cell.name] = _leak_moves(cell, leak)
        if moved[cell.name] > 20:
            return
    pytest.fail(f"{mode}: a {leak} leak moves its cells' checked outputs by {moved} of the tolerance only")



@pytest.mark.parametrize("mode", [m for m in om.MODES if m == "topk" or "topk" in om.runtime_options(m)])
def test_a_stale_topk_floor_changes_a_multi_tile_cells_lists(mode):
    """A tile that keeps the top-K floor of the CTA's previous row block offers only the keys above the previous rows'
    floor. That floor is at least the previous row's K-th best over the previous tile (a list holds the top K of every
    key offered so far), so a row whose top-K list holds a key of this tile below that bound loses it whatever the
    stale floor was, and the GPU test compares the lists exactly. The top-K cells of the family scale rank r's first
    row block (om.TOPK_FLOOR_SCALE): the CTAs that move on from it carry a floor above their new rows' lists."""
    cells = sorted([c for c in om.MULTI if c.mode == mode and c.opts.topk > 1], key=lambda c: c.W)
    assert cells
    lost = {}
    for cell in cells[:3]:
        o, r = cell.opts, cell.r
        P = om.planted(cell)
        Bs, Rs, Ts, imgs, txts = P.view(o)
        S = imgs[r] @ np.concatenate(txts).T
        lo = np.cumsum([0] + list(Ts))
        lists = om.retrieval(P, o, o.topk)[r]["i2t_topk"]
        rows_hit = set()
        for chunk, win, j, prev, cur, L in _later_tiles(cell):
            if prev[0] == cur[0]:
                continue
            rows, cols = _block(win, *cur, lo[chunk])
            prows, pcols = _block(win, *prev, lo[chunk])
            for k, i in enumerate(rows):
                if i >= len(lists) or k >= len(prows) or len(pcols) < o.topk:
                    continue
                floor = np.sort(S[prows[k], pcols])[::-1][o.topk - 1]
                if any(S[i, g] < floor for g in lists[i] if cols[0] <= g <= cols[-1]):
                    rows_hit.add(int(i))
        lost[cell.name] = len(rows_hit)
        if rows_hit:
            return
    pytest.fail(f"{mode}: a stale top-K floor changes no row's list: {lost}")


def test_cold_multi_tile_cells_run_both_paths_on_later_tiles():
    """In a cold multi-tile cell of every mode, the tiles after a CTA's first hold series slabs and general slabs off
    the diagonal (slab_paths): both epilogue paths run on state carried from an earlier tile."""
    seen = {}
    for mode in om.MODES:
        for cell in [c for c in om.MULTI_COLD if c.mode == mode][:2]:
            later = {}
            for chunk, win, j, prev, cur, L in _later_tiles(cell):
                later.setdefault((chunk, win), set()).add(cur)
            n = np.zeros(2, int)
            for _, m in _slabs(cell):
                tiles = later.get((m.chunk, (m.r0, m.rows, m.c0, m.cols)), set())
                if not tiles:
                    continue
                nb, nc = m.cls.shape
                t = np.zeros((nb, nc), bool)
                for mb, cb in tiles:
                    t[mb * 8:mb * 8 + 8, cb * 4:cb * 4 + 4] = True
                n += [int((t & _student_series(cell, m)).sum()), int((t & (m.cls == sp.FREE) & ~m.series).sum())]
            seen[cell.name] = tuple(n)
            if n.all():
                break
        else:
            pytest.fail(f"{mode}: no cold multi-tile cell runs both paths on later tiles: {seen}")
