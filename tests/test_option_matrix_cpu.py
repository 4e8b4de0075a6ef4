"""The option matrix (tests/option_matrix.py) on the CPU: the composed oracle against float64 autograd with every
non-distillation option on, its reduction to the single-feature oracles, every cell's sensitivity to each option it
turns on, the table's coverage of the loss kernel's instantiations and runtime branches, and the exactness of the
planted logits."""
import dataclasses
import itertools
import math

import numpy as np
import pytest
import torch

import option_matrix as om
from distill_oracle import closed_form_distill
from exclude_groups_oracle import torch_loss, torch_terms
from extra_images_oracle import closed_form_extras, retrieval_metrics_extras
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
    # a teacher: closed_form_distill
    o = om.Options(ids=True, weights=True, teacher=True)
    Bs, Rs, Ts, imgs, txts = f(o)
    _same(om.oracle(P, o), closed_form_distill(imgs, txts, om.TP, om.BIAS, P.timgs, P.ttxts, om.TTP, om.TBIAS, om.LAM,
                                               [x[:b] for x, b in zip(P.iw, Bs)], [x[:b] for x, b in zip(P.tw, Bs)],
                                               om.labels(P, o)), "distill")
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
    assert o.removals() or not (o.ids or o.weights or o.groups or o.teacher or o.xtexts or o.ximages)
    for what, less in o.removals().items():
        part = _outputs(cell, om.oracle(P, less), cell.r)
        moved = max(om.rel(*_cut(part[k], full[k])[::-1]) for k in full)
        assert moved > 20 * om.TOL, f"{cell.name}: removing {what} moves its outputs by {moved:.2e} only"


# ---------------------------------------------------------------------------------------------------------------------
# coverage, derived from the table
# ---------------------------------------------------------------------------------------------------------------------
def _coverage(table, fine=False):
    """(instantiations, runtime combinations, mode-axis pairings) the table runs. fine=False counts the iota ids of a
    positional step with extras of both kinds as ids (the branch they take); fine=True keeps them apart."""
    def norm(v):
        return v if fine else bool(v)

    inst, combos, pairs = set(), set(), set()
    for cell in table:
        for i, rt in om.route(cell):
            inst.add(tuple(norm(v) if k == 3 else v for k, v in enumerate(i)))
            combos.add((i[0], tuple((k, norm(v)) for k, v in rt)))
        for axis in om.axis_values(cell.mode):
            pairs.add((cell.mode, axis, om.axis_of(cell, axis)))
    return inst, combos, pairs


def _required():
    inst = set().union(*(om.instantiations(m) for m in om.MODES))
    combos = {(m, tuple(sorted(zip(om.runtime_options(m), v))))
              for m in om.MODES if m != "loss"
              for v in itertools.product((False, True), repeat=len(om.runtime_options(m)))}
    combos |= {("loss", ())}
    pairs = {(m, a, v) for m in om.MODES for a, vals in om.axis_values(m).items() for v in vals}
    return inst, combos, pairs


def test_coverage_of_instantiations_runtime_branches_and_axes():
    inst, combos, pairs = _coverage(om.TABLE)
    need_i, need_c, need_p = _required()
    counts = {m: len([i for i in need_i if i[0] == m]) for m in om.MODES}
    assert counts == dict(loss=48, sample_loss=6, topk=6, groups=6, distill=3)
    assert {m: len([c for c in need_c if c[0] == m]) for m in om.MODES if m != "loss"} == \
        dict(sample_loss=8, topk=16, groups=32, distill=8)
    assert need_i <= inst, f"instantiations never run: {sorted(need_i - inst)}"
    assert need_c <= combos, f"runtime combinations never run: {sorted(need_c - combos)}"
    assert need_p <= pairs, f"modes never paired with: {sorted(need_p - pairs)}"


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
    assert not om.Options(teacher=True, groups=True).valid() and not om.Options(xt_ids=True, xtexts=True).valid()


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
    # the weights are fp32 values, and the negatives carry weight: sigma(z) of a same-group negative is not small
    assert all(w.dtype == np.float32 for w in P.iw + P.tw)
    lab = om.labels(P, dataclasses.replace(ALL, groups=False))[0][0]
    z = math.exp(om.TP) * (P.imgs[0] @ P.txts[0].T) + om.BIAS
    same = P.ig[0][:, None] == P.tg[0][None, :]
    assert (1 / (1 + np.exp(-z[(lab < 0) & same]))).mean() > 0.1
