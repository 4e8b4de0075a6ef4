"""CPU checks of distillation from a frozen teacher: the float64 oracle against autograd of a direct restatement, its
lambda = 0 reduction to the hard-label oracle (with ids and weights too), and the modules' argument errors (raised
before any GPU work)."""
import math

import numpy as np
import pytest
import torch

from distill_oracle import closed_form_distill
from sample_weights_oracle import closed_form_weighted, label_blocks


def _unit(g, n, D):
    x = g.standard_normal((n, D))
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def _close(a, b, tol=1e-10):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    assert np.abs(a - b).max() <= tol * max(1.0, np.abs(b).max()), np.abs(a - b).max()


def _problem(Bs, D, DT, seed, ids=False):
    g = np.random.default_rng(seed)
    imgs = [_unit(g, b, D) for b in Bs]
    txts = [_unit(g, b, D) for b in Bs]
    timgs = [_unit(g, b, DT) for b in Bs]
    ttxts = [_unit(g, b, DT) for b in Bs]
    idb = [g.integers(0, max(Bs), b) for b in Bs] if ids else None
    iws = [g.random(b) for b in Bs]
    tws = [g.random(b) for b in Bs]
    return imgs, txts, timgs, ttxts, idb, iws, tws


@pytest.mark.parametrize("Bs,ids", [([7], False), ([5, 9, 4], False), ([6, 6], True)])
def test_oracle_matches_autograd_of_the_restatement(Bs, ids):
    imgs, txts, timgs, ttxts, idb, iws, tws = _problem(Bs, 12, 5, seed=len(Bs), ids=ids)
    tp, b, ttp, tb, lam = math.log(10.0), -6.0, math.log(14.0), -4.0, 0.35
    labels = label_blocks(Bs, Bs, idb)
    ref = closed_form_distill(imgs, txts, tp, b, timgs, ttxts, ttp, tb, lam, iws, tws, labels)
    T = [torch.tensor(x, dtype=torch.float64, requires_grad=True) for x in txts]
    for r, img in enumerate(imgs):
        I = torch.tensor(img, requires_grad=True)
        tpv = torch.tensor(tp, dtype=torch.float64, requires_grad=True)
        bv = torch.tensor(b, dtype=torch.float64, requires_grad=True)
        loss = 0.0
        for c, txt in enumerate(T):
            z = torch.exp(tpv) * I @ txt.T + bv
            p = torch.sigmoid(math.exp(ttp) * torch.tensor(timgs[r] @ ttxts[c].T) + tb)
            y = torch.tensor((labels[r][c] > 0).astype(np.float64))
            q = (1 - lam) * y + lam * p
            w = torch.tensor(iws[r][:, None] * tws[c][None, :])
            # binary cross-entropy against the soft target q, in its usual form
            bce = -(q * torch.nn.functional.logsigmoid(z) + (1 - q) * torch.nn.functional.logsigmoid(-z))
            loss = loss + (w * bce).sum() / img.shape[0]
        for x in T:
            x.grad = None
        loss.backward()
        # -(q log sigma(z) + (1 - q) log sigma(-z)) = softplus(z) - q z exactly
        _close(ref[r]["loss"], float(loss.detach()))
        _close(ref[r]["dimg"], I.grad.numpy())
        _close(ref[r]["dt_prime"], float(tpv.grad))
        _close(ref[r]["dbias"], float(bv.grad))
        for c, x in enumerate(T):
            _close(ref[r]["contrib"][c], x.grad.numpy())


@pytest.mark.parametrize("ids,weights", [(False, False), (True, False), (False, True), (True, True)])
def test_lambda_zero_is_the_hard_label_oracle(ids, weights):
    Bs = [6, 9, 5]
    imgs, txts, timgs, ttxts, idb, iws, tws = _problem(Bs, 10, 7, seed=3, ids=ids)
    iws, tws = (iws, tws) if weights else (None, None)
    labels = label_blocks(Bs, Bs, idb)
    got = closed_form_distill(imgs, txts, 2.0, -3.0, timgs, ttxts, 1.0, 0.5, 0.0, iws, tws, labels)
    ref = closed_form_weighted(imgs, txts, 2.0, -3.0, iws, tws, labels)
    for x, y in zip(got, ref):
        for k in ("loss", "dimg", "dt_prime", "dbias"):
            _close(x[k], y[k])
        for a, b in zip(x["contrib"], y["contrib"]):
            _close(a, b)


def test_teacher_equal_to_student_at_lambda_one_has_zero_gradient():
    imgs, txts, _, _, _, _, _ = _problem([8], 6, 6, seed=4)
    res = closed_form_distill(imgs, txts, 1.5, -2.0, imgs, txts, 1.5, -2.0, 1.0)[0]
    for k in ("dimg", "dt_prime", "dbias"):
        _close(res[k], np.zeros_like(np.asarray(res[k])), 1e-14)


def _mods():
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    return DDPSigmoidLoss, SigLipLoss


@pytest.mark.parametrize("bad", [0.0, -0.1, 1.5, True, "0.5", float("nan")])
def test_lambda_outside_the_unit_interval_is_refused(bad):
    for M in _mods():
        kw = dict(gpu_batch_size=4) if M.__name__ == "DDPSigmoidLoss" else {}
        with pytest.raises(RuntimeError, match="distill"):
            M(distill=bad, **kw)


@pytest.mark.parametrize("opt", [dict(hard_negatives=2), dict(multi_positive=True, extra_texts=2),
                                 dict(extra_images=2)])
def test_extras_are_refused(opt):
    for M in _mods():
        kw = dict(gpu_batch_size=4) if M.__name__ == "DDPSigmoidLoss" else {}
        with pytest.raises(RuntimeError, match="distill cannot be combined"):
            M(distill=0.5, **kw, **opt)


def _forward(M, mod, x, **teacher):
    if M.__name__ == "DDPSigmoidLoss":
        names = dict(scale="teacher_t_prime", bias="teacher_bias")
        return mod(x, x, **{names.get(k, k): v for k, v in teacher.items()})
    names = dict(scale="teacher_logit_scale", bias="teacher_logit_bias")
    return mod(x, x, torch.tensor(1.0), torch.tensor(-1.0), **{names.get(k, k): v for k, v in teacher.items()})


def test_teacher_arguments_are_checked_before_any_gpu_work():
    x = torch.randn(4, 8)
    t = torch.randn(4, 6)
    s = torch.tensor(1.0)
    for M in _mods():
        kw = dict(gpu_batch_size=4) if M.__name__ == "DDPSigmoidLoss" else {}
        plain, mod = M(**kw), M(distill=0.5, **kw)
        with pytest.raises(RuntimeError, match="without distill"):
            _forward(M, plain, x, teacher_image=t)
        with pytest.raises(RuntimeError, match="forward needs"):
            _forward(M, mod, x, teacher_image=t, teacher_text=t, scale=s)
        with pytest.raises(RuntimeError, match="requires grad"):
            _forward(M, mod, x, teacher_image=t.clone().requires_grad_(True), teacher_text=t, scale=s, bias=s)
        with pytest.raises(RuntimeError, match="shape"):
            _forward(M, mod, x, teacher_image=t[:3], teacher_text=t[:3], scale=s, bias=s)
        with pytest.raises(RuntimeError, match="same shape"):
            _forward(M, mod, x, teacher_image=t, teacher_text=torch.randn(4, 5), scale=s, bias=s)
        with pytest.raises(RuntimeError, match="floating-point"):
            _forward(M, mod, x, teacher_image=t.long(), teacher_text=t, scale=s, bias=s)
        with pytest.raises(RuntimeError, match="0-dim"):
            _forward(M, mod, x, teacher_image=t, teacher_text=t, scale=torch.ones(2), bias=s)
        if torch.cuda.is_available():
            with pytest.raises(RuntimeError, match="is on"):
                _forward(M, mod, x, teacher_image=t.cuda(), teacher_text=t, scale=s, bias=s)
