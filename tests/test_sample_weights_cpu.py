"""CPU checks of per-sample loss weights: the float64 oracle against autograd of the weighted op sequence, its unit-weight
reduction to the four existing oracles, the zero-weight equivalence with removing the samples, and the modules' argument
errors (raised before any GPU work)."""
import math

import numpy as np
import pytest
import torch

from extra_text_ids_oracle import closed_form_extra_text_ids
from hard_negatives_oracle import closed_form_hard_negatives
from oracle.siglip_oracle import closed_form_uneven
from sample_ids_oracle import closed_form_ids
from sample_weights_oracle import closed_form_weighted, label_blocks


def _unit(g, n, D):
    x = g.standard_normal((n, D))
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def _close(a, b, tol=1e-10):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    assert np.abs(a - b).max() <= tol * max(1.0, np.abs(b).max()), np.abs(a - b).max()


def _compare(got, ref, tol=1e-10):
    for x, y in zip(got, ref):
        for k in ("loss", "dimg", "dt_prime", "dbias"):
            _close(x[k], y[k], tol)
        assert len(x["contrib"]) == len(y["contrib"])
        for a, b in zip(x["contrib"], y["contrib"]):
            _close(a, b, tol)


def _autograd(imgs, texts, labels, a, cw, tp, bias):
    """Per rank: logits against every chunk -> w * -logsigmoid(y z) (BCE with a weight, w = a_i c_j) -> sum / B_r.
    Each rank's loss is differentiated on its own, so contrib[c] is that rank's share of chunk c's text gradient."""
    I = [torch.tensor(x, requires_grad=True) for x in imgs]
    C = [torch.tensor(x, requires_grad=True) for x in texts]
    out = []
    for r in range(len(I)):
        t_p = torch.tensor(tp, dtype=torch.float64, requires_grad=True)
        b_ = torch.tensor(bias, dtype=torch.float64, requires_grad=True)
        total = 0
        for c in range(len(C)):
            logits = I[r] @ C[c].T * t_p.exp() + b_
            w = torch.tensor(a[r])[:, None] * torch.tensor(cw[c])[None, :]
            total = total + (w * -torch.nn.functional.logsigmoid(torch.tensor(labels[r][c]) * logits)).sum()
        total = total / I[r].shape[0]
        grads = torch.autograd.grad(total, [I[r], t_p, b_] + C)
        out.append(dict(loss=float(total.detach()), dimg=grads[0].numpy(), dt_prime=float(grads[1]), dbias=float(grads[2]),
                        contrib=[x.numpy() for x in grads[3:]]))
    return out


@pytest.mark.parametrize("Bs,Ks,mode", [((6,), (0,), "pos"), ((5, 7, 4), (0, 0, 0), "pos"), ((6, 4), (3, 0), "pos"),
                                         ((5, 6, 3), (0, 0, 0), "ids"), ((6, 4), (2, 5), "ids"),
                                         ((5, 4), (3, 2), "extra_ids")])
def test_oracle_matches_autograd_of_the_weighted_op_sequence(Bs, Ks, mode):
    tp, bias = math.log(10.0), -4.0
    g = np.random.default_rng(sum(Bs) * 7 + sum(Ks))
    D = 20
    Ts = [b + k for b, k in zip(Bs, Ks)]
    imgs = [_unit(g, b, D) for b in Bs]
    texts = [_unit(g, t, D) for t in Ts]
    ids = extra_ids = None
    if mode != "pos":
        ids = [g.integers(0, 6, b) for b in Bs]            # duplicates within and across ranks
    if mode == "extra_ids":
        extra_ids = [g.integers(0, 9, k) for k in Ks]      # some match an image, some do not
    labels = label_blocks(Bs, Ts, ids, extra_ids)
    # weights in [0, 1], with exact zeros and ones among them
    a = [np.where(g.random(b) < 0.2, 0.0, np.where(g.random(b) < 0.2, 1.0, g.random(b))) for b in Bs]
    cw = [np.where(g.random(t) < 0.2, 0.0, g.random(t)) for t in Ts]
    _compare(closed_form_weighted(imgs, texts, tp, bias, a, cw, labels), _autograd(imgs, texts, labels, a, cw, tp, bias))


def test_unit_weights_reproduce_the_existing_oracles():
    tp, bias = math.log(10.0), -6.0
    g = np.random.default_rng(3)
    D = 16
    Bs, Ks = (5, 3, 6), (2, 0, 4)
    imgs = [_unit(g, b, D) for b in Bs]
    txts = [_unit(g, b, D) for b in Bs]
    extras = [_unit(g, k, D) for k in Ks]
    texts = [np.concatenate([t, e]) for t, e in zip(txts, extras)]
    Ts = [t.shape[0] for t in texts]
    ones_i = [np.ones(b) for b in Bs]
    ids = [g.integers(0, 5, b) for b in Bs]
    extra_ids = [g.integers(0, 8, k) for k in Ks]
    # positional labels, uneven batches
    _compare(closed_form_weighted(imgs, txts, tp, bias, ones_i, [np.ones(b) for b in Bs]),
             closed_form_uneven(imgs, txts, tp, bias))
    # sample ids
    _compare(closed_form_weighted(imgs, txts, tp, bias, labels=label_blocks(Bs, Bs, ids)),
             closed_form_ids(imgs, txts, ids, tp, bias))
    # hard negatives, positional and with ids
    _compare(closed_form_weighted(imgs, texts, tp, bias, ones_i, [np.ones(t) for t in Ts], label_blocks(Bs, Ts)),
             closed_form_hard_negatives(imgs, txts, extras, tp, bias))
    _compare(closed_form_weighted(imgs, texts, tp, bias, labels=label_blocks(Bs, Ts, ids)),
             closed_form_hard_negatives(imgs, txts, extras, tp, bias, ids))
    # extra texts with ids
    _compare(closed_form_weighted(imgs, texts, tp, bias, labels=label_blocks(Bs, Ts, ids, extra_ids)),
             closed_form_extra_text_ids(imgs, txts, extras, ids, extra_ids, tp, bias))


@pytest.mark.parametrize("with_ids", [False, True])
def test_zero_weight_equals_removing_the_sample(with_ids):
    """Samples with image and text weight 0 leave the loss and the gradients: the step equals the step on the batch
    without them, times (B - m) / B on the rank that lost m of its B samples (its loss still divides by B). Their own
    dimg / dtxt rows are exactly 0."""
    tp, bias = math.log(10.0), -5.0
    g = np.random.default_rng(11 + with_ids)
    D = 12
    Bs = (7, 5, 6)
    imgs = [_unit(g, b, D) for b in Bs]
    txts = [_unit(g, b, D) for b in Bs]
    ids = [g.integers(0, 6, b) for b in Bs] if with_ids else None
    drop = {0: [1, 4], 2: [0]}                               # rank -> samples dropped
    a = [np.ones(b) for b in Bs]
    for r, rows in drop.items():
        a[r][rows] = 0.0
    got = closed_form_weighted(imgs, txts, tp, bias, a, a, label_blocks(Bs, Bs, ids))
    keep = [np.setdiff1d(np.arange(b), drop.get(r, [])) for r, b in enumerate(Bs)]
    kB = [len(k) for k in keep]
    kids = None if ids is None else [i[k] for i, k in zip(ids, keep)]
    ref = closed_form_weighted([x[k] for x, k in zip(imgs, keep)], [x[k] for x, k in zip(txts, keep)], tp, bias,
                               labels=label_blocks(kB, kB, kids))
    for r, b in enumerate(Bs):
        f = kB[r] / b
        for k in ("loss", "dt_prime", "dbias"):
            _close(got[r][k], ref[r][k] * f, 1e-12)
        _close(got[r]["dimg"][keep[r]], ref[r]["dimg"] * f, 1e-12)
        assert not got[r]["dimg"][drop.get(r, [])].any()
        for c in range(len(Bs)):
            _close(got[r]["contrib"][c][keep[c]], ref[r]["contrib"][c] * f, 1e-12)
            assert not got[r]["contrib"][c][drop.get(c, [])].any()


def test_module_argument_errors_are_raised_without_a_gpu():
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    x, y = torch.randn(4, 8), torch.randn(4, 8)
    for bad in (1, "yes", None):
        with pytest.raises(RuntimeError, match="sample_weights must be a bool"):
            DDPSigmoidLoss(4, sample_weights=bad)
        with pytest.raises(RuntimeError, match="sample_weights must be a bool"):
            SigLipLoss(sample_weights=bad)
    sc = (torch.tensor(1.0), torch.tensor(0.0))
    plain = DDPSigmoidLoss(4)
    with pytest.raises(RuntimeError, match="image_weights given, but the loss was built without sample_weights"):
        plain(x, y, image_weights=torch.ones(4))
    with pytest.raises(RuntimeError, match="text_weights given, but the loss was built without sample_weights"):
        SigLipLoss()(x, y, *sc, text_weights=torch.ones(4))
    mod = DDPSigmoidLoss(4, sample_weights=True)
    sl = SigLipLoss(sample_weights=True)
    hn = DDPSigmoidLoss(4, sample_weights=True, hard_negatives=3)
    neg = torch.randn(3, 8)
    for call in (lambda **kw: mod(x, y, **kw), lambda **kw: sl(x, y, *sc, **kw)):
        with pytest.raises(RuntimeError, match="image_weights must be a floating-point tensor"):
            call(image_weights=torch.ones(4, dtype=torch.int64))
        with pytest.raises(RuntimeError, match="text_weights must be a floating-point tensor"):
            call(text_weights=[1.0, 1.0, 1.0, 1.0])
        with pytest.raises(RuntimeError, match=r"image_weights must have shape \[4\]"):
            call(image_weights=torch.ones(5))
        with pytest.raises(RuntimeError, match=r"text_weights must have shape \[4\]"):
            call(text_weights=torch.ones(4, 1))
        with pytest.raises(RuntimeError, match="image_weights requires grad"):
            call(image_weights=torch.ones(4, requires_grad=True))
        # valid arguments (None = ones, any floating dtype) get as far as the device check (no CPU path)
        with pytest.raises(RuntimeError, match="no CPU path"):
            call(image_weights=torch.ones(4, dtype=torch.float64), text_weights=None)
    # with extras, text_weights covers the captions and then the extras
    with pytest.raises(RuntimeError, match=r"text_weights must have shape \[7\]"):
        hn(x, y, negative_text=neg, text_weights=torch.ones(4))
    with pytest.raises(RuntimeError, match="no CPU path"):
        hn(x, y, negative_text=neg, text_weights=torch.ones(7))
    if torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="image_weights is on"):
            mod(x.cuda(), y.cuda(), image_weights=torch.ones(4))
