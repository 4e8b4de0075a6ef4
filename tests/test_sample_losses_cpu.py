"""Per-sample losses without a GPU: the float64 oracle in tests/sample_losses_oracle.py checked against float64 autograd
(the per-sample loss is B times the derivative of the rank's loss with respect to the sample's weight, at unit weights),
its sum identities, a model of the fixed-point encoding, and the modules' argument checks (raised before any GPU
work)."""
import math
import random

import numpy as np
import pytest
import torch

from extra_images_oracle import closed_form_extras, label_blocks
from sample_losses_oracle import MAX_PARTIAL, fixed_point_decode, fixed_point_partial, sample_losses


def _unit(g, n, d):
    x = g.standard_normal((n, d))
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def _problem(seed, Bs, Es, Ks, ids_mode):
    """Images [R_r = B_r + E_r], texts [T_r = B_r + K_r] and their labels: positional, sample ids, or sample ids with
    ids on the extra texts and extra images."""
    g = np.random.default_rng(seed)
    D = 12
    Rs = [b + e for b, e in zip(Bs, Es)]
    Ts = [b + k for b, k in zip(Bs, Ks)]
    imgs = [_unit(g, r, D) for r in Rs]
    txts = [_unit(g, t, D) for t in Ts]
    ids = xt = xi = None
    if ids_mode != "pos":
        ids = [g.integers(0, 6, b) for b in Bs]
    if ids_mode == "extras":
        xt = [g.integers(0, 9, k) for k in Ks]
        xi = [g.integers(0, 9, e) for e in Es]
    return g, imgs, txts, label_blocks(Bs, Rs, Ts, ids, xt, xi)


CASES = [((4, 4), (0, 0), (0, 0), "pos"),
         ((5, 3, 6), (0, 0, 0), (2, 0, 3), "pos"),        # hard negatives, T >= B
         ((5, 3, 6), (2, 1, 0), (0, 0, 0), "pos"),        # extra (hard-negative) images, R >= B
         ((5, 4), (0, 0), (0, 0), "ids"),
         ((5, 3, 4), (2, 0, 1), (1, 3, 0), "extras")]     # extra texts and extra images with ids


def _autograd(imgs, txts, labels, Bs, tp, bias):
    """float64 autograd of the weighted loss: d L_r / d a_r[i] and d L_r / d c_c[j] at unit weights."""
    t = math.exp(tp)
    a = [torch.ones(x.shape[0], dtype=torch.float64, requires_grad=True) for x in imgs]
    c = [torch.ones(x.shape[0], dtype=torch.float64, requires_grad=True) for x in txts]
    da = []
    dc = [torch.zeros(x.shape[0], dtype=torch.float64) for x in txts]
    for r, img in enumerate(imgs):
        L = 0.0
        for k, txt in enumerate(txts):
            z = t * torch.from_numpy(img) @ torch.from_numpy(txt).T + bias
            y = torch.from_numpy(labels[r][k])
            w = a[r][:, None] * c[k][None, :]
            L = L + (w * torch.nn.functional.softplus(-y * z)).sum() / Bs[r]
        grads = torch.autograd.grad(L, [a[r]] + c)
        da.append(grads[0] * Bs[r])
        for k in range(len(txts)):
            dc[k] += grads[1 + k] * Bs[r]
    return da, dc


@pytest.mark.parametrize("Bs,Es,Ks,mode", CASES)
def test_oracle_matches_autograd_at_unit_weights(Bs, Es, Ks, mode):
    tp, bias = math.log(10.0), -5.0
    _, imgs, txts, labels = _problem(sum(Bs) + 17 * sum(Ks) + 31 * sum(Es), Bs, Es, Ks, mode)
    got = sample_losses(imgs, txts, Bs, tp, bias, labels)
    da, dc = _autograd(imgs, txts, labels, Bs, tp, bias)
    for r in range(len(Bs)):
        np.testing.assert_allclose(got[r]["image_loss"], da[r].numpy(), rtol=1e-12, atol=0)
        np.testing.assert_allclose(got[r]["text_loss"], dc[r].numpy(), rtol=1e-12, atol=0)


@pytest.mark.parametrize("Bs,Es,Ks,mode", CASES)
def test_sum_identities_with_weights(Bs, Es, Ks, mode):
    """loss_r == image_loss_r.sum() / B_r (against closed_form_extras), the image and text sides carry the same total,
    and a sample whose weight is 0 reports exactly 0."""
    tp, bias = math.log(10.0), -4.0
    g, imgs, txts, labels = _problem(7 + sum(Bs), Bs, Es, Ks, mode)
    a = [np.where(g.random(x.shape[0]) < 0.25, 0.0, g.random(x.shape[0])) for x in imgs]
    cw = [np.where(g.random(x.shape[0]) < 0.25, 0.0, g.random(x.shape[0])) for x in txts]
    got = sample_losses(imgs, txts, Bs, tp, bias, labels, a, cw)
    ref = closed_form_extras(imgs, txts, Bs, tp, bias, labels, a, cw)
    for r in range(len(Bs)):
        assert abs(got[r]["loss"] - ref[r]["loss"]) <= 1e-12 * abs(ref[r]["loss"])
        assert not got[r]["image_loss"][a[r] == 0].any()
        assert not got[r]["text_loss"][cw[r] == 0].any()
    tot_i = sum(x["image_loss"].sum() for x in got)
    tot_t = sum(x["text_loss"].sum() for x in got)
    assert abs(tot_i - tot_t) <= 1e-12 * tot_i


def test_fixed_point_sums_do_not_depend_on_the_order():
    """Partials rounded once to 64-bit integers add up to the same bits in every order; the decoded value is the
    float64 sum within the 2^-32 quantum per partial."""
    g = np.random.default_rng(5)
    parts = np.float32(g.random(3000) * 40.0) * np.float32(g.random(3000) < 0.9)
    words = [fixed_point_partial(v)[0] for v in parts]
    want = fixed_point_decode(sum(words), 0)
    for seed in range(5):
        random.Random(seed).shuffle(words)
        acc = 0
        for w in words:
            acc = (acc + w) % (1 << 64)
        assert fixed_point_decode(acc, 0) == want
    assert abs(float(want) - float(parts.astype(np.float64).sum())) <= 1e-6 * float(want)


def test_fixed_point_poison():
    """A partial that is not finite or too large poisons its sample instead of wrapping into a finite number."""
    assert fixed_point_partial(MAX_PARTIAL) == (0, 1)
    assert fixed_point_partial(np.inf) == (0, 1)
    assert fixed_point_partial(np.nan) == (0, 2)
    assert fixed_point_partial(0.0) == (0, 0)
    w, p = fixed_point_partial(MAX_PARTIAL * 0.999)
    assert p == 0 and w < (1 << 48)
    assert np.isinf(fixed_point_decode(5, 1)) and np.isnan(fixed_point_decode(5, 3))
    # the largest total of 2^16 partials just below the limit still fits in 64 bits
    assert ((1 << 16) * int(MAX_PARTIAL * 2 ** 32)) <= (1 << 64)


# ---------------------------------------------------------------------------------------------------------------------
# module arguments
# ---------------------------------------------------------------------------------------------------------------------
def _mods(**kw):
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    return [(DDPSigmoidLoss(8, **kw), False), (SigLipLoss(**kw), True)]


def _call(mod, siglip, img, txt, **kw):
    if siglip:
        return mod(img, txt, torch.zeros(()), torch.zeros(()), **kw)
    return mod(img, txt, **kw)


@pytest.mark.parametrize("metrics", [False, True])
@pytest.mark.parametrize("flag", [1, "yes", None])
def test_flag_must_be_a_bool(flag, metrics):
    img, txt = torch.zeros(8, 16), torch.zeros(8, 16)
    for mod, sig in _mods():
        with pytest.raises(RuntimeError, match="return_sample_losses must be a bool"):
            _call(mod, sig, img, txt, return_metrics=metrics, return_sample_losses=flag)


@pytest.mark.parametrize("metrics", [False, True])
def test_distillation_is_refused_before_any_gpu_work(metrics):
    img, txt = torch.zeros(8, 16), torch.zeros(8, 16)
    for mod, sig in _mods(distill=0.5):
        with pytest.raises(RuntimeError, match="return_sample_losses is unavailable with distill"):
            _call(mod, sig, img, txt, return_metrics=metrics, return_sample_losses=True)


@pytest.mark.parametrize("metrics", [False, True])
def test_valid_flag_reaches_the_cpu_tensor_check(metrics):
    """With a valid flag the call goes on to the usual checks: CPU tensors are refused as before."""
    img, txt = torch.zeros(8, 16), torch.zeros(8, 16)
    for mod, sig in _mods():
        with pytest.raises(RuntimeError, match="CUDA"):
            _call(mod, sig, img, txt, return_metrics=metrics, return_sample_losses=True)


def test_outputs_come_in_the_documented_order():
    from distributed_sigmoid_loss_b200.loss import _with_outputs

    m = (torch.zeros(2), torch.zeros(3, dtype=torch.int64), torch.ones(3, dtype=torch.int64))
    l = (torch.full((4,), 2.0), torch.full((5,), 3.0))
    assert _with_outputs("loss", None, None) == "loss"
    out = _with_outputs("loss", None, l)
    assert out[0] == "loss" and set(out[1]) == {"image_loss", "text_loss"} and out[1]["text_loss"].shape == (5,)
    out = _with_outputs("loss", m, l)
    assert len(out) == 3 and "i2t_top1" in out[1] and out[2]["image_loss"].shape == (4,)
    out = _with_outputs("loss", m, None)
    assert len(out) == 2 and "t2i_index" in out[1]
