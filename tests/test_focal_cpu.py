"""CPU checks of the focal pair loss (focal_gamma / focal_alpha): the float64 oracle against torchvision's
sigmoid_focal_loss, against float64 autograd and against the SigLIP oracles at gamma = 0; the |g| bound that keeps every
pair derivative inside the fp16 sigma operand; and every argument check of the modules, which run before any GPU work."""
import math
import os

import numpy as np
import pytest
import torch

from exclude_groups_oracle import closed_form_groups, group_labels
from extra_images_oracle import label_blocks
from focal_oracle import closed_form_focal, focal_terms, g_bound, torch_focal_loss, torch_focal_terms
from label_sets_oracle import set_labels

GAMMAS = (0.0, 0.5, 2.0, 5.0)
ALPHAS = (None, 0.25)


def _blocks(Rs, Ts, D, seed, scale=3.0):
    rng = np.random.default_rng(seed)
    imgs = [rng.standard_normal((r, D)) / math.sqrt(D) * scale for r in Rs]
    txts = [rng.standard_normal((t, D)) / math.sqrt(D) * scale for t in Ts]
    return imgs, txts


@pytest.mark.parametrize("gamma", GAMMAS + (8.0,))
@pytest.mark.parametrize("alpha", ALPHAS + (0.0, 1.0))
def test_terms_are_torchvision_sigmoid_focal_loss(gamma, alpha):
    ops = pytest.importorskip("torchvision.ops")
    z = np.concatenate([np.linspace(-30.0, 30.0, 601), [-80.0, 80.0]])
    for y in (-1.0, 1.0):
        term, _ = focal_terms(z, np.full_like(z, y), gamma, alpha)
        tgt = torch.full((len(z),), (y + 1) / 2, dtype=torch.float64)
        want = ops.sigmoid_focal_loss(torch.tensor(z), tgt, alpha=-1 if alpha is None else alpha, gamma=gamma,
                                      reduction="none").numpy()
        # torchvision forms the cross-entropy as (1 - t) z + log(1 + exp(-z)): absolute error ~1e-15 on tiny terms
        np.testing.assert_allclose(term, want, rtol=1e-9, atol=1e-14)


@pytest.mark.parametrize("gamma", GAMMAS + (8.0,))
@pytest.mark.parametrize("alpha", ALPHAS)
def test_closed_form_g_is_autograd_of_the_terms(gamma, alpha):
    z = np.linspace(-25.0, 25.0, 501)
    for y in (-1.0, 1.0):
        # one image per z and the identity as texts: z_ii = t s_ii + b with t = 1, b = 0, s_ii = z
        zt = torch.tensor(z, requires_grad=True)
        y_mat = torch.full((len(z), len(z)), 0.0, dtype=torch.float64)
        y_mat.diagonal().fill_(y)
        loss = torch_focal_terms(torch.diag(zt), torch.eye(len(z), dtype=torch.float64),
                                 torch.tensor(0.0, dtype=torch.float64), 0.0, y_mat, gamma, alpha).diagonal()
        loss.sum().backward()
        term, g = focal_terms(z, np.full_like(z, y), gamma, alpha)
        # torch's softplus returns x itself above 20: up to gamma e^-20 < 2e-8 relative
        np.testing.assert_allclose(term, loss.detach().numpy(), rtol=5e-8, atol=1e-300)
        np.testing.assert_allclose(g, zt.grad.numpy(), rtol=5e-8, atol=1e-300)


@pytest.mark.parametrize("gamma,alpha", [(0.5, None), (2.0, 0.25), (5.0, None)])
def test_closed_form_matches_autograd_with_every_label_rule(gamma, alpha):
    """Label sets, ids of extras, weights and excluded groups composed: the oracle's loss, gradients, dt' and dbias are
    float64 autograd of the torch restatement on the dense labels."""
    Bs, Es, Ks, D = [6, 5], [1, 2], [2, 1], 8
    Rs = [b + e for b, e in zip(Bs, Es)]
    Ts = [b + k for b, k in zip(Bs, Ks)]
    rng = np.random.default_rng(3)
    imgs, txts = _blocks(Rs, Ts, D, 4)
    iw = [rng.random(r) for r in Rs]
    tw = [rng.random(t) for t in Ts]
    isets = [rng.integers(-1, 4, (r, 2)) for r in Rs]
    tsets = [rng.integers(-1, 4, (t, 2)) for t in Ts]
    ig = [rng.integers(-1, 3, r) for r in Rs]
    tg = [rng.integers(-1, 3, t) for t in Ts]
    lab = group_labels(set_labels(isets, tsets, Bs), ig, tg)
    assert any((y == 0).any() for row in lab for y in row) and sum((y > 0).sum() for row in lab for y in row) > sum(Bs)
    tp, b = 0.4, -1.1
    res = closed_form_focal(imgs, txts, tp, b, lab, gamma, alpha, Bs, iw, tw)
    T = torch.cat([torch.tensor(t) for t in txts])
    cw = torch.cat([torch.tensor(w) for w in tw])
    for r, img in enumerate(imgs):
        y = torch.tensor(np.concatenate(lab[r], axis=1))
        xi = torch.tensor(img, requires_grad=True)
        xt = T.detach().clone().requires_grad_(True)
        tpt = torch.tensor(tp, dtype=torch.float64, requires_grad=True)
        bt = torch.tensor(b, dtype=torch.float64, requires_grad=True)
        loss = torch_focal_loss(xi, xt, tpt, bt, y, gamma, alpha, torch.tensor(iw[r]), cw, batch=Bs[r])
        loss.backward()
        assert float(loss.detach()) == pytest.approx(res[r]["loss"], rel=1e-12)
        np.testing.assert_allclose(xi.grad.numpy(), res[r]["dimg"], rtol=1e-9, atol=1e-13)
        np.testing.assert_allclose(xt.grad.numpy(), np.concatenate(res[r]["contrib"]), rtol=1e-9, atol=1e-13)
        assert float(tpt.grad) == pytest.approx(res[r]["dt_prime"], rel=1e-9, abs=1e-13)
        assert float(bt.grad) == pytest.approx(res[r]["dbias"], rel=1e-9, abs=1e-13)


def test_gamma_zero_without_alpha_is_the_siglip_oracle():
    Bs, Es, Ks, D = [5, 7, 4], [2, 0, 1], [1, 3, 0], 8
    Rs = [b + e for b, e in zip(Bs, Es)]
    Ts = [b + k for b, k in zip(Bs, Ks)]
    imgs, txts = _blocks(Rs, Ts, D, 9)
    rng = np.random.default_rng(2)
    ids = [rng.integers(0, 3, b) for b in Bs]
    xt = [rng.integers(0, 3, k) for k in Ks]
    lab = group_labels(label_blocks(Bs, Rs, Ts, ids, xt), [rng.integers(-1, 2, r) for r in Rs],
                       [rng.integers(-1, 2, t) for t in Ts])
    iw = [rng.random(r) for r in Rs]
    tw = [rng.random(t) for t in Ts]
    a = closed_form_focal(imgs, txts, 0.2, -2.0, lab, 0.0, None, Bs, iw, tw)
    b = closed_form_groups(imgs, txts, 0.2, -2.0, lab, Bs, iw, tw)
    for x, z in zip(a, b):
        assert x["loss"] == pytest.approx(z["loss"], rel=1e-13)
        np.testing.assert_allclose(x["dimg"], z["dimg"], rtol=1e-12, atol=1e-15)
        np.testing.assert_allclose(x["image_loss"], z["image_loss"], rtol=1e-12, atol=1e-15)
        for c in range(len(Bs)):
            np.testing.assert_allclose(x["contrib"][c], z["contrib"][c], rtol=1e-12, atol=1e-15)
            np.testing.assert_allclose(x["text_part"][c], z["text_part"][c], rtol=1e-12, atol=1e-15)
        assert x["dt_prime"] == pytest.approx(z["dt_prime"], rel=1e-12)
        assert x["dbias"] == pytest.approx(z["dbias"], rel=1e-12)


@pytest.mark.parametrize("gamma", GAMMAS)
@pytest.mark.parametrize("alpha", ALPHAS + (1.0,))
def test_terms_are_nonnegative_and_excluded_pairs_are_zero(gamma, alpha):
    z = np.linspace(-40.0, 40.0, 801)
    for y in (-1.0, 1.0, 0.0):
        term, g = focal_terms(z, np.full_like(z, y), gamma, alpha)
        assert (term >= 0).all()
        if y == 0:
            assert (term == 0).all() and (g == 0).all()
        elif y < 0:
            assert (g >= 0).all()
        else:
            assert (g <= 0).all()


def test_g_bound_fits_the_fp16_operand_over_the_accepted_gammas():
    bounds = [g_bound(gm) for gm in np.linspace(0.0, 8.0, 33)]
    assert max(bounds) < 1.44
    assert max(bounds) * 2.0 ** 14 < 65504.0   # g * 2^14 is stored as fp16
    # the bound grows with gamma: 8 is where the accepted range ends
    assert bounds[-1] == max(bounds)


# ---- argument checks and refusals (before any GPU work) -----------------------------------------------------------
def _mods():
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    return DDPSigmoidLoss, SigLipLoss


@pytest.mark.parametrize("which", ["ddp", "siglip"])
def test_focal_arguments_are_checked_before_any_gpu_work(which):
    DDP, SL = _mods()
    cls = DDP if which == "ddp" else SL
    args = (8,) if which == "ddp" else ()
    for bad in (-0.5, 8.5, float("nan"), float("inf"), True, "2", [2.0]):
        with pytest.raises(RuntimeError, match="focal_gamma must be None or a number in"):
            cls(*args, focal_gamma=bad)
    for bad in (-0.1, 1.5, float("nan"), False, "0.25"):
        with pytest.raises(RuntimeError, match="focal_alpha must be None or a number in"):
            cls(*args, focal_gamma=2.0, focal_alpha=bad)
    with pytest.raises(RuntimeError, match="focal_alpha given, but the loss was built without focal_gamma"):
        cls(*args, focal_alpha=0.25)
    with pytest.raises(RuntimeError, match="focal_gamma cannot be combined with distill"):
        cls(*args, focal_gamma=2.0, distill=0.5)
    with pytest.raises(RuntimeError, match="focal_gamma cannot be combined with distill"):
        cls(*args, focal_gamma=0.0, focal_alpha=0.25, distill=1.0)
    assert cls(*args).focal is None
    assert cls(*args, focal_gamma=2).focal == (2.0, None)
    assert cls(*args, focal_gamma=0.0, focal_alpha=1).focal == (0.0, 1.0)
    assert cls(*args, focal_gamma=8.0, focal_alpha=0.0).focal == (8.0, 0.0)
    # every other option composes
    cls(*args, focal_gamma=2.0, focal_alpha=0.25, multi_label=2, extra_texts=3, extra_images=2, exclude_groups=True,
        sample_weights=True, sigma_budget_bytes=1 << 20)
    cls(*args, focal_gamma=2.0, multi_positive=True, extra_texts=2)
    cls(*args, focal_gamma=2.0, hard_negatives=3)


def test_existing_distill_refusals_are_unchanged_without_focal():
    DDP, _ = _mods()
    with pytest.raises(RuntimeError, match="multi_label cannot be combined with distill"):
        DDP(8, multi_label=1, distill=0.5)
    with pytest.raises(RuntimeError, match="exclude_groups cannot be combined with distill"):
        DDP(8, exclude_groups=True, distill=0.5)


def test_c_abi_declares_the_new_entries():
    from distributed_sigmoid_loss_b200 import _capi

    hdr = open(os.path.join(os.path.dirname(__file__), "..", "include", "siglip_b200.h")).read()
    assert "SIGLIP_OPT_FOCAL = 29" in hdr and _capi.SIGLIP_OPT_FOCAL == 29
    assert "int siglip_set_focal(siglip_ctx* ctx, float gamma, float alpha);" in hdr
    assert "siglip_set_focal" in _capi.EXPORTED_SYMBOLS
