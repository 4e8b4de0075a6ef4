"""CPU checks of excluded same-group pairs (exclude_groups=True): the float64 oracle against autograd of a direct torch
restatement and against the weighted oracle, and every argument check and refusal of the modules, which run before any
GPU work."""
import math

import numpy as np
import pytest
import torch

from exclude_groups_oracle import closed_form_groups, clustered, group_labels, pad_rows, torch_loss
from sample_weights_oracle import closed_form_weighted, label_blocks


def _problem(Bs, Ks, Es, D, seed, ids=False):
    rng = np.random.default_rng(seed)
    imgs = [rng.standard_normal((b + e, D)) / math.sqrt(D) * 3 for b, e in zip(Bs, Es)]
    txts = [rng.standard_normal((b + k, D)) / math.sqrt(D) * 3 for b, k in zip(Bs, Ks)]
    id_blocks = [rng.integers(0, max(Bs), b) for b in Bs] if ids else None
    labels = pad_rows(label_blocks(Bs, [b + k for b, k in zip(Bs, Ks)], id_blocks), [b + e for b, e in zip(Bs, Es)])
    ig = [rng.integers(-1, 4, b + e) for b, e in zip(Bs, Es)]
    tg = [rng.integers(-1, 4, b + k) for b, k in zip(Bs, Ks)]
    iw = [rng.random(b + e) for b, e in zip(Bs, Es)]
    tw = [rng.random(b + k) for b, k in zip(Bs, Ks)]
    return imgs, txts, labels, ig, tg, iw, tw


@pytest.mark.parametrize("ids", [False, True])
@pytest.mark.parametrize("Bs,Ks,Es", [([7], [0], [0]), ([5, 6, 4], [2, 0, 3], [1, 2, 0])])
def test_oracle_matches_autograd_of_the_restatement(Bs, Ks, Es, ids):
    imgs, txts, labels, ig, tg, iw, tw = _problem(Bs, Ks, Es, 9, seed=len(Bs) + ids, ids=ids)
    y = group_labels(labels, ig, tg)
    assert any((b == 0).any() for row in y for b in row)
    tp, b = 0.4, -0.7
    res = closed_form_groups(imgs, txts, tp, b, y, Bs, iw, tw)
    T = torch.cat([torch.tensor(t) for t in txts]).requires_grad_(True)
    cw = torch.cat([torch.tensor(w) for w in tw])
    dtxt = torch.zeros_like(T)
    for r, img in enumerate(imgs):
        xi = torch.tensor(img, requires_grad=True)
        xt = T.detach().clone().requires_grad_(True)
        tpt = torch.tensor(tp, dtype=torch.float64, requires_grad=True)
        bt = torch.tensor(b, dtype=torch.float64, requires_grad=True)
        loss = torch_loss(xi, xt, tpt, bt, torch.tensor(np.concatenate(y[r], axis=1)), torch.tensor(iw[r]), cw,
                          batch=Bs[r])
        loss.backward()
        assert float(loss.detach()) == pytest.approx(res[r]["loss"], rel=1e-12)
        np.testing.assert_allclose(xi.grad.numpy(), res[r]["dimg"], rtol=1e-10, atol=1e-13)
        np.testing.assert_allclose(xt.grad.numpy(), np.concatenate(res[r]["contrib"]), rtol=1e-10, atol=1e-13)
        assert float(tpt.grad) == pytest.approx(res[r]["dt_prime"], rel=1e-10, abs=1e-13)
        assert float(bt.grad) == pytest.approx(res[r]["dbias"], rel=1e-10, abs=1e-13)
        dtxt += xt.grad
        # per-sample sums: the row and column sums of the terms, without 1/B
        assert float(res[r]["image_loss"].sum()) == pytest.approx(res[r]["loss"] * Bs[r], rel=1e-12)
        assert float(sum(p.sum() for p in res[r]["text_part"])) == pytest.approx(res[r]["loss"] * Bs[r], rel=1e-12)


def test_without_excluded_pairs_it_is_the_weighted_oracle():
    Bs, Ks = [6, 5], [2, 1]
    imgs, txts, labels, _, _, iw, tw = _problem(Bs, Ks, [0, 0], 8, seed=3, ids=True)
    none = [np.full(b, -1) for b in Bs]
    y = group_labels(labels, none, [np.full(b + k, -1) for b, k in zip(Bs, Ks)])
    a = closed_form_groups(imgs, txts, 0.3, -1.0, y, Bs, iw, tw)
    b = closed_form_weighted(imgs, txts, 0.3, -1.0, iw, tw, labels)
    for x, z in zip(a, b):
        assert x["loss"] == pytest.approx(z["loss"], rel=1e-13)
        np.testing.assert_allclose(x["dimg"], z["dimg"], rtol=1e-12)


def test_positives_are_never_excluded_and_negative_groups_match_nothing():
    y = [[np.array([[1.0, -1.0, -1.0], [-1.0, 1.0, -1.0]])]]
    out = group_labels(y, [np.array([0, -1])], [np.array([0, 0, -1])])[0][0]
    assert out.tolist() == [[1.0, 0.0, -1.0], [-1.0, 1.0, -1.0]]


def test_clustered_embeddings_make_the_excluded_pairs_heavy():
    g = np.arange(40) % 5
    img, txt = clustered(g, 64, 5, 0, 1), clustered(g, 64, 5, 0, 2)
    s = img @ txt.T
    same = g[:, None] == g[None, :]
    assert s[same].mean() > 0.5 > 0.2 > abs(s[~same].mean())


# ---- argument checks and refusals (before any GPU work) -----------------------------------------------------------
def _mods():
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    return DDPSigmoidLoss, SigLipLoss


def test_exclude_groups_must_be_a_bool_and_refuses_distill():
    DDP, SL = _mods()
    for cls in (DDP, SL):
        args = (8,) if cls is DDP else ()
        with pytest.raises(RuntimeError, match="exclude_groups must be a bool"):
            cls(*args, exclude_groups=1)
        with pytest.raises(RuntimeError, match="cannot be combined with distill"):
            cls(*args, exclude_groups=True, distill=0.5)
        cls(*args, exclude_groups=True)


def _call(mod, img, txt, **kw):
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss

    if isinstance(mod, DDPSigmoidLoss):
        return mod(img, txt, **kw)
    return mod(img, txt, torch.tensor(2.3), torch.tensor(-10.0), **kw)


@pytest.mark.parametrize("which", ["ddp", "siglip"])
def test_group_arguments_are_checked_before_any_gpu_work(which):
    DDP, SL = _mods()
    B, D, K, E = 8, 16, 3, 2
    img, txt = torch.randn(B, D), torch.randn(B, D)
    gi, gt = torch.zeros(B, dtype=torch.int64), torch.zeros(B, dtype=torch.int64)
    plain = DDP(B) if which == "ddp" else SL()
    with pytest.raises(RuntimeError, match="image_groups given, but the loss was built without exclude_groups"):
        _call(plain, img, txt, image_groups=gi)
    with pytest.raises(RuntimeError, match="text_groups given, but the loss was built without exclude_groups"):
        _call(plain, img, txt, text_groups=gt)
    mod = DDP(B, exclude_groups=True) if which == "ddp" else SL(exclude_groups=True)
    with pytest.raises(RuntimeError, match=r"forward needs image_groups \(\[8\] integer tensor"):
        _call(mod, img, txt, text_groups=gt)
    with pytest.raises(RuntimeError, match=r"forward needs text_groups \(\[8\]"):
        _call(mod, img, txt, image_groups=gi)
    with pytest.raises(RuntimeError, match="image_groups must be an integer tensor"):
        _call(mod, img, txt, image_groups=gi.float(), text_groups=gt)
    with pytest.raises(RuntimeError, match=r"text_groups must have shape \[8\]"):
        _call(mod, img, txt, image_groups=gi, text_groups=gt[:5])
    # with extras the groups cover the paired samples, then the extras
    ext = DDP(B, exclude_groups=True, hard_negatives=K, extra_images=E) if which == "ddp" else \
        SL(exclude_groups=True, hard_negatives=K, extra_images=E)
    neg, xim = torch.randn(K, D), torch.randn(E, D)
    with pytest.raises(RuntimeError, match=r"image_groups must have shape \[10\]"):
        _call(ext, img, txt, negative_text=neg, extra_image=xim, image_groups=gi, text_groups=torch.zeros(B + K))
    with pytest.raises(RuntimeError, match=r"text_groups must have shape \[11\]"):
        _call(ext, img, txt, negative_text=neg, extra_image=xim, image_groups=torch.zeros(B + E, dtype=torch.int32),
              text_groups=gt)


def test_existing_refusals_are_unchanged():
    DDP, _ = _mods()
    with pytest.raises(RuntimeError, match="extra_texts=K needs multi_positive=True"):
        DDP(8, extra_texts=2, exclude_groups=True)
    with pytest.raises(RuntimeError, match="distill cannot be combined with hard_negatives"):
        DDP(8, hard_negatives=2, distill=0.5, exclude_groups=True)


def test_c_abi_declares_the_new_entries():
    import os

    from distributed_sigmoid_loss_b200 import _capi

    hdr = open(os.path.join(os.path.dirname(__file__), "..", "include", "siglip_b200.h")).read()
    assert "SIGLIP_OPT_EXCLUDE_GROUPS = 27" in hdr and _capi.SIGLIP_OPT_EXCLUDE_GROUPS == 27
    for sym in ("siglip_set_groups", "siglip_debug_set_chunk_groups"):
        assert sym in hdr and sym in _capi.EXPORTED_SYMBOLS
