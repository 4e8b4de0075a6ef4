"""CPU checks of multi-label positives (multi_label=M): the float64 oracle against the sample-id oracle, the positional
labels and float64 autograd of a dense label matrix, the retrieval variant, and every argument check and refusal of the
modules, which run before any GPU work."""
import math

import numpy as np
import pytest
import torch

from exclude_groups_oracle import torch_loss
from label_sets_oracle import closed_form_sets, dense_labels, hierarchy_sets, meet, set_labels, topk_retrieval_sets
from retrieval_topk_oracle import topk_retrieval
from sample_ids_oracle import closed_form_ids


def _blocks(Rs, Ts, D, seed):
    rng = np.random.default_rng(seed)
    imgs = [rng.standard_normal((r, D)) / math.sqrt(D) * 3 for r in Rs]
    txts = [rng.standard_normal((t, D)) / math.sqrt(D) * 3 for t in Ts]
    return imgs, txts


def test_meet_ignores_empty_slots_and_duplicates():
    a = np.array([[3, -1], [-1, -1], [5, 5]])
    b = np.array([[-1, 3], [-1, -1], [5, -2]])
    assert meet(a, b).tolist() == [[True, False, False], [False, False, False], [False, False, True]]


def test_m1_nonnegative_labels_are_the_sample_id_oracle():
    Bs, D = [6, 5, 7], 8
    imgs, txts = _blocks(Bs, Bs, D, 1)
    ids = [np.random.default_rng(10 + r).integers(0, 4, b) for r, b in enumerate(Bs)]
    sets = [x[:, None] for x in ids]
    a = closed_form_sets(imgs, txts, 0.3, -1.2, sets, sets, Bs)
    b = closed_form_ids(imgs, txts, ids, 0.3, -1.2)
    for x, z in zip(a, b):
        assert x["loss"] == pytest.approx(z["loss"], rel=1e-13)
        np.testing.assert_allclose(x["dimg"], z["dimg"], rtol=1e-12, atol=1e-15)
        for c in range(len(Bs)):
            np.testing.assert_allclose(x["contrib"][c], z["contrib"][c], rtol=1e-12, atol=1e-15)
        assert x["dt_prime"] == pytest.approx(z["dt_prime"], rel=1e-12)
        assert x["dbias"] == pytest.approx(z["dbias"], rel=1e-12)


def test_empty_sets_give_the_positional_labels():
    Bs, Es, Ks = [5, 4], [2, 0], [1, 3]
    Rs = [b + e for b, e in zip(Bs, Es)]
    Ts = [b + k for b, k in zip(Bs, Ks)]
    y = set_labels([np.full((r, 3), -1) for r in Rs], [np.full((t, 3), -7) for t in Ts], Bs)
    for r in range(2):
        for c in range(2):
            want = -np.ones((Rs[r], Ts[c]))
            if r == c:
                want[np.arange(Bs[r]), np.arange(Bs[r])] = 1.0
            assert (y[r][c] == want).all()


def test_padding_and_duplicates_do_not_change_the_labels():
    si = np.array([[4], [7], [-1]])
    st = np.array([[7], [4], [9]])
    pad_i = np.array([[4, -1, 4, -5], [-1, 7, 7, -1], [-1, -1, -1, -1]])
    pad_t = np.array([[7, 7, -1, -1], [-3, 4, -1, 4], [9, -1, 9, 9]])
    assert (set_labels([si], [st], [3])[0][0] == set_labels([pad_i], [pad_t], [3])[0][0]).all()


def test_two_level_hierarchy_matches_autograd_of_the_dense_labels():
    # leaves 10 (golden retriever), 11 (poodle) under 1 (dog); 20 (tabby) under 2 (cat)
    parents = {10: 1, 11: 1, 20: 2}
    Bs, Ks, Es, D = [6, 5], [2, 1], [1, 2], 8
    rng = np.random.default_rng(7)
    leaves = [rng.choice([10, 11, 20], b) for b in Bs]
    sample = [hierarchy_sets(x, parents, 2) for x in leaves]
    # extra texts are class prompts ({dog}, {golden retriever}, ...): one label each
    xt = [np.array([[1, -1], [10, -1]])[:k] for k in Ks]
    xi = [hierarchy_sets(rng.choice([10, 11, 20], e), parents, 2) for e in Es]
    isets = [np.concatenate([s, x]) for s, x in zip(sample, xi)]
    tsets = [np.concatenate([s, x]) for s, x in zip(sample, xt)]
    Rs = [b + e for b, e in zip(Bs, Es)]
    Ts = [b + k for b, k in zip(Bs, Ks)]
    imgs, txts = _blocks(Rs, Ts, D, 8)
    iw = [rng.random(r) for r in Rs]
    tw = [rng.random(t) for t in Ts]
    ig = [rng.integers(-1, 3, r) for r in Rs]
    tg = [rng.integers(-1, 3, t) for t in Ts]
    Y = dense_labels(isets, tsets, Bs)
    # a poodle image is a positive for the {dog} prompt and a negative for {golden retriever}
    toff = np.cumsum([0] + Ts)
    for r in range(2):
        for i in range(Bs[r]):
            if leaves[r][i] == 11 and Ks[0] >= 2:
                gi = sum(Rs[:r]) + i
                assert Y[gi, toff[0] + Bs[0]] == 1 and Y[gi, toff[0] + Bs[0] + 1] == -1
    assert (Y > 0).sum() > sum(Bs)
    tp, b = 0.35, -0.8
    for groups in (False, True):
        res = closed_form_sets(imgs, txts, tp, b, isets, tsets, Bs, iw, tw, ig if groups else None,
                               tg if groups else None)
        y = torch.tensor(Y)
        if groups:
            gsame = (np.concatenate(ig)[:, None] == np.concatenate(tg)[None, :]) & (np.concatenate(ig)[:, None] >= 0)
            y = torch.where(torch.tensor(gsame) & (y < 0), torch.zeros_like(y), y)
        T = torch.cat([torch.tensor(t) for t in txts])
        cw = torch.cat([torch.tensor(w) for w in tw])
        r0 = 0
        for r, img in enumerate(imgs):
            xi_ = torch.tensor(img, requires_grad=True)
            xt_ = T.detach().clone().requires_grad_(True)
            tpt = torch.tensor(tp, dtype=torch.float64, requires_grad=True)
            bt = torch.tensor(b, dtype=torch.float64, requires_grad=True)
            loss = torch_loss(xi_, xt_, tpt, bt, y[r0:r0 + Rs[r]], torch.tensor(iw[r]), cw, batch=Bs[r])
            loss.backward()
            r0 += Rs[r]
            assert float(loss.detach()) == pytest.approx(res[r]["loss"], rel=1e-12)
            np.testing.assert_allclose(xi_.grad.numpy(), res[r]["dimg"], rtol=1e-10, atol=1e-13)
            np.testing.assert_allclose(xt_.grad.numpy(), np.concatenate(res[r]["contrib"]), rtol=1e-10, atol=1e-13)
            assert float(tpt.grad) == pytest.approx(res[r]["dt_prime"], rel=1e-10, abs=1e-13)
            assert float(bt.grad) == pytest.approx(res[r]["dbias"], rel=1e-10, abs=1e-13)


def test_retrieval_variant_with_m1_sets_is_the_id_rule():
    Bs, D, k = [6, 5], 8, 3
    imgs, txts = _blocks(Bs, Bs, D, 3)
    ids = [np.random.default_rng(20 + r).integers(0, 3, b) for r, b in enumerate(Bs)]
    a = topk_retrieval_sets(imgs, txts, Bs, k, [x[:, None] for x in ids], [x[:, None] for x in ids])
    b = topk_retrieval(imgs, txts, Bs, k, ids, ids)
    for x, z in zip(a, b):
        for key in ("i2t_topk", "t2i_topk", "i2t_first", "t2i_first", "i2t_recall", "t2i_recall"):
            np.testing.assert_array_equal(x[key], z[key])


def test_retrieval_variant_with_empty_sets_is_the_positional_rule():
    Bs, D, k = [5, 4], 8, 2
    imgs, txts = _blocks(Bs, Bs, D, 4)
    e = [np.full((b, 2), -1) for b in Bs]
    a = topk_retrieval_sets(imgs, txts, Bs, k, e, e)
    b = topk_retrieval(imgs, txts, Bs, k)
    for x, z in zip(a, b):
        np.testing.assert_array_equal(x["i2t_first"], z["i2t_first"])
        np.testing.assert_array_equal(x["t2i_first"], z["t2i_first"])


# ---- argument checks and refusals (before any GPU work) -----------------------------------------------------------
def _mods():
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    return DDPSigmoidLoss, SigLipLoss


def _call(mod, img, txt, **kw):
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss

    if isinstance(mod, DDPSigmoidLoss):
        return mod(img, txt, **kw)
    return mod(img, txt, torch.tensor(2.3), torch.tensor(-10.0), **kw)


def test_multi_label_values_and_refusals():
    DDP, SL = _mods()
    for cls in (DDP, SL):
        args = (8,) if cls is DDP else ()
        for bad in (True, 5, -1, 2.0, "2"):
            with pytest.raises(RuntimeError, match="multi_label must be None or an int in 1 .. 4"):
                cls(*args, multi_label=bad)
        with pytest.raises(RuntimeError, match="multi_label cannot be combined with multi_positive"):
            cls(*args, multi_label=2, multi_positive=True)
        with pytest.raises(RuntimeError, match="multi_label cannot be combined with distill"):
            cls(*args, multi_label=1, distill=0.5)
        for m in (1, 2, 4):
            assert cls(*args, multi_label=m).multi_label == m
        assert cls(*args, multi_label=None).multi_label == 0
        # extras carry label sets under multi_label, as they carry ids under multi_positive
        cls(*args, multi_label=2, extra_texts=3, extra_images=2, exclude_groups=True, sample_weights=True)
        cls(*args, multi_label=2, hard_negatives=3)


def test_existing_refusals_are_unchanged_without_multi_label():
    DDP, SL = _mods()
    with pytest.raises(RuntimeError, match="extra_texts=K needs multi_positive=True"):
        DDP(8, extra_texts=2)
    with pytest.raises(RuntimeError, match="extra_texts=K needs multi_positive=True"):
        SL(extra_texts=2)
    with pytest.raises(RuntimeError, match="distill cannot be combined with hard_negatives"):
        DDP(8, hard_negatives=2, distill=0.5)
    with pytest.raises(RuntimeError, match="extra_texts and hard_negatives cannot be combined"):
        DDP(8, multi_label=1, extra_texts=2, hard_negatives=1)


@pytest.mark.parametrize("which", ["ddp", "siglip"])
def test_label_arguments_are_checked_before_any_gpu_work(which):
    DDP, SL = _mods()
    B, D, K, E, M = 8, 16, 3, 2, 2
    img, txt = torch.randn(B, D), torch.randn(B, D)
    sl = torch.zeros(B, M, dtype=torch.int64)
    plain = DDP(B) if which == "ddp" else SL()
    for name in ("sample_labels", "extra_text_labels", "extra_image_labels"):
        with pytest.raises(RuntimeError, match=f"{name} given, but the loss was built without multi_label=M"):
            _call(plain, img, txt, **{name: sl})
    mod = DDP(B, multi_label=M) if which == "ddp" else SL(multi_label=M)
    with pytest.raises(RuntimeError, match=r"forward needs sample_labels \(\[8, 2\] integer tensor"):
        _call(mod, img, txt)
    with pytest.raises(RuntimeError, match="sample_labels must be an integer tensor"):
        _call(mod, img, txt, sample_labels=sl.float())
    with pytest.raises(RuntimeError, match=r"sample_labels must have shape \[8, 2\]"):
        _call(mod, img, txt, sample_labels=sl[:, :1])
    with pytest.raises(RuntimeError, match=r"sample_labels must have shape \[8, 2\]"):
        _call(mod, img, txt, sample_labels=sl[:5])
    with pytest.raises(RuntimeError, match="extra_text_labels given, but the loss was built without extra_texts"):
        _call(mod, img, txt, sample_labels=sl, extra_text_labels=sl[:K])
    with pytest.raises(RuntimeError, match="extra_image_labels given, but the loss was built without extra_images"):
        _call(mod, img, txt, sample_labels=sl, extra_image_labels=sl[:E])
    with pytest.raises(RuntimeError, match="sample_ids given, but the loss was built without multi_positive"):
        _call(mod, img, txt, sample_labels=sl, sample_ids=torch.zeros(B, dtype=torch.int64))
    ext = DDP(B, multi_label=M, extra_texts=K, extra_images=E) if which == "ddp" else \
        SL(multi_label=M, extra_texts=K, extra_images=E)
    xt, xi = torch.randn(K, D), torch.randn(E, D)
    with pytest.raises(RuntimeError, match=r"forward needs extra_text_labels \(\[3, 2\]"):
        _call(ext, img, txt, extra_text=xt, extra_image=xi, sample_labels=sl, extra_image_labels=sl[:E])
    with pytest.raises(RuntimeError, match=r"forward needs extra_image_labels \(\[2, 2\]"):
        _call(ext, img, txt, extra_text=xt, extra_image=xi, sample_labels=sl, extra_text_labels=sl[:K])
    with pytest.raises(RuntimeError, match=r"extra_text_labels must have shape \[3, 2\]"):
        _call(ext, img, txt, extra_text=xt, extra_image=xi, sample_labels=sl, extra_text_labels=sl[:2],
              extra_image_labels=sl[:E])
    with pytest.raises(RuntimeError, match="extra_text_ids given"):
        _call(ext, img, txt, extra_text=xt, extra_image=xi, sample_labels=sl, extra_text_labels=sl[:K],
              extra_image_labels=sl[:E], extra_text_ids=torch.zeros(K, dtype=torch.int64))
    with pytest.raises(RuntimeError, match="extra_image_ids given"):
        _call(ext, img, txt, extra_text=xt, extra_image=xi, sample_labels=sl, extra_text_labels=sl[:K],
              extra_image_labels=sl[:E], extra_image_ids=torch.zeros(E, dtype=torch.int64))
    hn = DDP(B, multi_label=M, hard_negatives=K) if which == "ddp" else SL(multi_label=M, hard_negatives=K)
    with pytest.raises(RuntimeError, match="extra_text_labels given, but the loss was built without extra_texts"):
        _call(hn, img, txt, negative_text=xt, sample_labels=sl, extra_text_labels=sl[:K])


def test_c_abi_declares_the_new_entries():
    import os

    from distributed_sigmoid_loss_b200 import _capi
    from distributed_sigmoid_loss_b200.loss import MAX_LABELS

    hdr = open(os.path.join(os.path.dirname(__file__), "..", "include", "siglip_b200.h")).read()
    assert "SIGLIP_OPT_LABEL_SETS = 28" in hdr and _capi.SIGLIP_OPT_LABEL_SETS == 28
    assert "#define SIGLIP_MAX_LABELS 4" in hdr and _capi.SIGLIP_MAX_LABELS == MAX_LABELS == 4
    for sym in ("siglip_ctx_create_labels", "siglip_set_label_sets", "siglip_debug_set_chunk_label_sets",
                "siglip_debug_set_peer_extra_image_label_sets"):
        assert sym in hdr and sym in _capi.EXPORTED_SYMBOLS
