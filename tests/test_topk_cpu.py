"""Top-K retrieval without a GPU: the float64 oracle in tests/retrieval_topk_oracle.py (sorted lists, lowest-index ties,
recall@k under positional labels, ids, extra texts and extra images), the model of the kernel's atomic insertion chain
under random interleavings (and a broken variant it must catch), the cross-rank merge, and the modules' argument checks
(raised before any GPU work)."""
import random

import numpy as np
import pytest
import torch

from retrieval_metrics_oracle import retrieval_metrics
from retrieval_topk_oracle import insert_chain, merge_lists, recall_counts, run_interleaved, topk_retrieval

import distributed_sigmoid_loss_b200 as pkg
from distributed_sigmoid_loss_b200.loss import TOPK_MAX, _topk_buffers, _validate_metrics_topk


def _unit(g, n, d):
    x = g.standard_normal((n, d))
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def test_oracle_sorted_with_lowest_index_ties():
    # one image, texts with repeated similarities: ties go to the lower global index
    img = [np.array([[1.0, 0.0]])]
    txt = [np.array([[0.5, 0.0], [1.0, 0.0], [0.5, 0.0], [1.0, 0.0], [0.2, 0.0]])]
    o = topk_retrieval(img, txt, [1], 5)[0]
    assert o["i2t_topk"].tolist() == [[1, 3, 0, 2, 4]]
    # fewer candidates than K: -1 tail
    o = topk_retrieval([np.eye(2)], [np.eye(2)], [2], 4)[0]
    assert o["i2t_topk"].tolist() == [[0, 1, -1, -1], [1, 0, -1, -1]]
    assert o["i2t_recall"].tolist() == [1.0, 1.0, 1.0, 1.0]


@pytest.mark.parametrize("Bs", [(6,), (5, 3, 7)])
def test_oracle_column_zero_and_recall_one_match_top1(Bs):
    g = np.random.default_rng(len(Bs))
    imgs = [_unit(g, b, 8) for b in Bs]
    txts = [_unit(g, b, 8) for b in Bs]
    ref = retrieval_metrics(imgs, txts)
    for k in (1, 3, 5):
        for r, o in enumerate(topk_retrieval(imgs, txts, Bs, k)):
            assert np.array_equal(o["i2t_topk"][:, 0], ref[r]["i2t_index"])
            assert np.array_equal(o["t2i_topk"][:, 0], ref[r]["t2i_index"])
            assert o["i2t_recall"][0] == ref[r]["i2t_top1"] and o["t2i_recall"][0] == ref[r]["t2i_top1"]
            assert np.all(np.diff(o["i2t_recall"]) >= 0) and np.all(np.diff(o["t2i_recall"]) >= 0)


def test_oracle_prefix_property():
    g = np.random.default_rng(3)
    Bs = (7, 4)
    imgs = [_unit(g, b, 6) for b in Bs]
    txts = [_unit(g, b, 6) for b in Bs]
    o5, o10 = topk_retrieval(imgs, txts, Bs, 5), topk_retrieval(imgs, txts, Bs, 10)
    for a, b in zip(o5, o10):
        assert np.array_equal(a["i2t_topk"], b["i2t_topk"][:, :5])
        assert np.array_equal(a["t2i_topk"], b["t2i_topk"][:, :5])
        assert np.array_equal(a["i2t_recall"], b["i2t_recall"][:5])


def test_oracle_recall_with_ids_extra_texts_and_images():
    # rank 0: 2 paired samples (ids 0, 1), extra texts with ids (1, 7), one extra image with id 0; rank 1: 1 sample (id 1)
    e = np.eye(4)
    imgs = [np.stack([e[0], e[1], e[2]]), np.stack([e[3]])]
    # texts of rank 0: caption 0 points away from image 0, its extra caption (id 1 text) at image 1, id 7 at image 0
    txts = [np.stack([0.1 * e[0] + e[3], e[1], e[1] * 0.9, e[0] * 0.95]), np.stack([e[3] * 0.5 + e[1] * 0.6])]
    img_ids = [np.array([0, 1, 0]), np.array([1])]
    txt_ids = [np.array([0, 1, 1, 7]), np.array([1])]
    out = topk_retrieval(imgs, txts, [2, 1], 3, img_ids, txt_ids, rank_all_images=True, rank_all_texts=True)
    o = out[0]
    # image 0 (id 0): best texts are 3 (id 7, miss), then 0 (id 0, hit)
    assert o["i2t_topk"][0, :2].tolist() == [3, 0]
    assert o["i2t_first"][0] == 1
    # the extra image 2 (id 0, ranked under rank_all_images) has no id-0 text near it: s = 0 ties, lowest index first
    assert o["i2t_topk"].shape == (3, 3)
    # text 3 (id 7) has no image with id 7: never a hit
    assert o["t2i_first"][3] == 3
    # text 1 (id 1): best image 1 (id 1): a hit at rank 0
    assert o["t2i_first"][1] == 0
    # without ids on the extras: the extra texts are never hits, the extra image neither
    out = topk_retrieval(imgs, txts, [2, 1], 3, [np.array([0, 1]), np.array([1])], [np.array([0, 1]), np.array([1])])
    assert out[0]["i2t_first"][0] == 1   # text 3 is no hit, text 0 is
    assert out[0]["i2t_topk"].shape == (2, 3) and out[0]["t2i_topk"].shape == (2, 3)


def test_recall_counts_are_fp32_divisions():
    first = np.array([0, 2, 5, 1, 0, 5, 3])
    r = recall_counts(first, 5)
    assert r.dtype == np.float32
    assert r[0] == np.float32(2) / np.float32(7) and r[4] == np.float32(5) / np.float32(7)


def _keys(rng, n):
    return rng.sample(range(1, 1 << 40), n)   # distinct non-zero keys


@pytest.mark.parametrize("k", [2, 5, 10])
def test_insertion_chain_is_exact_under_any_interleaving(k):
    rng = random.Random(k)
    for seed in range(300):
        keys = _keys(rng, rng.randint(1, 40))
        want = sorted(keys, reverse=True)[:k] + [0] * max(0, k - len(keys))
        assert run_interleaved(k, keys, seed) == want
        assert run_interleaved(k, keys, seed, prefilter=True) == want


def test_stopping_the_chain_at_a_rejecting_slot_is_caught():
    rng = random.Random(1)
    wrong = 0
    for seed in range(300):
        keys = _keys(rng, 30)
        want = sorted(keys, reverse=True)[:5]
        wrong += run_interleaved(5, keys, seed, stop_on_reject=True) != want
    assert wrong > 0


def test_chain_ends_on_an_empty_slot():
    gen = insert_chain(5, 9)
    assert gen.send(None) == (0, 9)
    with pytest.raises(StopIteration):
        gen.send(0)   # slot 0 was empty: the key stays there, the carried 0 ends the chain


def test_cross_rank_merge():
    rng = random.Random(7)
    for _ in range(200):
        W, k = rng.randint(1, 6), rng.randint(1, 10)
        keys = _keys(rng, rng.randint(0, 60))
        parts = [sorted(keys[q::W], reverse=True)[:k] for q in range(W)]
        lists = [p + [0] * (k - len(p)) for p in parts]
        want = sorted(keys, reverse=True)[:k]
        assert merge_lists(lists, k) == want + [0] * (k - len(want))


def test_topk_max_matches_the_header():
    import pathlib
    import re
    hdr = (pathlib.Path(pkg.__file__).resolve().parents[1] / "include" / "siglip_b200.h").read_text()
    assert int(re.search(r"#define SIGLIP_TOPK_MAX (\d+)", hdr).group(1)) == TOPK_MAX == 10


def test_metrics_topk_validation():
    assert _validate_metrics_topk(None, False, None) == 1
    assert _validate_metrics_topk(5, True, None) == 5
    for bad in (0, 11, -1, 2.0, True, "5"):
        with pytest.raises(RuntimeError, match="metrics_topk"):
            _validate_metrics_topk(bad, True, None)
    with pytest.raises(RuntimeError, match="return_metrics"):
        _validate_metrics_topk(5, False, None)
    with pytest.raises(RuntimeError, match="distill"):
        _validate_metrics_topk(5, True, 0.5)


def test_k1_keeps_todays_buffers():
    bufs = (torch.empty(2), torch.empty(3, dtype=torch.int64), torch.empty(3, dtype=torch.int64))
    assert _topk_buffers(None, 1, bufs) is bufs
    assert _topk_buffers(None, 5, None) is None


def test_modules_refuse_before_gpu_work():
    x = torch.randn(4, 8)
    with pytest.raises(RuntimeError, match="metrics_topk"):
        pkg.DDPSigmoidLoss(4)(x, x, return_metrics=True, metrics_topk=11)
    with pytest.raises(RuntimeError, match="return_metrics"):
        pkg.SigLipLoss()(x, x, torch.tensor(1.0), torch.tensor(0.0), metrics_topk=5)
