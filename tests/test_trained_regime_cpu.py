"""The trained-regime generator and helpers (tests/trained_regime.py), on the CPU: every configuration that
tests/test_gpu_trained_regime.py runs is in the regime it claims, the own-diagonal split adds up to the oracle, the
stationary bias zeroes sum G, and the cold regime of the rest of the suite leaves the negatives under 1 % of dimg."""
import math

import numpy as np
import pytest
import torch

from sample_weights_oracle import closed_form_weighted, label_blocks
from trained_regime import (REGIMES, SIGMA_NORMAL_MIN, cold_batch, logit_stats, make_batch, negative_share,
                            pair_terms, random_weights, slab_fast_fraction, split_own_diagonal, stationary_bias)

# (Bs, Ks, D, mode): the shapes of the GPU file (its 1000 x 264 single-rank cases, its loopback cases, and the large
# batch of the trained and t300 regimes)
SINGLE = [((1000,), (136 if m in ("hn", "extra") else 0,), 264, m) for m in ("pos", "ids", "hn", "extra")]
LOOPBACK = [((160, 96, 130), (0, 0, 0), 264, "pos"), ((160, 96, 130), (40, 0, 200), 264, "extra"),
            ((128, 128, 128, 128), (0, 0, 0, 0), 264, "ids"), ((128, 128, 128, 128), (16, 300, 5, 64), 264, "hn")]


def _labels(Bs, Ks, ids, eids, mode):
    Ts = [b + k for b, k in zip(Bs, Ks)]
    f = (lambda xs: None if xs is None else [x.numpy() for x in xs])  # noqa: E731
    return label_blocks(list(Bs), Ts, f(ids), f(eids) if mode == "extra" else None)


def _bias(R, imgs, texts, labels):
    return stationary_bias(imgs, texts, R.t_prime, labels=labels) if R.bias is None else R.bias


def _assert_regime(R, imgs, texts, labels, bias):
    fast, n = slab_fast_fraction(imgs, texts, R.t_prime, bias, labels)
    st = logit_stats(imgs, texts, R.t_prime, bias, labels)
    # slabs of both paths in every configuration
    assert n >= 200 and 0.2 <= fast <= 0.8, f"{R.name}: {fast:.2f} of {n} slabs take the series path"
    # a tail of negatives above z = 0, up to where sigma * 2^14 is within 1 % of 16384
    assert st["neg_above_0"] > 1e-4 and st["neg_max"] > 5.0, st
    if R.bias is not None:
        # positives spread over the regime's range
        lo, hi = R.pos_z
        assert lo - 8 <= st["pos_q05"] <= lo + 6 and hi - 6 <= st["pos_q95"] <= hi + 8, st
        assert st["pos_max"] > hi, st
    else:
        # the stationary bias moves every logit: positives on both sides of 0 and far above it
        assert st["pos_q05"] < 0.0 and st["pos_q95"] > 15.0, st
    # a large share of the negatives below the fp16-normal sigma (z < -19.4), most of them in the separated batch
    assert st["neg_subnormal"] > (0.8 if R.name == "separated" else 0.3), st


@pytest.mark.parametrize("Bs,Ks,D,mode", SINGLE + LOOPBACK)
@pytest.mark.parametrize("regime", list(REGIMES))
def test_generator_meets_the_regime_targets(regime, Bs, Ks, D, mode):
    R = REGIMES[regime]
    # seeds as the GPU file draws them
    seed = 11 + ["pos", "ids", "hn", "extra"].index(mode) if len(Bs) == 1 else sum(Bs) + sum(Ks)
    imgs, texts, ids, eids = make_batch(R, Bs, Ks, D, seed, mode)
    for x in imgs + texts:
        assert x.dtype == torch.bfloat16
        assert torch.allclose(x.double().norm(dim=1), torch.ones(x.shape[0], dtype=torch.float64), atol=4e-3)
    labels = _labels(Bs, Ks, ids, eids, mode)
    _assert_regime(R, imgs, texts, labels, _bias(R, imgs, texts, labels))


@pytest.mark.parametrize("regime", ["trained", "t300"])
def test_generator_meets_the_regime_targets_at_the_large_batch(regime):
    R = REGIMES[regime]
    imgs, texts, _, _ = make_batch(R, (4096,), (0,), 768, 4096, "pos")
    _assert_regime(R, imgs, texts, None, R.bias)


@pytest.mark.parametrize("regime", ["trained", "t300"])
def test_fp32_rows_of_the_module_tests_are_in_the_regime(regime):
    R = REGIMES[regime]
    imgs, texts, _, _ = make_batch(R, (1000,), (0,), 264, 31, "pos", dtype=torch.float32)
    assert imgs[0].dtype == torch.float32
    _assert_regime(R, imgs, texts, None, R.bias)


def test_generator_is_deterministic_and_ids_follow_the_twins():
    R = REGIMES["trained"]
    a = make_batch(R, (160, 96), (40, 0), 136, 5, "extra")
    b = make_batch(R, (160, 96), (40, 0), 136, 5, "extra")
    for xs, ys in zip(a, b):
        for x, y in zip(xs, ys):
            assert torch.equal(x, y)
    imgs, texts, ids, eids = a
    allids = torch.cat(ids)
    assert len(torch.unique(allids)) < len(allids)                       # duplicated ids: the twins
    assert len(eids[0]) == 40 and len(eids[1]) == 0
    assert bool(torch.isin(eids[0], allids).any()) and not bool(torch.isin(eids[0], allids).all())


def _random_problem(W=2, weighted=True, mode="extra"):
    R = REGIMES["trained"]
    Bs, Ks = (96, 64)[:W], (24, 8)[:W]
    imgs, texts, ids, eids = make_batch(R, Bs, Ks, 72, 9, mode)
    g = torch.Generator().manual_seed(9)
    iws = [random_weights(g, b) for b in Bs] if weighted else None
    tws = [random_weights(g, b + k) for b, k in zip(Bs, Ks)] if weighted else None
    return R, imgs, texts, iws, tws, _labels(Bs, Ks, ids, eids, mode)


@pytest.mark.parametrize("W,weighted,mode", [(1, False, "pos"), (2, True, "extra"), (2, False, "ids")])
def test_own_diagonal_split_adds_up_to_the_oracle(W, weighted, mode):
    R, imgs, texts, iws, tws, labels = _random_problem(W, weighted, mode)
    d = (lambda xs: None if xs is None else [x.double().numpy() for x in xs])  # noqa: E731
    ref = closed_form_weighted(d(imgs), d(texts), R.t_prime, R.bias, d(iws), d(tws), labels)
    parts = split_own_diagonal(imgs, texts, R.t_prime, R.bias, iws, tws, labels)
    for r, (x, p) in enumerate(zip(ref, parts)):
        np.testing.assert_allclose(p["diag_dimg"] + p["rest_dimg"], x["dimg"], rtol=0, atol=1e-13 * abs(x["dimg"]).max())
        np.testing.assert_allclose(p["diag_contrib"] + p["rest_contrib"], x["contrib"][r], rtol=0,
                                   atol=1e-13 * abs(x["contrib"][r]).max())
        # the diagonal part is the positional diagonal only: rows of the own chunk's paired texts
        B = imgs[r].shape[0]
        assert not p["diag_contrib"][B:].any()
        assert np.abs(p["rest_dimg"]).max() > 0.05 * np.abs(x["dimg"]).max()


def test_pair_terms_match_the_oracle_scalars():
    R, imgs, texts, iws, tws, labels = _random_problem()
    d = (lambda xs: [x.double().numpy() for x in xs])  # noqa: E731
    ref = closed_form_weighted(d(imgs), d(texts), R.t_prime, R.bias, d(iws), d(tws), labels)
    t = math.exp(R.t_prime)
    for r, row in enumerate(pair_terms(imgs, texts, R.t_prime, R.bias, iws, tws, labels)):
        assert math.isclose(sum(x["G"].sum() for x in row), ref[r]["dbias"], rel_tol=1e-12, abs_tol=1e-300)
        assert math.isclose(t * sum((x["G"] * x["s"]).sum() for x in row), ref[r]["dt_prime"], rel_tol=1e-12)


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("regime", ["stationary", "trained", "separated"])
def test_stationary_bias_zeroes_the_bias_gradient(regime, weighted):
    R = REGIMES[regime]
    imgs, texts, ids, eids = make_batch(R, (300, 200), (0, 50), 136, 3, "ids")
    labels = _labels((300, 200), (0, 50), ids, eids, "ids")
    g = torch.Generator().manual_seed(4)
    iws = [random_weights(g, b) for b in (300, 200)] if weighted else None
    tws = [random_weights(g, t) for t in (300, 250)] if weighted else None
    b = stationary_bias(imgs, texts, R.t_prime, iws, tws, labels)
    terms = pair_terms(imgs, texts, R.t_prime, b, iws, tws, labels)
    total = sum(float(x["G"].sum()) for row in terms for x in row)
    scale = sum(float(np.abs(x["G"]).sum()) for row in terms for x in row)
    assert abs(total) <= 1e-12 * scale, (b, total, scale)
    assert scale > 1e-6      # the sums do not vanish: negatives and positives both carry weight


def test_cold_regime_hides_the_negatives():
    """t = 10, b = -10 with independent random unit embeddings (the rest of the suite): the part of dimg that passes
    through the sigma operand is under 1 % of its norm, so a 1e-3 check of dimg says little about it."""
    for Bs, Ks, D, mode in [((1000,), (0,), 136, "pos"), ((300,), (0,), 136, "pos"), ((1000,), (136,), 264, "pos")]:
        imgs, texts, ids, eids = cold_batch(Bs, Ks, D, 1, mode)
        share = negative_share(imgs, texts, math.log(10.0), -10.0, labels=_labels(Bs, Ks, ids, eids, mode))
        assert share < 0.01, (Bs, mode, share)
    R = REGIMES["trained"]
    imgs, texts, _, _ = make_batch(R, (1000,), (0,), 264, 11, "pos")
    assert negative_share(imgs, texts, R.t_prime, R.bias) > 0.5      # and the trained regime does not


def test_sigma_normal_bound_is_the_fp16_scale():
    """sigma * 2^14 is below fp16's smallest normal (2^-14) exactly when sigma < 2^-28 = 3.7e-9, z < -19.4."""
    assert SIGMA_NORMAL_MIN * 2.0 ** 14 == float(np.finfo(np.float16).tiny)
    assert abs(math.log(SIGMA_NORMAL_MIN / (1 - SIGMA_NORMAL_MIN)) + 19.4) < 0.05
