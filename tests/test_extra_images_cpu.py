"""Extra images per rank without a GPU: the modules' argument checks (raised before any GPU work), self-checks of the
float64 oracle in tests/extra_images_oracle.py, and a model of how a metrics step publishes the extra images' ids
through the two step-parity key blocks."""
import random

import numpy as np
import pytest
import torch

from extra_images_oracle import closed_form_extras, dtxt_of, label_blocks, retrieval_metrics_extras
from retrieval_metrics_oracle import retrieval_metrics


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


@pytest.mark.parametrize("k", [-1, 1.5, True, "2"])
def test_extra_images_must_be_a_non_negative_int(k):
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    with pytest.raises(RuntimeError, match="extra_images"):
        DDPSigmoidLoss(8, extra_images=k)
    with pytest.raises(RuntimeError, match="extra_images"):
        SigLipLoss(extra_images=k)


def test_extra_image_checks_before_any_gpu_work():
    img, txt = torch.zeros(8, 16), torch.zeros(8, 16)
    for mod, sig in _mods(extra_images=3):
        with pytest.raises(RuntimeError, match=r"extra_images=3: forward needs extra_image"):
            _call(mod, sig, img, txt)
        with pytest.raises(RuntimeError, match=r"must have shape \[3, 16\]"):
            _call(mod, sig, img, txt, extra_image=torch.zeros(2, 16))
        with pytest.raises(RuntimeError, match="the images torch.float32"):
            _call(mod, sig, img, txt, extra_image=torch.zeros(3, 16, dtype=torch.bfloat16))
        with pytest.raises(RuntimeError, match="extra_image_ids given"):   # no ids without multi_positive
            _call(mod, sig, img, txt, extra_image=torch.zeros(3, 16), extra_image_ids=torch.arange(3))
    for mod, sig in _mods():
        with pytest.raises(RuntimeError, match="extra_image given"):
            _call(mod, sig, img, txt, extra_image=torch.zeros(3, 16))
    ids = torch.arange(8)
    for mod, sig in _mods(extra_images=3, multi_positive=True):
        with pytest.raises(RuntimeError, match="needs extra_image_ids"):
            _call(mod, sig, img, txt, sample_ids=ids, extra_image=torch.zeros(3, 16))
        with pytest.raises(RuntimeError, match=r"extra_image_ids must have shape \[3\]"):
            _call(mod, sig, img, txt, sample_ids=ids, extra_image=torch.zeros(3, 16), extra_image_ids=torch.arange(4))
        with pytest.raises(RuntimeError, match="integer tensor"):
            _call(mod, sig, img, txt, sample_ids=ids, extra_image=torch.zeros(3, 16),
                  extra_image_ids=torch.zeros(3))
    for mod, sig in _mods(extra_images=3, sample_weights=True):
        with pytest.raises(RuntimeError, match=r"image_weights must have shape \[11\]"):
            _call(mod, sig, img, txt, extra_image=torch.zeros(3, 16), image_weights=torch.ones(8))
    # everything valid: the CPU tensors are refused last, by the device check
    for mod, sig in _mods(extra_images=3, multi_positive=True, sample_weights=True):
        with pytest.raises(RuntimeError, match="CUDA"):
            _call(mod, sig, img, txt, sample_ids=ids, extra_image=torch.zeros(3, 16), extra_image_ids=torch.arange(3),
                  image_weights=torch.ones(11))


# ---------------------------------------------------------------------------------------------------------------------
# oracle self-checks
# ---------------------------------------------------------------------------------------------------------------------
def _blocks(Bs, Rs, Ts, D, seed):
    rng = np.random.default_rng(seed)
    n = lambda x: x / np.linalg.norm(x, axis=1, keepdims=True)  # noqa: E731
    return [n(rng.standard_normal((r, D))) for r in Rs], [n(rng.standard_normal((t, D))) for t in Ts]


def test_without_extras_it_is_the_plain_loss():
    from oracle.siglip_oracle import closed_form

    Bs = [6]
    imgs, txts = _blocks(Bs, Bs, Bs, 8, 0)
    got = closed_form_extras(imgs, txts, Bs, 1.3, -4.0)[0]
    ref = closed_form(imgs[0], txts[0], 1.3, -4.0, 1)[0]
    assert np.isclose(got["loss"], ref["loss"], rtol=1e-12)
    assert np.allclose(got["dimg"], ref["dimg"], rtol=1e-12)
    assert np.allclose(got["contrib"][0], ref["dtxt"], rtol=1e-12)


@pytest.mark.parametrize("mode", ["pos", "ids", "ids+ximg"])
def test_weight_zero_extras_equal_no_extras(mode):
    Bs, Es, Ts, D = [5, 7, 4], [3, 0, 6], [9, 7, 4], 12
    Rs = [b + e for b, e in zip(Bs, Es)]
    imgs, txts = _blocks(Bs, Rs, Ts, D, 1)
    rng = np.random.default_rng(2)
    ids = [rng.integers(0, 9, b) for b in Bs] if mode != "pos" else None
    xt = [rng.integers(0, 9, t - b) for b, t in zip(Bs, Ts)] if mode != "pos" else None
    xi = [rng.integers(0, 9, e) for e in Es] if "ximg" in mode else None
    wi = [np.concatenate([rng.random(b), np.zeros(e)]) for b, e in zip(Bs, Es)]
    wt = [rng.random(t) for t in Ts]
    a = closed_form_extras(imgs, txts, Bs, 0.7, -2.0, label_blocks(Bs, Rs, Ts, ids, xt, xi), wi, wt)
    b = closed_form_extras([x[:n] for x, n in zip(imgs, Bs)], txts, Bs, 0.7, -2.0,
                           label_blocks(Bs, Bs, Ts, ids, xt, None), [w[:n] for w, n in zip(wi, Bs)], wt)
    for r in range(len(Bs)):
        assert a[r]["loss"] == pytest.approx(b[r]["loss"], rel=1e-12)
        assert a[r]["dt_prime"] == pytest.approx(b[r]["dt_prime"], rel=1e-12)
        assert a[r]["dbias"] == pytest.approx(b[r]["dbias"], rel=1e-12)
        assert np.allclose(a[r]["dimg"][:Bs[r]], b[r]["dimg"], rtol=1e-12, atol=1e-15)
        assert not a[r]["dimg"][Bs[r]:].any()
        assert np.allclose(dtxt_of(a, r), dtxt_of(b, r), rtol=1e-12, atol=1e-15)


def test_duplicate_extra_image_adds_exactly_the_paired_row():
    """An extra image equal to paired image i, under i's id, adds exactly row i's terms to the loss, dt' and dbias,
    gets row i's gradient and doubles row i's contribution to every text gradient."""
    Bs, Ts, D = [5, 4], [5, 6], 10
    imgs, txts = _blocks(Bs, Bs, Ts, D, 3)
    ids = [np.array([0, 1, 2, 3, 4]), np.array([5, 6, 7, 8])]
    xt = [np.zeros(0, np.int64), np.array([2, 99])]
    i = 2
    base = closed_form_extras(imgs, txts, Bs, 1.0, -3.0, label_blocks(Bs, Bs, Ts, ids, xt, None))
    imgs2 = [np.concatenate([imgs[0], imgs[0][i:i + 1]]), imgs[1]]
    Rs = [6, 4]
    dup = closed_form_extras(imgs2, txts, Bs, 1.0, -3.0,
                             label_blocks(Bs, Rs, Ts, ids, xt, [np.array([ids[0][i]]), np.zeros(0, np.int64)]))
    # row i's own terms: the same closed form restricted to that one row
    row = closed_form_extras([imgs[0][i:i + 1], imgs[1][:0]], txts, [Bs[0], 1], 1.0, -3.0,
                             [[label_blocks(Bs, Bs, Ts, ids, xt, None)[0][c][i:i + 1] for c in range(2)],
                              [np.zeros((0, t)) for t in Ts]])[0]
    assert dup[0]["loss"] == pytest.approx(base[0]["loss"] + row["loss"], rel=1e-12)
    assert dup[0]["dt_prime"] == pytest.approx(base[0]["dt_prime"] + row["dt_prime"], rel=1e-12)
    assert dup[0]["dbias"] == pytest.approx(base[0]["dbias"] + row["dbias"], rel=1e-12)
    assert np.allclose(dup[0]["dimg"][5], dup[0]["dimg"][i], rtol=1e-12)
    assert np.allclose(dup[0]["dimg"][:5], base[0]["dimg"], rtol=1e-12)
    for c in range(2):
        assert np.allclose(dup[0]["contrib"][c], base[0]["contrib"][c] + row["contrib"][c], rtol=1e-12, atol=1e-15)


def test_labels_positional_diagonal_is_bounded_to_the_batch():
    y = label_blocks([3], [5], [6])[0][0]
    assert (y == 1).sum() == 3 and all(y[i, i] == 1 for i in range(3)) and y[3, 3] == -1 and y[4, 4] == -1


def test_labels_extra_images_match_no_id_without_their_own():
    ids, xt = [np.array([1, 2])], [np.array([1, 1])]
    y = label_blocks([2], [4], [4], ids, xt, None)[0][0]
    assert (y[2:] == -1).all()
    y = label_blocks([2], [4], [4], ids, xt, [np.array([1, 5])])[0][0]
    assert list(y[2]) == [1, -1, 1, 1] and (y[3] == -1).all()


def test_metrics_oracle_without_extras_is_the_retrieval_oracle():
    Bs = [4, 6]
    imgs, txts = _blocks(Bs, Bs, Bs, 8, 4)
    a = retrieval_metrics_extras(imgs, txts, Bs)
    b = retrieval_metrics(imgs, txts)
    for x, y in zip(a, b):
        assert np.array_equal(x["i2t_index"], y["i2t_index"]) and np.array_equal(x["t2i_index"], y["t2i_index"])
        assert x["i2t_top1"] == y["i2t_top1"] and x["t2i_top1"] == y["t2i_top1"]


def test_metrics_oracle_extra_image_rules():
    """Text 0's best image is an extra image: a miss without image ids, a hit with its id, a miss with another id;
    i2t covers the extras only with ids, and an extra whose id matches no text is an i2t miss."""
    D = 4
    img = np.eye(D)[:3].copy()           # images 0, 1 paired; image 2 extra, equal to text 0
    txt = np.array([[0, 0, 1, 0], [0, 1, 0, 0]], np.float64)
    img[0] = [0.5, 0, 0.5, 0]
    m = retrieval_metrics_extras([img], [txt], [2])[0]
    assert m["t2i_index"][0] == 2 and m["t2i_top1"] == 0.5 and len(m["i2t_index"]) == 2
    ids = [np.array([10, 11])]
    m = retrieval_metrics_extras([img], [txt], [2], ids, None, [np.array([10])])[0]
    assert m["t2i_top1"] == 1.0 and len(m["i2t_index"]) == 3
    m = retrieval_metrics_extras([img], [txt], [2], ids, None, [np.array([12])])[0]
    assert m["t2i_top1"] == 0.5 and m["i2t_top1"] == pytest.approx(2 / 3)


# ---------------------------------------------------------------------------------------------------------------------
# published extra-image ids: two step-parity blocks, written next to the key memset before the first loss kernel,
# read by the peers after flag kind 5
# ---------------------------------------------------------------------------------------------------------------------
def _run_protocol(W, steps, armed, nbuf, seed):
    """One random interleaving of W ranks (stream order per rank as the library issues it). Per step n:
    [metrics: zero my key block n % nbuf and copy my extra-image ids into it] -> wait flag2 of every peer >= n - 1 ->
    publish my text (flag0 = n) -> pull every peer's text (wait flag0 >= n) -> [metrics: loss kernels write my
    partials] -> flag2 = n -> [metrics finalize: flag5 = n to every rank, wait every flag5 >= n, read every peer's
    published ids of step n (begin / end)]. Returns the violations: a read of another step's ids or of ids rewritten
    while they were read."""
    rnd = random.Random(seed)
    flag0, flag2, flag5 = [0] * W, [0] * W, [0] * W
    xids = [[("none", 0, 0)] * nbuf for _ in range(W)]   # (state, step, version)
    version = [0]
    errors = []

    def _write(r, q, state, n):
        version[0] += 1
        xids[r][q] = (state, n, version[0])

    def _begin(p, q, seen):
        seen[p] = xids[p][q]

    def _end(r, p, q, n, seen):
        a, b = seen[p], xids[p][q]
        if a[0] != "ids" or a[1] != n:
            errors.append(f"rank {r} step {n}: read rank {p}'s ids of another step {a}")
        elif b != a:
            errors.append(f"rank {r} step {n}: rank {p}'s ids were rewritten during the read ({b})")

    def program(r):
        for n in range(1, steps + 1):
            q = n % nbuf
            if n in armed:
                yield ("act", lambda r=r, q=q, n=n: _write(r, q, "zeroing", n))
                yield ("act", lambda r=r, q=q, n=n: _write(r, q, "ids", n))
            yield ("wait", lambda n=n: all(flag2[p] >= n - 1 for p in range(W)))
            yield ("act", lambda r=r, n=n: flag0.__setitem__(r, n))
            for p in range(W):
                if p != r:
                    yield ("wait", lambda p=p, n=n: flag0[p] >= n)
            yield ("act", lambda r=r, n=n: flag2.__setitem__(r, n))
            if n in armed:
                yield ("act", lambda r=r, n=n: flag5.__setitem__(r, n))
                yield ("wait", lambda n=n: all(flag5[p] >= n for p in range(W)))
                seen = {}
                for p in range(W):
                    if p != r:
                        yield ("act", lambda p=p, q=q, seen=seen: _begin(p, q, seen))
                for p in range(W):
                    if p != r:
                        yield ("act", lambda p=p, q=q, n=n, seen=seen, r=r: _end(r, p, q, n, seen))

    progs = [program(r) for r in range(W)]
    pending = [next(g, None) for g in progs]
    while any(x is not None for x in pending):
        ready = [r for r in range(W) if pending[r] is not None and (pending[r][0] == "act" or pending[r][1]())]
        assert ready, "deadlock"
        r = rnd.choice(ready)
        if pending[r][0] == "act":
            pending[r][1]()
        pending[r] = next(progs[r], None)
    return errors


@pytest.mark.parametrize("W", [2, 3, 5, 8])
def test_parity_blocks_never_expose_stale_or_rewritten_ids(W):
    rnd = random.Random(100 + W)
    for trial in range(150):
        steps = 6
        armed = {n for n in range(1, steps + 1) if rnd.random() < 0.6}
        errs = _run_protocol(W, steps, armed, nbuf=2, seed=trial)
        assert not errs, errs[:3]


def test_single_block_fails():
    found = []
    for trial in range(400):
        found += _run_protocol(3, 4, {1, 2, 3, 4}, nbuf=1, seed=trial)
        if found:
            break
    assert found, "the single-block model should expose rewritten ids"
