"""CPU checks of the in-batch retrieval metrics: the float64 oracle against brute force, the kernels' argmax key packing,
a model of the cross-rank exchange of the column partials (flag kind 5 + step-parity buffers), and the modules'
argument errors."""
import random

import numpy as np
import pytest
import torch

from retrieval_metrics_oracle import hits, key_index, metric_key, retrieval_metrics


# ---------------------------------------------------------------------------------------------------------------------
# oracle vs brute force
# ---------------------------------------------------------------------------------------------------------------------
def _brute(imgs, txts, ids):
    I = [row for x in imgs for row in np.asarray(x, np.float64)]
    T = [row for x in txts for row in np.asarray(x, np.float64)]
    gid = [int(v) for x in ids for v in x] if ids is not None else list(range(len(I)))
    i2t, t2i = [], []
    for i in range(len(I)):
        best, bj = None, None
        for j in range(len(T)):
            s = float(np.dot(I[i], T[j]))
            if best is None or s > best:
                best, bj = s, j
        i2t.append(bj)
    for j in range(len(T)):
        best, bi = None, None
        for i in range(len(I)):
            s = float(np.dot(I[i], T[j]))
            if best is None or s > best:
                best, bi = s, i
        t2i.append(bi)
    return i2t, t2i, gid


@pytest.mark.parametrize("Bs,with_ids", [([7], False), ([5, 3, 6], False), ([4, 4], True), ([6, 2, 5], True)])
def test_oracle_matches_brute_force(Bs, with_ids):
    rng = np.random.default_rng(sum(Bs))
    D = 5
    # small integers: many exact ties, which must go to the lowest global index
    imgs = [rng.integers(-2, 3, size=(b, D)).astype(np.float64) for b in Bs]
    txts = [rng.integers(-2, 3, size=(b, D)).astype(np.float64) for b in Bs]
    ids = [rng.integers(0, 4, size=b) for b in Bs] if with_ids else None
    res = retrieval_metrics(imgs, txts, ids)
    i2t, t2i, gid = _brute(imgs, txts, ids)
    gid = np.asarray(gid)
    off = np.concatenate([[0], np.cumsum(Bs)])
    for r, b in enumerate(Bs):
        assert list(res[r]["i2t_index"]) == i2t[off[r]:off[r + 1]]
        assert list(res[r]["t2i_index"]) == t2i[off[r]:off[r + 1]]
        assert res[r]["i2t_top1"] == pytest.approx(hits(i2t[off[r]:off[r + 1]], gid, off[r]).mean())
        assert res[r]["t2i_top1"] == pytest.approx(hits(t2i[off[r]:off[r + 1]], gid, off[r]).mean())


def test_oracle_ids_count_off_diagonal_duplicates():
    img = np.eye(3)
    txt = np.array([[0, 1, 0], [1, 0, 0], [0, 0, 1]], np.float64)   # image 0's best text is text 1 and vice versa
    pos = retrieval_metrics([img], [txt])[0]
    assert pos["i2t_top1"] == pytest.approx(1 / 3)
    same = retrieval_metrics([img], [txt], [np.array([7, 7, 9])])[0]
    assert same["i2t_top1"] == 1.0 and same["t2i_top1"] == 1.0


# ---------------------------------------------------------------------------------------------------------------------
# key packing
# ---------------------------------------------------------------------------------------------------------------------
def _interesting_floats(rng, n):
    specials = [0.0, -0.0, 1e-45, -1e-45, 1e-40, -1e-40, 1.17549435e-38, -1.17549435e-38, 1.0, -1.0, 3.4e38, -3.4e38,
                np.inf, -np.inf]
    vals = list(rng.standard_normal(n).astype(np.float32)) + [np.float32(v) for v in specials]
    vals += list((rng.standard_normal(n) * 1e-39).astype(np.float32))   # subnormals of both signs
    return vals


def test_key_is_monotone_in_s():
    rng = np.random.default_rng(0)
    vals = sorted(set(float(v) for v in _interesting_floats(rng, 300)))
    keys = [metric_key(v, 5) for v in vals]
    assert all(a < b for a, b in zip(keys, keys[1:])), "key order must follow the float order"
    assert all(k > 0 for k in keys), "0 is reserved for 'no candidate'"


def test_key_ties_go_to_the_lowest_index():
    rng = np.random.default_rng(1)
    for v in _interesting_floats(rng, 50):
        assert metric_key(v, 3) > metric_key(v, 4) > metric_key(v, 1 << 31)
        assert key_index(metric_key(v, 12345)) == 12345
    # +0 and -0 are equal values: the index decides
    assert metric_key(-0.0, 1) > metric_key(0.0, 2)
    assert metric_key(0.0, 1) > metric_key(-0.0, 2)


def test_key_max_is_argmax_with_lowest_index():
    rng = np.random.default_rng(2)
    for _ in range(200):
        n = int(rng.integers(1, 40))
        s = rng.choice(np.array(_interesting_floats(rng, 5), np.float32), size=n)
        s = s[~np.isnan(s)]
        if len(s) == 0:
            continue
        best = max(metric_key(v, i) for i, v in enumerate(s))
        s0 = np.where(s == 0, np.float32(0), s)   # -0 == +0
        assert key_index(best) == int(np.argmax(s0))


# ---------------------------------------------------------------------------------------------------------------------
# exchange model: flag kind 5 + parity buffers, random interleavings
# ---------------------------------------------------------------------------------------------------------------------
def _run_protocol(W, steps, armed, nbuf, seed):
    """One random interleaving of W ranks running `steps` forwards (stream order per rank, as issued by the library).
    Per step n: [metrics: zero my key buffer n % nbuf] -> wait flag2 of every peer >= n-1 -> publish my text (flag0 = n)
    -> pull every peer's text (wait flag0 >= n) -> [metrics: loss kernels write my partials] -> flag2 = n ->
    [metrics finalize: flag5 = n to every rank, wait every flag5 >= n, read every peer's buffer (begin / end)].
    Returns a list of violations (a read that saw a partial of another step or a buffer written while it was read)."""
    rnd = random.Random(seed)
    flag0 = [0] * W
    flag2 = [0] * W
    flag5 = [0] * W
    buf = [[("none", 0, 0)] * nbuf for _ in range(W)]   # (state, step, version)
    version = [0]
    errors = []

    def program(r):
        for n in range(1, steps + 1):
            q = n % nbuf
            if n in armed:
                yield ("act", lambda r=r, q=q, n=n: _write(r, q, "zero", n))
            yield ("wait", lambda n=n: all(flag2[p] >= n - 1 for p in range(W)))
            yield ("act", lambda r=r, n=n: flag0.__setitem__(r, n))
            for p in range(W):
                if p != r:
                    yield ("wait", lambda p=p, n=n: flag0[p] >= n)
            if n in armed:
                yield ("act", lambda r=r, q=q, n=n: _write(r, q, "writing", n))
                yield ("act", lambda r=r, q=q, n=n: _write(r, q, "done", n))
            yield ("act", lambda r=r, n=n: flag2.__setitem__(r, n))
            if n in armed:
                yield ("act", lambda r=r, n=n: flag5.__setitem__(r, n))
                yield ("wait", lambda n=n: all(flag5[p] >= n for p in range(W)))
                seen = {}
                for p in range(W):
                    if p != r:
                        yield ("act", lambda p=p, q=q, n=n, seen=seen: _begin(p, q, n, seen))
                for p in range(W):
                    if p != r:
                        yield ("act", lambda p=p, q=q, n=n, seen=seen, r=r: _end(r, p, q, n, seen))

    def _write(r, q, state, n):
        version[0] += 1
        buf[r][q] = (state, n, version[0])

    def _begin(p, q, n, seen):
        seen[p] = buf[p][q]

    def _end(r, p, q, n, seen):
        a, b = seen[p], buf[p][q]
        if a[0] != "done" or a[1] != n:
            errors.append(f"rank {r} step {n}: stale read of rank {p}'s partials {a}")
        elif b != a:
            errors.append(f"rank {r} step {n}: rank {p}'s partials were overwritten during the read ({b})")

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
def test_parity_buffers_never_expose_a_stale_or_torn_partial(W):
    rnd = random.Random(W)
    for trial in range(150):
        steps = 6
        armed = {n for n in range(1, steps + 1) if rnd.random() < 0.6}
        errs = _run_protocol(W, steps, armed, nbuf=2, seed=trial)
        assert not errs, errs[:3]


def test_single_buffer_fails():
    found = []
    for trial in range(400):
        found += _run_protocol(3, 4, {1, 2, 3, 4}, nbuf=1, seed=trial)
        if found:
            break
    assert found, "the single-buffer model should expose an overwritten partial"


# ---------------------------------------------------------------------------------------------------------------------
# module argument errors (raised before any GPU work)
# ---------------------------------------------------------------------------------------------------------------------
def test_return_metrics_must_be_bool():
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    x = torch.zeros(4, 8)
    with pytest.raises(RuntimeError, match="return_metrics must be a bool"):
        DDPSigmoidLoss(4)(x, x, return_metrics=1)
    with pytest.raises(RuntimeError, match="return_metrics must be a bool"):
        SigLipLoss()(x, x, torch.ones(()), torch.zeros(()), return_metrics="yes")


def test_return_metrics_keeps_the_other_argument_errors():
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss

    x = torch.zeros(4, 8)
    with pytest.raises(RuntimeError, match="gpu_batch_size"):
        DDPSigmoidLoss(5)(x, x, return_metrics=True)
    with pytest.raises(RuntimeError, match="no CPU path"):
        DDPSigmoidLoss(4)(x, x, return_metrics=True)
    with pytest.raises(RuntimeError, match="sample_ids given"):
        DDPSigmoidLoss(4)(x, x, sample_ids=torch.arange(4), return_metrics=True)
