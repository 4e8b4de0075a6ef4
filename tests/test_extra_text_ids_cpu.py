"""CPU checks of extra texts with ids (several captions per image): the float64 oracle against autograd of the
reference's op sequence with the id label matrix, against the hard-negatives oracle when no extra id matches an image,
against the sample-ids oracle on repeated images, the metrics oracle, and the modules' argument errors (raised before
any GPU work)."""
import math

import numpy as np
import pytest
import torch

from extra_text_ids_oracle import closed_form_extra_text_ids, retrieval_metrics_extra_text_ids
from hard_negatives_oracle import closed_form_hard_negatives
from sample_ids_oracle import closed_form_ids


def _blocks(Bs, Ks, D, seed):
    g = np.random.default_rng(seed)

    def unit(n):
        x = g.standard_normal((n, D))
        return x / np.linalg.norm(x, axis=1, keepdims=True)
    return [unit(b) for b in Bs], [unit(b) for b in Bs], [unit(k) for k in Ks]


def _autograd(imgs, txts, extras, ids, extra_ids, tp, bias):
    """Per rank: logits against every chunk [txt_c; extras_c] -> labels (+1 iff the image's id equals the text's id,
    the text's id being its sample id or its extra id) -> -logsigmoid -> sum / B_r, as distributed_sigmoid_loss.py:22-47.
    Each rank's loss is differentiated on its own, so contrib[c] is that rank's share of chunk c's text gradient."""
    I = [torch.tensor(x, requires_grad=True) for x in imgs]
    C = [torch.tensor(np.concatenate([t, e]), requires_grad=True) for t, e in zip(txts, extras)]
    tid = [torch.tensor(np.concatenate([np.asarray(i), np.asarray(e, np.int64)])) for i, e in zip(ids, extra_ids)]
    out = []
    for r in range(len(I)):
        t_p = torch.tensor(tp, dtype=torch.float64, requires_grad=True)
        b_ = torch.tensor(bias, dtype=torch.float64, requires_grad=True)
        rid = torch.tensor(np.asarray(ids[r]))
        total = 0
        for c in range(len(C)):
            logits = I[r] @ C[c].T * t_p.exp() + b_
            labels = torch.where(rid[:, None] == tid[c][None, :], 1.0, -1.0).double()
            total = total + (-torch.nn.functional.logsigmoid(labels * logits)).sum()
        total = total / I[r].shape[0]
        contrib = torch.autograd.grad(total, [I[r], t_p, b_] + C)
        out.append(dict(loss=float(total), dimg=contrib[0].numpy(), dt_prime=float(contrib[1]),
                        dbias=float(contrib[2]), contrib=[x.numpy() for x in contrib[3:]]))
    return out


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


@pytest.mark.parametrize("Bs,Ks", [((5,), (3,)), ((6, 4, 7), (2, 0, 5)), ((8, 8), (8, 8))])
def test_oracle_matches_autograd_of_the_reference_op_sequence(Bs, Ks):
    """Extras that caption images of their own rank, of other ranks, and extras that match nothing."""
    tp, bias = math.log(10.0), -4.0
    imgs, txts, extras = _blocks(Bs, Ks, 24, sum(Bs) + sum(Ks))
    g = np.random.default_rng(len(Bs))
    ids = list(np.split(np.arange(sum(Bs)) * 3, np.cumsum(Bs)[:-1]))
    all_ids = np.concatenate(ids)
    # each extra: the id of a random image of the global batch, or an id no image has (1 + 3n is never a multiple of 3)
    extra_ids = [np.where(g.random(k) < 0.7, g.choice(all_ids, k), 1 + 3 * g.integers(0, 50, k)) for k in Ks]
    ref = _autograd(imgs, txts, extras, ids, extra_ids, tp, bias)
    _compare(closed_form_extra_text_ids(imgs, txts, extras, ids, extra_ids, tp, bias), ref)
    if len(Bs) > 1:
        assert any(np.isin(extra_ids[c], ids[r]).any() for c in range(len(Bs)) for r in range(len(Bs)) if r != c)


def test_unmatched_extras_are_the_hard_negatives_oracle():
    tp, bias = math.log(10.0), -7.0
    Bs, Ks = (7, 3, 5), (4, 0, 6)
    imgs, txts, extras = _blocks(Bs, Ks, 32, 3)
    ids = [np.array([0, 1, 1, 2, 3, 4, 5]), np.array([1, 6, 7]), np.array([8, 8, 0, 9, 10])]
    extra_ids = [np.array([100, 101, 100, 102]), np.zeros(0, np.int64), -np.arange(1, 7)]
    _compare(closed_form_extra_text_ids(imgs, txts, extras, ids, extra_ids, tp, bias),
             closed_form_hard_negatives(imgs, txts, extras, tp, bias, ids))


@pytest.mark.parametrize("Bs,M", [((6,), 4), ((5, 3), 3)])
def test_several_captions_equal_repeated_images(Bs, M):
    """B images with M captions each (caption 0 paired, captions 1..M-1 as extras, in caption-major order) equal the
    sample-ids oracle on M·B repeated image rows, each paired with one caption: loss, dt', dbias and dtxt are equal, and
    each image's dimg is the sum over its copies. Same labels, same logits; only the float64 summation order differs."""
    tp, bias = math.log(10.0), -5.0
    D = 16
    g = np.random.default_rng(sum(Bs) * M)
    unit = lambda n: (lambda x: x / np.linalg.norm(x, axis=1, keepdims=True))(g.standard_normal((n, D)))  # noqa: E731
    imgs = [unit(b) for b in Bs]
    caps = [[unit(b) for _ in range(M)] for b in Bs]                    # caps[r][m]: caption m of rank r's images
    ids = list(np.split(np.arange(sum(Bs)) + 10, np.cumsum(Bs)[:-1]))
    got = closed_form_extra_text_ids(imgs, [c[0] for c in caps], [np.concatenate(c[1:]) for c in caps], ids,
                                     [np.tile(i, M - 1) for i in ids], tp, bias)
    ref = closed_form_ids([np.tile(x, (M, 1)) for x in imgs], [np.concatenate(c) for c in caps],
                          [np.tile(i, M) for i in ids], tp, bias)
    for r, b in enumerate(Bs):
        for k in ("loss", "dt_prime", "dbias"):
            _close(got[r][k], ref[r][k], 1e-12)
        _close(got[r]["dimg"], ref[r]["dimg"].reshape(M, b, D).sum(0), 1e-12)
        for c in range(len(Bs)):
            _close(got[r]["contrib"][c], ref[r]["contrib"][c], 1e-12)


def test_metrics_oracle_extra_caption_is_a_hit_and_pure_negative_a_miss():
    D = 8
    imgs = [np.eye(D)[:3], np.eye(D)[3:5]]
    txts = [np.eye(D)[:3] * 0.5, np.eye(D)[3:5] * 0.5]
    # rank 0: extra 0 is a closer caption of image 1 (id 11), extra 1 a pure negative closest to image 2
    extras = [np.stack([np.eye(D)[1], np.eye(D)[2] * 0.9]), np.eye(D)[[0]] * 0.8]
    ids = [np.array([10, 11, 12]), np.array([13, 14])]
    extra_ids = [np.array([11, 99]), np.array([10])]       # rank 1's extra captions rank 0's image 0
    m = retrieval_metrics_extra_text_ids(imgs, txts, extras, ids, extra_ids)
    assert list(m[0]["i2t_index"]) == [7, 3, 4]             # texts: 0..2 paired, 3..4 rank 0's extras, rank 1 from 5
    assert m[0]["i2t_top1"] == pytest.approx(2 / 3)         # image 0 -> rank 1's extra (id 10): hit; image 2 -> miss
    assert list(m[0]["t2i_index"]) == [0, 1, 2, 1, 2]       # t2i over all T_0 = 5 texts
    assert m[0]["t2i_top1"] == pytest.approx(4 / 5)         # the pure negative (id 99) is the miss
    assert list(m[1]["i2t_index"]) == [5, 6] and m[1]["i2t_top1"] == 1.0
    assert list(m[1]["t2i_index"]) == [3, 4, 0] and m[1]["t2i_top1"] == 1.0


def test_module_argument_errors_are_raised_without_a_gpu():
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    x, y = torch.randn(4, 8), torch.randn(4, 8)
    ids, e, eid = torch.arange(4), torch.randn(3, 8), torch.tensor([0, 1, 7])
    for bad in (-1, 1.5, True, "2"):
        with pytest.raises(RuntimeError, match="extra_texts must be an int"):
            DDPSigmoidLoss(4, multi_positive=True, extra_texts=bad)
        with pytest.raises(RuntimeError, match="extra_texts must be an int"):
            SigLipLoss(multi_positive=True, extra_texts=bad)
    for ctor in (lambda **kw: DDPSigmoidLoss(4, **kw), lambda **kw: SigLipLoss(**kw)):
        with pytest.raises(RuntimeError, match="needs multi_positive=True"):
            ctor(extra_texts=3)
        with pytest.raises(RuntimeError, match="cannot be combined"):
            ctor(multi_positive=True, extra_texts=3, hard_negatives=2)
    mod = DDPSigmoidLoss(4, multi_positive=True, extra_texts=3)
    sl = SigLipLoss(multi_positive=True, extra_texts=3)
    sc = (torch.tensor(1.0), torch.tensor(0.0))
    for call in (lambda **kw: mod(x, y, sample_ids=ids, **kw), lambda **kw: sl(x, y, *sc, sample_ids=ids, **kw)):
        with pytest.raises(RuntimeError, match="needs extra_text "):
            call(extra_text_ids=eid)
        with pytest.raises(RuntimeError, match=r"extra_text must have shape \[3, 8\]"):
            call(extra_text=torch.randn(2, 8), extra_text_ids=eid)
        with pytest.raises(RuntimeError, match="extra_text is torch.float64"):
            call(extra_text=e.double(), extra_text_ids=eid)
        with pytest.raises(RuntimeError, match="needs extra_text_ids"):
            call(extra_text=e)
        with pytest.raises(RuntimeError, match=r"extra_text_ids must have shape \[3\]"):
            call(extra_text=e, extra_text_ids=torch.arange(4))
        with pytest.raises(RuntimeError, match="extra_text_ids must be an integer tensor"):
            call(extra_text=e, extra_text_ids=eid.float())
        with pytest.raises(RuntimeError, match="extra_text_ids must be an integer tensor"):
            call(extra_text=e, extra_text_ids=[0, 1, 7])
        # valid arguments get as far as the device check (no CPU path)
        with pytest.raises(RuntimeError, match="no CPU path"):
            call(extra_text=e, extra_text_ids=eid)
    with pytest.raises(RuntimeError, match="needs sample_ids"):
        mod(x, y, extra_text=e, extra_text_ids=eid)
    plain = DDPSigmoidLoss(4, multi_positive=True)
    with pytest.raises(RuntimeError, match="without extra_texts"):
        plain(x, y, sample_ids=ids, extra_text=e)
    with pytest.raises(RuntimeError, match="without extra_texts"):
        plain(x, y, sample_ids=ids, extra_text_ids=eid)
    with pytest.raises(RuntimeError, match="without extra_texts"):
        SigLipLoss()(x, y, *sc, extra_text=e)
    if torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="extra_text_ids are on"):
            mod(x.cuda(), y.cuda(), sample_ids=ids.cuda(), extra_text=e.cuda(), extra_text_ids=eid)
