"""CPU checks of hard-negative captions: the float64 oracle against autograd of the reference's op sequence with the
extras appended to each rank's text chunk (labels forced to -1), against the existing closed forms when K = 0, and the
argument errors of the C creator and of the modules (raised before any GPU work)."""
import ctypes
import math

import numpy as np
import pytest
import torch

from hard_negatives_oracle import closed_form_hard_negatives, retrieval_metrics_hard_negatives
from oracle.siglip_oracle import closed_form_uneven
from sample_ids_oracle import closed_form_ids


def _blocks(Bs, Ks, D, seed):
    g = np.random.default_rng(seed)

    def unit(n):
        x = g.standard_normal((n, D))
        return x / np.linalg.norm(x, axis=1, keepdims=True)
    return [unit(b) for b in Bs], [unit(b) for b in Bs], [unit(k) for k in Ks]


def _autograd(imgs, txts, extras, tp, bias, ids=None):
    """Per rank: logits against every chunk [txt_c; extras_c] -> labels (+1 on the own diagonal or a paired same-id
    text, -1 elsewhere, in particular on every extra) -> -logsigmoid -> sum / B_r, as distributed_sigmoid_loss.py:22-47.
    All ranks' losses are summed over one set of leaves, so each text gradient is the sum over ranks."""
    I = [torch.tensor(x, requires_grad=True) for x in imgs]
    C = [torch.tensor(np.concatenate([t, e]), requires_grad=True) for t, e in zip(txts, extras)]
    out = []
    for r in range(len(I)):
        t_p = torch.tensor(tp, dtype=torch.float64, requires_grad=True)
        b_ = torch.tensor(bias, dtype=torch.float64, requires_grad=True)
        br = I[r].shape[0]
        total = 0
        for c in range(len(C)):
            logits = I[r] @ C[c].T * t_p.exp() + b_
            labels = -torch.ones_like(logits)
            bc = txts[c].shape[0]
            if ids is not None:
                labels[:, :bc] = torch.where(torch.tensor(ids[r])[:, None] == torch.tensor(ids[c])[None, :], 1.0, -1.0)
            elif c == r:
                labels[torch.arange(br), torch.arange(br)] = 1.0
            total = total + (-torch.nn.functional.logsigmoid(labels * logits)).sum()
        total = total / br
        contrib = torch.autograd.grad(total, [I[r], t_p, b_] + C)
        out.append(dict(loss=float(total), dimg=contrib[0].numpy(), dt_prime=float(contrib[1]),
                        dbias=float(contrib[2]), contrib=[x.numpy() for x in contrib[3:]]))
    return out


def _close(a, b, tol=1e-10):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert np.abs(a - b).max() <= tol * max(1.0, np.abs(b).max()), np.abs(a - b).max()


def _compare(got, ref):
    for r, (x, y) in enumerate(zip(got, ref)):
        for k in ("loss", "dimg", "dt_prime", "dbias"):
            _close(x[k], y[k])
        assert len(x["contrib"]) == len(y["contrib"])
        for a, b in zip(x["contrib"], y["contrib"]):
            assert a.shape == b.shape
            _close(a, b)


@pytest.mark.parametrize("Bs,Ks", [((5,), (3,)), ((6, 4, 7), (2, 0, 5)), ((8, 8), (8, 8))])
def test_oracle_matches_autograd_of_the_reference_op_sequence(Bs, Ks):
    tp, bias = math.log(10.0), -4.0
    imgs, txts, extras = _blocks(Bs, Ks, 24, sum(Bs) + sum(Ks))
    _compare(closed_form_hard_negatives(imgs, txts, extras, tp, bias), _autograd(imgs, txts, extras, tp, bias))


def test_oracle_with_ids_never_makes_an_extra_positive():
    """Duplicated ids, and extras that are copies of paired captions: the copies stay negatives."""
    Bs, Ks, D = (6, 5), (3, 4), 16
    tp, bias = math.log(10.0), -3.0
    imgs, txts, extras = _blocks(Bs, Ks, D, 9)
    extras[0][0] = txts[0][0]                    # an extra identical to a caption
    extras[1][1] = txts[0][2]
    ids = [np.array([1, 1, 2, 3, 4, 4]), np.array([2, 5, 1, 6, 6])]
    _compare(closed_form_hard_negatives(imgs, txts, extras, tp, bias, ids),
             _autograd(imgs, txts, extras, tp, bias, ids))


def test_no_extras_reduce_to_the_existing_closed_forms():
    tp, bias = math.log(10.0), -7.0
    Bs = (7, 3, 5)
    imgs, txts, extras = _blocks(Bs, (0, 0, 0), 32, 3)
    _compare(closed_form_hard_negatives(imgs, txts, extras, tp, bias), closed_form_uneven(imgs, txts, tp, bias))
    ids = [np.array([0, 1, 1, 2, 3, 4, 5]), np.array([1, 6, 7]), np.array([8, 8, 0, 9, 10])]
    _compare(closed_form_hard_negatives(imgs, txts, extras, tp, bias, ids),
             closed_form_ids(imgs, txts, ids, tp, bias))


def test_metrics_oracle_counts_a_winning_extra_as_a_miss():
    D = 8
    imgs = [np.eye(D)[:3], np.eye(D)[3:5]]
    txts = [np.eye(D)[:3] * 0.9, np.eye(D)[3:5] * 0.9]
    extras = [np.eye(D)[[1]], np.zeros((2, D))]          # rank 0's extra beats image 1's caption
    m = retrieval_metrics_hard_negatives(imgs, txts, extras)
    assert list(m[0]["i2t_index"]) == [0, 3, 2]           # global text index of the extra: 3 (B_0 = 3, first extra)
    assert m[0]["i2t_top1"] == pytest.approx(2 / 3)
    assert list(m[1]["i2t_index"]) == [4, 5]              # rank 1's texts start at T_0 = 4
    assert m[1]["i2t_top1"] == 1.0
    assert list(m[0]["t2i_index"]) == [0, 1, 2] and m[0]["t2i_top1"] == 1.0


def test_creator_rejects_invalid_text_counts_before_touching_the_gpu():
    from distributed_sigmoid_loss_b200 import _capi

    L = _capi.lib()
    h = ctypes.c_void_p()

    def create(rank, world, bs, ts, D=64):
        arr = lambda v: (ctypes.c_int * len(v))(*v) if v is not None else None
        return L.siglip_ctx_create_texts(ctypes.byref(h), 0, rank, world, arr(bs), arr(ts), D)

    inv = _capi.SIGLIP_ERR_INVALID
    assert create(0, 2, [4, 4], [4, 3]) == inv            # fewer texts than images on a rank
    assert create(1, 2, [4, 4], [0, 8]) == inv
    assert create(0, 1, [0], [4]) == inv                  # B >= 1
    assert create(0, 1, [4], None) == inv                 # null list
    assert create(0, 1, None, [4]) == inv
    assert create(2, 2, [4, 4], [5, 5]) == inv            # rank >= world
    assert create(0, 33, [4] * 33, [5] * 33) == inv       # world > 32
    assert create(0, 1, [4], [6], D=60) == inv            # D % 8 != 0
    assert "texts_per_rank" in _capi.last_error() or "D" in _capi.last_error()
    if not torch.cuda.is_available():
        assert create(0, 2, [4, 4], [6, 4]) == _capi.SIGLIP_ERR_NO_DEVICE   # valid: gets as far as the device check


def test_module_argument_errors_are_raised_without_a_gpu():
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    x, y = torch.randn(4, 8), torch.randn(4, 8)
    for bad in (-1, 1.5, True, "2"):
        with pytest.raises(RuntimeError, match="hard_negatives must be an int"):
            DDPSigmoidLoss(4, hard_negatives=bad)
        with pytest.raises(RuntimeError, match="hard_negatives must be an int"):
            SigLipLoss(hard_negatives=bad)
    mod = DDPSigmoidLoss(4, hard_negatives=3)
    with pytest.raises(RuntimeError, match="needs negative_text"):
        mod(x, y)
    with pytest.raises(RuntimeError, match="must be a tensor"):
        mod(x, y, negative_text=[[0.0] * 8] * 3)
    with pytest.raises(RuntimeError, match=r"shape \[3, 8\]"):
        mod(x, y, negative_text=torch.randn(2, 8))
    with pytest.raises(RuntimeError, match=r"shape \[3, 8\]"):
        mod(x, y, negative_text=torch.randn(3, 9))
    with pytest.raises(RuntimeError, match=r"shape \[3, 8\]"):
        mod(x, y, negative_text=torch.randn(24))
    with pytest.raises(RuntimeError, match="float64, the texts torch.float32"):
        mod(x, y, negative_text=torch.randn(3, 8, dtype=torch.float64))
    with pytest.raises(RuntimeError, match="without hard_negatives"):
        DDPSigmoidLoss(4)(x, y, negative_text=torch.randn(3, 8))
    sl = SigLipLoss(hard_negatives=2)
    with pytest.raises(RuntimeError, match="needs negative_text"):
        sl(x, y, torch.tensor(1.0), torch.tensor(0.0))
    with pytest.raises(RuntimeError, match="without hard_negatives"):
        SigLipLoss()(x, y, torch.tensor(1.0), torch.tensor(0.0), negative_text=torch.randn(2, 8))
    # a valid negative_text gets as far as the device check (no CPU path)
    with pytest.raises(RuntimeError, match="no CPU path"):
        mod(x, y, negative_text=torch.randn(3, 8))
    with pytest.raises(RuntimeError, match="no CPU path"):
        sl(x, y, torch.tensor(1.0), torch.tensor(0.0), negative_text=torch.randn(2, 8))
