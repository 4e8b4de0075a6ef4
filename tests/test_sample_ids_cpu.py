"""Multi-positive labels from sample ids (SIGLIP_OPT_SAMPLE_IDS), the parts that need no GPU: the float64 oracle with the
id label matrix, a model of how the sm_90a loss epilogue routes its warp slabs, and the module's argument checks."""
import math

import numpy as np
import pytest
import torch

from oracle.siglip_oracle import closed_form, closed_form_uneven
from sample_ids_oracle import closed_form_ids


def _blocks(Bs, D, seed):
    g = torch.Generator().manual_seed(seed)
    imgs = [torch.nn.functional.normalize(torch.randn(b, D, generator=g, dtype=torch.float64)) for b in Bs]
    txts = [torch.nn.functional.normalize(torch.randn(b, D, generator=g, dtype=torch.float64)) for b in Bs]
    return imgs, txts


def _unique_ids(Bs, seed):
    g = torch.Generator().manual_seed(seed)
    total = sum(Bs)
    ids = (torch.randperm(total, generator=g).to(torch.int64) - total // 2) * 8589934597   # negatives, beyond 2^32
    return list(torch.split(ids, list(Bs)))


def test_unique_ids_reduce_to_the_positional_closed_forms():
    tp, bias = math.log(10.0), -9.0
    W, B, D = 3, 24, 40
    imgs, txts = _blocks([B] * W, D, 5)
    ids = _unique_ids([B] * W, 6)
    got = closed_form_ids([x.numpy() for x in imgs], [x.numpy() for x in txts], [x.numpy() for x in ids], tp, bias)
    ref = closed_form(torch.cat(imgs).numpy(), torch.cat(txts).numpy(), tp, bias, W)
    for r in range(W):
        for k in ("loss", "dt_prime", "dbias"):
            assert abs(got[r][k] - ref[r][k]) <= 1e-12 * abs(ref[r][k])
        assert np.allclose(got[r]["dimg"], ref[r]["dimg"], rtol=1e-12, atol=1e-15)
        dtxt = sum(got[q]["contrib"][r] for q in range(W))
        assert np.allclose(dtxt, ref[r]["dtxt"], rtol=1e-12, atol=1e-15)
    Bs = (40, 24, 33)
    imgs, txts = _blocks(Bs, D, 7)
    ids = _unique_ids(Bs, 8)
    got = closed_form_ids([x.numpy() for x in imgs], [x.numpy() for x in txts], [x.numpy() for x in ids], tp, bias)
    ref = closed_form_uneven([x.numpy() for x in imgs], [x.numpy() for x in txts], tp, bias)
    for r in range(len(Bs)):
        for k in ("loss", "dt_prime", "dbias"):
            assert abs(got[r][k] - ref[r][k]) <= 1e-12 * abs(ref[r][k])
        assert np.allclose(got[r]["dimg"], ref[r]["dimg"], rtol=1e-12, atol=1e-15)
        for c in range(len(Bs)):
            assert np.allclose(got[r]["contrib"][c], ref[r]["contrib"][c], rtol=1e-12, atol=1e-15)


def test_duplicated_ids_match_autograd_of_the_reference_op_sequence():
    """Logits -> -logsigmoid(y z) -> sum / B_r per rank with the explicit id label matrix, text blocks concatenated so
    that autograd sums each text gradient over the ranks (the backward of all_gather)."""
    tp, bias = math.log(10.0), -6.0
    Bs, D = (20, 12, 17), 24
    imgs, txts = _blocks(Bs, D, 11)
    g = torch.Generator().manual_seed(12)
    ids = list(torch.split(torch.randint(0, 9, (sum(Bs),), generator=g), list(Bs)))
    ref = closed_form_ids([x.numpy() for x in imgs], [x.numpy() for x in txts], [x.numpy() for x in ids], tp, bias)
    txt_all = torch.cat(txts).requires_grad_(True)
    ids_all = torch.cat(ids)
    for r in range(len(Bs)):
        img = imgs[r].clone().requires_grad_(True)
        t_prime = torch.tensor(tp, dtype=torch.float64, requires_grad=True)
        b = torch.tensor(bias, dtype=torch.float64, requires_grad=True)
        logits = img @ txt_all.T * t_prime.exp() + b
        labels = torch.where(ids[r][:, None] == ids_all[None, :], 1.0, -1.0).double()
        assert labels.diagonal(offset=sum(Bs[:r])).eq(1.0).all()          # own pairs are always positive
        loss = -torch.nn.functional.logsigmoid(labels * logits).sum() / Bs[r]
        loss.backward()
        assert abs(float(loss.detach()) - ref[r]["loss"]) <= 1e-12 * abs(ref[r]["loss"])
        assert np.allclose(img.grad.numpy(), ref[r]["dimg"], rtol=1e-10, atol=1e-14)
        assert abs(float(t_prime.grad) - ref[r]["dt_prime"]) <= 1e-10 * abs(ref[r]["dt_prime"])
        assert abs(float(b.grad) - ref[r]["dbias"]) <= 1e-10 * abs(ref[r]["dbias"])
    for c in range(len(Bs)):
        sl = slice(sum(Bs[:c]), sum(Bs[:c + 1]))
        total = sum(ref[r]["contrib"][c] for r in range(len(Bs)))
        assert np.allclose(txt_all.grad[sl].numpy(), total, rtol=1e-10, atol=1e-14)


# ---------------------------------------------------------------------------------------------------------------------
# the slab routing of the sm_90a loss epilogue (csrc/siglip_kernels.cu, kModeLoss): 128 x 128 tiles per CTA, 8 consumer
# warps of 16 rows each, 4 slabs of 32 columns per warp; lane l holds rows 16 w + l / 4 (+ 8) and columns
# 8 j + 2 (l % 4) (+ 1) of a slab, j = 0..3, as fragment element i = 4 j + 2 h + e
# ---------------------------------------------------------------------------------------------------------------------
def _route(M, N, own_chunk, row_ids, col_ids):
    """Per element: (in a general-path slab, bit of `pos` set in the owning thread). Mirrors the kernel's per-thread
    id loads (rows clamped to M - 1), per-slab 16-bit masks and the warp vote."""
    general = np.zeros((M, N), dtype=bool)
    posbit = np.zeros((M, N), dtype=bool)
    covered = np.zeros((M, N), dtype=np.int64)
    for row0 in range(0, M, 128):
        for col_base in range(0, N, 128):
            edge = row0 + 128 > M or col_base + 128 > N
            diag = own_chunk and row0 == col_base
            for w in range(8):
                band = row0 + 16 * w
                for c in range(4):
                    col0 = col_base + 32 * c
                    slab_diag = diag and band < col0 + 32 and col0 < band + 16
                    slab_edge = edge and (band + 16 > M or col0 + 32 > N)
                    masks, elems = [], []
                    for lane in range(32):
                        r_lo, c_lo = band + lane // 4, 2 * (lane % 4)
                        rid = [row_ids[min(r_lo, M - 1)], row_ids[min(r_lo + 8, M - 1)]]
                        pos = 0
                        for j in range(4):
                            for e1 in range(2):
                                col = col0 + 8 * j + c_lo + e1
                                if col < N:
                                    for h in range(2):
                                        if col_ids[col] == rid[h]:
                                            pos |= 1 << (4 * j + 2 * h + e1)
                        masks.append(pos)
                        for i in range(16):
                            elems.append((r_lo + 8 * ((i >> 1) & 1), col0 + 8 * (i >> 2) + c_lo + (i & 1), pos >> i & 1))
                    slab_pos = any(m != 0 for m in masks)
                    gen = slab_edge or slab_diag or slab_pos
                    for (rr, cc, bit) in elems:
                        if rr < M and cc < N:
                            covered[rr, cc] += 1
                            general[rr, cc] = gen
                            posbit[rr, cc] = bool(bit)
    assert (covered == 1).all()                      # every element of the matrix belongs to exactly one thread / slab
    return general, posbit


@pytest.mark.parametrize("M,N,own,kind", [
    (300, 300, True, "groups4"), (300, 300, True, "classes10"), (256, 136, False, "classes10"),
    (300, 300, True, "unique"), (256, 136, False, "unique"), (256, 256, True, "all_equal"), (140, 260, False, "groups4"),
])
def test_loss_epilogue_routes_every_id_match_to_the_label_applying_path(M, N, own, kind):
    """Every element whose ids match lies in a slab routed to the general (label-applying) path, with its bit set in the
    owning thread's mask; with unique ids no slab outside today's diagonal / edge classes is added (bit-identity)."""
    g = np.random.default_rng(M * 7 + N)
    n = max(M, N)
    if kind == "groups4":
        base = np.arange(n) // 4
    elif kind == "classes10":
        base = g.integers(0, 10, n)
    elif kind == "all_equal":
        base = np.zeros(n, dtype=np.int64)
    else:
        base = g.permutation(n) * 3 - n
    row_ids = base[:M].astype(np.int64) + (2 ** 35)
    # own chunk: the text ids are the image ids; another chunk: other samples that share some of the classes
    col_ids = row_ids.copy() if own else (base[::-1][:N] if kind != "unique" else base[:N] + 10 * n).astype(np.int64) + (2 ** 35)
    general, posbit = _route(M, N, own, row_ids, col_ids)
    match = row_ids[:, None] == col_ids[None, :]
    assert (posbit == match).all()
    assert general[match].all()
    today, _ = _route(M, N, own, np.arange(M), np.arange(N) if own else np.arange(N) + M)   # positional labels
    if kind == "unique":
        assert (general == today).all()
    else:
        assert general.sum() >= today.sum()


def test_module_argument_errors_are_raised_without_a_gpu():
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    x, y = torch.randn(4, 8), torch.randn(4, 8)
    mod = DDPSigmoidLoss(4, multi_positive=True)
    with pytest.raises(RuntimeError, match="needs sample_ids"):
        mod(x, y)
    with pytest.raises(RuntimeError, match="integer tensor"):
        mod(x, y, sample_ids=torch.zeros(4))
    with pytest.raises(RuntimeError, match="integer tensor"):
        mod(x, y, sample_ids=[0, 1, 2, 3])
    with pytest.raises(RuntimeError, match=r"shape \[4\]"):
        mod(x, y, sample_ids=torch.arange(5))
    with pytest.raises(RuntimeError, match=r"shape \[4\]"):
        mod(x, y, sample_ids=torch.arange(4).reshape(2, 2))
    with pytest.raises(RuntimeError, match="without multi_positive"):
        DDPSigmoidLoss(4)(x, y, sample_ids=torch.arange(4))
    with pytest.raises(RuntimeError, match="needs sample_ids"):
        SigLipLoss(multi_positive=True)(x, y, torch.tensor(1.0), torch.tensor(0.0))
    with pytest.raises(RuntimeError, match="without multi_positive"):
        SigLipLoss()(x, y, torch.tensor(1.0), torch.tensor(0.0), sample_ids=torch.arange(4))
    # valid ids get as far as the device check (no CPU path), for every integer dtype
    for dt in (torch.int32, torch.int64, torch.int16, torch.uint8):
        with pytest.raises(RuntimeError, match="no CPU path"):
            mod(x, y, sample_ids=torch.arange(4, dtype=dt))
