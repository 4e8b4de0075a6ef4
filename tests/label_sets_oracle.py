"""Float64 oracle of the loss with multi-label positives (SIGLIP_OPT_LABEL_SETS) — test infrastructure, never the
product path. Every image and text carries a set of M int64 labels (a negative entry is an empty slot). Pair (image i of
rank r, text j of chunk c) is positive iff it is the own-chunk positional pair (r == c, i == j < B_r) or the two sets
share a label >= 0. The label blocks this builds go through ``exclude_groups_oracle.closed_form_groups`` (weights and
excluded groups included), and the retrieval variant below follows ``retrieval_topk_oracle.topk_retrieval`` with the
set-intersection hit rule."""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np

from exclude_groups_oracle import closed_form_groups, group_labels
from retrieval_topk_oracle import _ranked


def meet(a, b) -> np.ndarray:
    """[n, m] bool: does set a[i] ([n, M]) share a label >= 0 with set b[j] ([m, M])?"""
    a = np.asarray(a, np.int64)
    b = np.asarray(b, np.int64)
    eq = (a[:, None, :, None] == b[None, :, None, :]) & (a[:, None, :, None] >= 0)
    return eq.any(axis=(2, 3))


def set_labels(image_sets, text_sets, batches) -> List[List[np.ndarray]]:
    """labels[r][c] ([R_r, T_c] in {+1, -1}) from the per-rank image sets ([R_r, M]: paired, then extra images) and the
    per-chunk text sets ([T_c, M]: paired, then extra texts)."""
    out = []
    for r, si in enumerate(image_sets):
        row = []
        for c, st in enumerate(text_sets):
            pos = meet(si, st)
            if r == c:
                b = batches[r]
                pos[np.arange(b), np.arange(b)] = True
            row.append(np.where(pos, 1.0, -1.0))
        out.append(row)
    return out


def closed_form_sets(img_blocks, text_blocks, t_prime: float, bias: float, image_sets, text_sets, batches=None,
                     image_weights=None, text_weights=None, image_groups=None, text_groups=None) -> List[Dict]:
    """``closed_form_groups`` on the labels of ``set_labels``; with image_groups / text_groups the same-group negatives are
    excluded after the positives (``group_labels``)."""
    bs = [np.asarray(x).shape[0] for x in img_blocks] if batches is None else list(batches)
    labels = set_labels(image_sets, text_sets, bs)
    if image_groups is not None:
        labels = group_labels(labels, image_groups, text_groups)
    return closed_form_groups(img_blocks, text_blocks, t_prime, bias, labels, batches, image_weights, text_weights)


def dense_labels(image_sets, text_sets, batches) -> np.ndarray:
    """The global [sum R_r, sum T_c] label matrix of ``set_labels``, blocks side by side."""
    return np.block(set_labels(image_sets, text_sets, batches))


def topk_retrieval_sets(imgs, txts, batches, k, image_sets, text_sets) -> List[Dict]:
    """``topk_retrieval`` with the label-set hit rule: i2t ranks all R_r images of each rank, t2i all T_r texts; a hit
    is the positional pair (i == j < B_r on the own rank) or a pair whose sets meet. Returns the same keys."""
    I = np.concatenate([np.asarray(x, np.float64) for x in imgs])
    T = np.concatenate([np.asarray(x, np.float64) for x in txts])
    S = I @ T.T
    off = np.concatenate([[0], np.cumsum([len(x) for x in imgs])]).astype(np.int64)
    toff = np.concatenate([[0], np.cumsum([len(x) for x in txts])]).astype(np.int64)
    W = len(imgs)
    hit = np.where(dense_labels(image_sets, text_sets, batches) > 0, True, False)

    def gaps(M):
        srt = -np.sort(-M, axis=1)
        if M.shape[1] <= k:
            return np.full(M.shape[0], np.inf)
        return srt[:, k - 1] - srt[:, k]

    rows, cols = _ranked(S, k), _ranked(S.T, k)
    g_i2t, g_t2i = gaps(S), gaps(S.T)
    out = []
    for r in range(W):
        ni, nt = len(imgs[r]), len(txts[r])
        i2t = rows[off[r]:off[r] + ni]
        t2i = cols[toff[r]:toff[r] + nt]

        def first(lst, is_hit):
            f = np.full(len(lst), k, np.int64)
            for i, row in enumerate(lst):
                for s, j in enumerate(row.tolist()):
                    if j >= 0 and is_hit(i, j):
                        f[i] = s
                        break
            return f

        fi = first(i2t, lambda i, j: hit[off[r] + i, j])
        ft = first(t2i, lambda i, g: hit[g, toff[r] + i])
        out.append(dict(i2t_topk=i2t, t2i_topk=t2i,
                        i2t_recall=np.array([(fi < q).mean() for q in range(1, k + 1)]),
                        t2i_recall=np.array([(ft < q).mean() for q in range(1, k + 1)]),
                        i2t_first=fi, t2i_first=ft,
                        i2t_gap=g_i2t[off[r]:off[r] + ni], t2i_gap=g_t2i[toff[r]:toff[r] + nt], S=S, off=off, toff=toff))
    return out


def hierarchy_sets(leaves, parents: Dict[int, int], m: int) -> np.ndarray:
    """[n, m] sets of a label hierarchy: leaf, then its parent, grandparent, ... (parents[x] = parent of x), -1 padded."""
    out = np.full((len(leaves), m), -1, np.int64)
    for i, x in enumerate(leaves):
        chain: List[int] = []
        cur: Optional[int] = int(x)
        while cur is not None and len(chain) < m:
            chain.append(cur)
            cur = parents.get(cur)
        out[i, :len(chain)] = chain
    return out
