"""Float64 oracle of the loss with extra images per rank (siglip_ctx_create_extras) — test infrastructure, never the
product path.

Rank r holds R_r = B_r + E_r images (its B_r paired images, then its E_r extra images) and T_r >= B_r texts. Over every
text of the global batch:
    L_r    = (1/B_r) sum_{i < R_r} sum_j w_ij softplus(-y_ij z_ij)        (the divisor stays the PAIRED batch)
    dimg_r = [R_r, D]  (rank r's loss only),   dtxt_c = sum_r t G_{r,c}^T img_r  (contraction over R_r rows)
Labels: without ids the positional pair (own chunk, row == col < B_r) only; with ids an image and a text are positive
iff both carry an id and the ids are equal. A paired sample's image and text carry its sample id; an extra text carries
one only with extra_text_ids, an extra image only with extra_image_ids."""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import numpy as np

from oracle.siglip_oracle import _sigmoid, _softplus


def row_ids_of(r, Bs, Rs, ids, extra_image_ids):
    """Ids of rank r's R_r images (None where an image has none)."""
    out = [int(x) for x in ids[r]]
    ext = [None] * (Rs[r] - Bs[r]) if extra_image_ids is None else [int(x) for x in extra_image_ids[r]]
    return out + ext


def col_ids_of(c, Bs, Ts, ids, extra_text_ids):
    """Ids of chunk c's T_c texts (None where a text has none)."""
    out = [int(x) for x in ids[c]]
    ext = [None] * (Ts[c] - Bs[c]) if extra_text_ids is None else [int(x) for x in extra_text_ids[c]]
    return out + ext


def label_blocks(Bs, Rs, Ts, ids=None, extra_text_ids=None, extra_image_ids=None) -> List[List[np.ndarray]]:
    """labels[r][c]: the [R_r, T_c] +-1 labels of rank r's images against chunk c."""
    out = []
    for r in range(len(Bs)):
        row = []
        for c in range(len(Bs)):
            y = -np.ones((Rs[r], Ts[c]))
            if ids is None:
                if r == c:
                    y[np.arange(Bs[r]), np.arange(Bs[r])] = 1.0
            else:
                ri = row_ids_of(r, Bs, Rs, ids, extra_image_ids)
                ci = col_ids_of(c, Bs, Ts, ids, extra_text_ids)
                for i, a in enumerate(ri):
                    for j, b in enumerate(ci):
                        if a is not None and b is not None and a == b:
                            y[i, j] = 1.0
            row.append(y)
        out.append(row)
    return out


def closed_form_extras(img_blocks, text_blocks, Bs, t_prime: float, bias: float, labels=None, image_weights=None,
                       text_weights=None) -> List[Dict]:
    """img_blocks[r]: [R_r, D]; text_blocks[c]: [T_c, D]; Bs: paired batches (the divisors); labels as label_blocks
    returns (default: positional); weights per rank ([R_r] / [T_c]) or None for ones. Returns per rank: loss,
    dimg [R_r, D], dt_prime, dbias and contrib[c] ([T_c, D], its contribution to chunk c's text gradient)."""
    t = math.exp(t_prime)
    imgs = [np.asarray(x, np.float64) for x in img_blocks]
    txts = [np.asarray(x, np.float64) for x in text_blocks]
    Rs = [x.shape[0] for x in imgs]
    Ts = [x.shape[0] for x in txts]
    if labels is None:
        labels = label_blocks(Bs, Rs, Ts)
    a = [np.ones(Rs[r]) if image_weights is None else np.asarray(image_weights[r], np.float64) for r in range(len(imgs))]
    cw = [np.ones(Ts[c]) if text_weights is None else np.asarray(text_weights[c], np.float64) for c in range(len(txts))]
    out = []
    for r, img in enumerate(imgs):
        b = Bs[r]
        res = dict(loss=0.0, dimg=np.zeros_like(img), dt_prime=0.0, dbias=0.0, contrib=[])
        for c, txt in enumerate(txts):
            s = img @ txt.T
            z = t * s + bias
            y = labels[r][c]
            w = a[r][:, None] * cw[c][None, :]
            g = w * (-y * _sigmoid(-y * z)) / b
            res["loss"] += float((w * _softplus(-y * z)).sum() / b)
            res["dimg"] += t * (g @ txt)
            res["contrib"].append(t * (g.T @ img))
            res["dt_prime"] += float(t * (g * s).sum())
            res["dbias"] += float(g.sum())
        out.append(res)
    return out


def dtxt_of(res: List[Dict], c: int) -> np.ndarray:
    """Text gradient of chunk c: the sum over ranks of their contributions (what rank c's step returns)."""
    return sum(x["contrib"][c] for x in res)


def retrieval_metrics_extras(imgs, txts, Bs, ids=None, extra_text_ids=None, extra_image_ids=None) -> List[Dict]:
    """Per rank: i2t_index over its B paired images ([R] with extra_image_ids), t2i_index over its B paired texts ([T]
    with extra_text_ids), global indices (prefix sums of R for images, of T for texts; ties to the lowest index), the
    top-1 rates and the margins (best minus second-best similarity of each ranked row / column)."""
    I = np.concatenate([np.asarray(x, np.float64) for x in imgs])
    T = np.concatenate([np.asarray(x, np.float64) for x in txts])
    S = I @ T.T
    Rs = [len(x) for x in imgs]
    Ts = [len(x) for x in txts]
    off = np.concatenate([[0], np.cumsum(Rs)]).astype(np.int64)
    toff = np.concatenate([[0], np.cumsum(Ts)]).astype(np.int64)
    i2t = np.argmax(S, axis=1)
    t2i = np.argmax(S, axis=0)

    def owner(o_off, g):
        return int(np.searchsorted(o_off, g, side="right") - 1)

    def img_id(g):
        o = owner(off, g)
        l = g - off[o]
        if ids is None:
            return ("pos", o, l) if l < Bs[o] else None
        return row_ids_of(o, Bs, Rs, ids, extra_image_ids)[l]

    def txt_id(j):
        o = owner(toff, j)
        l = j - toff[o]
        if ids is None:
            return ("pos", o, l) if l < Bs[o] else None
        return col_ids_of(o, Bs, Ts, ids, extra_text_ids)[l]

    def margin(M):
        if M.shape[1] < 2:
            return np.full(M.shape[0], np.inf)
        part = np.sort(M, axis=1)
        return part[:, -1] - part[:, -2]

    m_i2t, m_t2i = margin(S), margin(S.T)
    out = []
    for r in range(len(imgs)):
        ni = Rs[r] if (ids is not None and extra_image_ids is not None) else Bs[r]
        nt = Ts[r] if (ids is not None and extra_text_ids is not None) else Bs[r]
        gi = off[r] + np.arange(ni)
        gt = toff[r] + np.arange(nt)
        hi = [(img_id(g) is not None and img_id(g) == txt_id(int(i2t[g]))) for g in gi]
        ht = [(txt_id(j) is not None and txt_id(j) == img_id(int(t2i[j]))) for j in gt]
        out.append(dict(i2t_index=i2t[gi].astype(np.int64), t2i_index=t2i[gt].astype(np.int64),
                        i2t_top1=float(np.mean(hi)), t2i_top1=float(np.mean(ht)),
                        i2t_margin=m_i2t[gi], t2i_margin=m_t2i[gt]))
    return out
