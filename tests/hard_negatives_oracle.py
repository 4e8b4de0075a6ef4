"""Float64 oracle of the loss with hard-negative captions (siglip_ctx_create_texts) — test infrastructure, never the
product path. It extends ``oracle.siglip_oracle.closed_form_uneven`` (pinned on the reference's fixtures) and
``tests/sample_ids_oracle.closed_form_ids`` with extra text rows per rank that are negatives for every image;
``tests/test_hard_negatives_cpu.py`` checks it against both for K = 0 and against float64 autograd of the reference's op
sequence otherwise."""
from __future__ import annotations

import math
from typing import Dict, List

import numpy as np

from oracle.siglip_oracle import _sigmoid, _softplus


def closed_form_hard_negatives(img_blocks, txt_blocks, extra_blocks, t_prime: float, bias: float,
                               id_blocks=None) -> List[Dict]:
    """Rank r holds img_blocks[r] ([B_r, D]), its paired captions txt_blocks[r] ([B_r, D]) and its hard negatives
    extra_blocks[r] ([K_r, D], K_r may be 0). Text chunk c is [txt_blocks[c]; extra_blocks[c]] (T_c = B_c + K_c rows).
    Labels: +1 for the positional pair (own chunk, row i, column i < B_r) or, with id_blocks ([B_r] integers per rank),
    for a PAIRED text of any chunk with the same id; -1 for everything else, so an extra is never positive. Loss and
    gradients keep the formulas of distributed_sigmoid_loss.py:24-47 (loss divided by the rank's image batch).
    Returns per rank: loss, dimg [B_r, D], dt_prime, dbias and contrib[c] ([T_c, D], that rank's contribution to the
    text gradient of chunk c, extras' rows last)."""
    t = math.exp(t_prime)
    chunks = []
    for txt, ext in zip(txt_blocks, extra_blocks):
        txt = np.asarray(txt, dtype=np.float64)
        ext = np.asarray(ext, dtype=np.float64).reshape(-1, txt.shape[1])
        chunks.append((np.concatenate([txt, ext]), txt.shape[0]))
    ids = None if id_blocks is None else [np.asarray(x, dtype=np.int64) for x in id_blocks]
    out = []
    for r, img in enumerate(img_blocks):
        img = np.asarray(img, dtype=np.float64)
        br = img.shape[0]
        res = dict(loss=0.0, dimg=np.zeros_like(img), dt_prime=0.0, dbias=0.0, contrib=[])
        for c, (txt, bc) in enumerate(chunks):
            s = img @ txt.T
            z = t * s + bias
            y = -np.ones_like(z)
            if ids is not None:
                y[:, :bc] = np.where(ids[r][:, None] == ids[c][None, :], 1.0, -1.0)
            elif c == r:
                y[np.arange(br), np.arange(br)] = 1.0
            g = -y * _sigmoid(-y * z) / br
            res["loss"] += float(_softplus(-y * z).sum() / br)
            res["dimg"] += t * (g @ txt)
            res["contrib"].append(t * (g.T @ img))
            res["dt_prime"] += float(t * (g * s).sum())
            res["dbias"] += float(g.sum())
        out.append(res)
    return out


def retrieval_metrics_hard_negatives(img_blocks, txt_blocks, extra_blocks, id_blocks=None) -> List[Dict]:
    """In-batch top-1 with hard negatives: i2t over every text of the global batch (global text index = prefix sums of
    B_p + K_p), a hit only when the best text is a PAIRED one that matches (position, or id); t2i over every image for
    each paired text. Ties go to the lowest index."""
    I = np.concatenate([np.asarray(x, np.float64) for x in img_blocks])
    rows, paired_of, counts = [], [], []
    for c, (txt, ext) in enumerate(zip(txt_blocks, extra_blocks)):
        txt = np.asarray(txt, np.float64)
        ext = np.asarray(ext, np.float64).reshape(-1, txt.shape[1])
        rows += [txt, ext]
        paired_of += [(c, i) for i in range(len(txt))] + [None] * len(ext)
        counts.append(len(txt) + len(ext))
    T = np.concatenate(rows)
    S = I @ T.T
    off = np.concatenate([[0], np.cumsum([len(x) for x in img_blocks])]).astype(np.int64)
    toff = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    gid = np.concatenate([np.asarray(x, np.int64) for x in id_blocks]) if id_blocks is not None else np.arange(len(I))
    i2t = np.argmax(S, axis=1)
    out = []
    for r in range(len(img_blocks)):
        b = off[r + 1] - off[r]
        i2t_r = i2t[off[r]:off[r + 1]]
        hit_i = []
        for i, j in enumerate(i2t_r):
            p = paired_of[j]
            hit_i.append(p is not None and gid[off[p[0]] + p[1]] == gid[off[r] + i])
        cols = toff[r] + np.arange(b)                  # my paired texts
        t2i_r = np.argmax(S[:, cols], axis=0)
        hit_t = gid[t2i_r] == gid[off[r] + np.arange(b)]
        out.append(dict(i2t_index=i2t_r.astype(np.int64), t2i_index=t2i_r.astype(np.int64),
                        i2t_top1=float(np.mean(hit_i)), t2i_top1=float(hit_t.mean()), S=S, toff=toff, off=off))
    return out
