"""Float64 oracle of the loss with extra texts that carry ids (SIGLIP_OPT_EXTRA_TEXT_IDS) — test infrastructure, never
the product path. It extends ``tests/hard_negatives_oracle.closed_form_hard_negatives`` (which it equals when no extra
id matches an image) with ids on the extras; ``tests/test_extra_text_ids_cpu.py`` checks it against float64 autograd
of the reference's op sequence and against ``closed_form_ids`` on repeated images."""
from __future__ import annotations

import math
from typing import Dict, List

import numpy as np

from oracle.siglip_oracle import _sigmoid, _softplus


def _text_ids(id_blocks, extra_id_blocks):
    """Per chunk c: the [T_c] ids of its texts, the sample ids of its paired texts first, then its extras' ids."""
    return [np.concatenate([np.asarray(i, np.int64), np.asarray(e, np.int64).reshape(-1)])
            for i, e in zip(id_blocks, extra_id_blocks)]


def closed_form_extra_text_ids(img_blocks, txt_blocks, extra_blocks, id_blocks, extra_id_blocks, t_prime: float,
                               bias: float) -> List[Dict]:
    """Rank r holds img_blocks[r] ([B_r, D]) with sample ids id_blocks[r] ([B_r]), its paired captions txt_blocks[r]
    ([B_r, D]) and its extra texts extra_blocks[r] ([K_r, D], K_r may be 0) with ids extra_id_blocks[r] ([K_r]). Text
    chunk c is [txt_blocks[c]; extra_blocks[c]] with ids [id_blocks[c]; extra_id_blocks[c]]. Pair (i, j) of rank r and
    chunk c is positive iff id_blocks[r][i] equals the id of text j, so the [B_r, sum T] label matrix comes from the ids
    alone. Loss and gradients keep the formulas of distributed_sigmoid_loss.py:24-47 (loss divided by the rank's image
    batch). Returns per rank: loss, dimg [B_r, D], dt_prime, dbias and contrib[c] ([T_c, D], that rank's contribution to
    the text gradient of chunk c, extras' rows last)."""
    t = math.exp(t_prime)
    tids = _text_ids(id_blocks, extra_id_blocks)
    chunks = []
    for txt, ext in zip(txt_blocks, extra_blocks):
        txt = np.asarray(txt, dtype=np.float64)
        chunks.append(np.concatenate([txt, np.asarray(ext, dtype=np.float64).reshape(-1, txt.shape[1])]))
    out = []
    for r, img in enumerate(img_blocks):
        img = np.asarray(img, dtype=np.float64)
        br = img.shape[0]
        rid = np.asarray(id_blocks[r], np.int64)
        res = dict(loss=0.0, dimg=np.zeros_like(img), dt_prime=0.0, dbias=0.0, contrib=[])
        for c, txt in enumerate(chunks):
            s = img @ txt.T
            z = t * s + bias
            y = np.where(rid[:, None] == tids[c][None, :], 1.0, -1.0)
            g = -y * _sigmoid(-y * z) / br
            res["loss"] += float(_softplus(-y * z).sum() / br)
            res["dimg"] += t * (g @ txt)
            res["contrib"].append(t * (g.T @ img))
            res["dt_prime"] += float(t * (g * s).sum())
            res["dbias"] += float(g.sum())
        out.append(res)
    return out


def retrieval_metrics_extra_text_ids(img_blocks, txt_blocks, extra_blocks, id_blocks, extra_id_blocks) -> List[Dict]:
    """In-batch top-1 when every text carries an id: i2t over every text of the global batch (global text index =
    prefix sums of T_p), t2i over every image for each of the rank's T_r texts (paired ones, then extras). A top-1 is
    a hit iff its image and text ids are equal, so an extra caption can be a hit and an extra whose id matches no image
    never is. Ties go to the lowest index."""
    I = np.concatenate([np.asarray(x, np.float64) for x in img_blocks])
    tids = _text_ids(id_blocks, extra_id_blocks)
    texts = []
    for txt, ext in zip(txt_blocks, extra_blocks):
        txt = np.asarray(txt, np.float64)
        texts += [txt, np.asarray(ext, np.float64).reshape(-1, txt.shape[1])]
    S = I @ np.concatenate(texts).T
    off = np.concatenate([[0], np.cumsum([len(x) for x in img_blocks])]).astype(np.int64)
    toff = np.concatenate([[0], np.cumsum([len(x) for x in tids])]).astype(np.int64)
    gid = np.concatenate([np.asarray(x, np.int64) for x in id_blocks])
    tgid = np.concatenate(tids)
    i2t = np.argmax(S, axis=1)
    t2i = np.argmax(S, axis=0)
    out = []
    for r in range(len(img_blocks)):
        i2t_r = i2t[off[r]:off[r + 1]]
        t2i_r = t2i[toff[r]:toff[r + 1]]
        hit_i = tgid[i2t_r] == gid[off[r]:off[r + 1]]
        hit_t = gid[t2i_r] == tgid[toff[r]:toff[r + 1]]
        out.append(dict(i2t_index=i2t_r.astype(np.int64), t2i_index=t2i_r.astype(np.int64),
                        i2t_top1=float(hit_i.mean()), t2i_top1=float(hit_t.mean()), S=S, off=off, toff=toff))
    return out
