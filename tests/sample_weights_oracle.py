"""Float64 oracle of the loss with per-sample weights (SIGLIP_OPT_SAMPLE_WEIGHTS) — test infrastructure, never the
product path. With unit weights it is ``closed_form_uneven`` / ``closed_form_ids`` / the hard-negatives and extra-text-ids
oracles (``tests/test_sample_weights_cpu.py`` checks all four, and checks this one against float64 autograd of the
weighted op sequence)."""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import numpy as np

from oracle.siglip_oracle import _sigmoid, _softplus


def label_blocks(Bs, Ts, id_blocks=None, extra_id_blocks=None) -> List[List[np.ndarray]]:
    """labels[r][c]: the [B_r, T_c] +-1 labels of rank r's images against chunk c (paired texts first, then extras).
    Without ids: +1 for the own chunk's diagonal only. With id_blocks ([B_p] per rank): +1 iff the image's id equals a
    PAIRED text's id; an extra is never positive unless extra_id_blocks ([T_p - B_p] per rank) give the extras ids."""
    out = []
    for r, br in enumerate(Bs):
        row = []
        for c, (bc, tc) in enumerate(zip(Bs, Ts)):
            if id_blocks is None:
                y = -np.ones((br, tc))
                if r == c:
                    y[np.arange(br), np.arange(br)] = 1.0
            else:
                rid = np.asarray(id_blocks[r], np.int64)
                tid = np.asarray(id_blocks[c], np.int64)
                y = -np.ones((br, tc))
                y[:, :bc] = np.where(rid[:, None] == tid[None, :], 1.0, -1.0)
                if extra_id_blocks is not None and tc > bc:
                    eid = np.asarray(extra_id_blocks[c], np.int64)
                    y[:, bc:] = np.where(rid[:, None] == eid[None, :], 1.0, -1.0)
            row.append(y)
        out.append(row)
    return out


def closed_form_weighted(img_blocks, text_blocks, t_prime: float, bias: float, image_weights=None,
                         text_weights=None, labels: Optional[List[List[np.ndarray]]] = None) -> List[Dict]:
    """Rank r holds img_blocks[r] ([B_r, D]) with weights image_weights[r] ([B_r]); text chunk c is text_blocks[c]
    ([T_c, D]: its paired texts, then its extras) with weights text_weights[c] ([T_c]). None = ones. labels: as
    label_blocks returns (default: positional). Pair (i, j) of rank r and chunk c has weight w = a_r[i] c_c[j]:
        L_r = (1/B_r) sum w softplus(-y z),   G = w (-y sigma(-y z)) / B_r
        dimg_r = t G txt_c,  contrib_c = t G^T img_r,  dt' = t sum G s,  dbias = sum G
    Returns per rank: loss, dimg [B_r, D], dt_prime, dbias and contrib[c] ([T_c, D], that rank's contribution to the
    text gradient of chunk c)."""
    t = math.exp(t_prime)
    imgs = [np.asarray(x, np.float64) for x in img_blocks]
    txts = [np.asarray(x, np.float64) for x in text_blocks]
    if labels is None:
        labels = label_blocks([x.shape[0] for x in imgs], [x.shape[0] for x in txts])
    a = [np.ones(x.shape[0]) if image_weights is None else np.asarray(image_weights[r], np.float64)
         for r, x in enumerate(imgs)]
    cw = [np.ones(x.shape[0]) if text_weights is None else np.asarray(text_weights[c], np.float64)
          for c, x in enumerate(txts)]
    out = []
    for r, img in enumerate(imgs):
        br = img.shape[0]
        res = dict(loss=0.0, dimg=np.zeros_like(img), dt_prime=0.0, dbias=0.0, contrib=[])
        for c, txt in enumerate(txts):
            s = img @ txt.T
            z = t * s + bias
            y = labels[r][c]
            w = a[r][:, None] * cw[c][None, :]
            g = w * (-y * _sigmoid(-y * z)) / br
            res["loss"] += float((w * _softplus(-y * z)).sum() / br)
            res["dimg"] += t * (g @ txt)
            res["contrib"].append(t * (g.T @ img))
            res["dt_prime"] += float(t * (g * s).sum())
            res["dbias"] += float(g.sum())
        out.append(res)
    return out


def dtxt_of(res: List[Dict], c: int) -> np.ndarray:
    """Text gradient of chunk c: the sum over ranks of their contributions (what rank c's step returns)."""
    return sum(x["contrib"][c] for x in res)
