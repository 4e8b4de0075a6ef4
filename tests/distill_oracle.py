"""Float64 oracle of distillation from a frozen teacher (SIGLIP_OPT_DISTILL) — test infrastructure, never the product
path. With lambda = 0 it is ``closed_form_weighted`` (``tests/test_distill_cpu.py`` checks that, and checks this oracle
against float64 autograd of a direct restatement).

Per rank r and text chunk c, with the student logits z = t s + b (s = img_r txt_c^T, t = exp(t')), the teacher's
p = sigma(t_T s^T + b_T) (s^T = timg_r ttxt_c^T), the hard labels y in {0, 1} and the weights w:
    q = (1 - lambda) y + lambda p
    L_r = (1/B_r) sum w (softplus(z) - q z),   G = w (sigma(z) - q) / B_r
    dimg_r = t G txt_c,  contrib_c = t G^T img_r,  dt' = t sum G s,  dbias = sum G
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import numpy as np

from oracle.siglip_oracle import _sigmoid, _softplus
from sample_weights_oracle import label_blocks


def closed_form_distill(img_blocks, text_blocks, t_prime: float, bias: float, timg_blocks, ttxt_blocks,
                        t_prime_T: float, bias_T: float, lam: float, image_weights=None, text_weights=None,
                        labels: Optional[List[List[np.ndarray]]] = None) -> List[Dict]:
    """Rank r holds img_blocks[r] ([B_r, D]) and timg_blocks[r] ([B_r, D_T]); chunk c is text_blocks[c] ([B_c, D]) and
    ttxt_blocks[c] ([B_c, D_T]). labels: the +-1 labels of label_blocks (default: positional). Weights as in
    closed_form_weighted. Returns per rank: loss, dimg, dt_prime, dbias and contrib[c]."""
    t, tT = math.exp(t_prime), math.exp(t_prime_T)
    imgs = [np.asarray(x, np.float64) for x in img_blocks]
    txts = [np.asarray(x, np.float64) for x in text_blocks]
    timgs = [np.asarray(x, np.float64) for x in timg_blocks]
    ttxts = [np.asarray(x, np.float64) for x in ttxt_blocks]
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
            p = _sigmoid(tT * (timgs[r] @ ttxts[c].T) + bias_T)
            y = (labels[r][c] > 0).astype(np.float64)
            q = (1.0 - lam) * y + lam * p
            w = a[r][:, None] * cw[c][None, :]
            g = w * (_sigmoid(z) - q) / br
            res["loss"] += float((w * (_softplus(z) - q * z)).sum() / br)
            res["dimg"] += t * (g @ txt)
            res["contrib"].append(t * (g.T @ img))
            res["dt_prime"] += float(t * (g * s).sum())
            res["dbias"] += float(g.sum())
        out.append(res)
    return out
