"""Float64 oracle of the per-sample losses (siglip_request_sample_losses) — test infrastructure, never the product path.

Built on the conventions of ``closed_form_extras``: rank r holds R_r images (paired, then extra) and chunk c holds T_c
texts (paired, then extras), with labels as ``extra_images_oracle.label_blocks`` returns and per-sample weights (None =
ones). Over every pair of the global batch, with w_ij = a_r[i] c_c[j] and the loss's own term l_ij = softplus(-y_ij z_ij):
    image_loss_r[i] = sum_c sum_j w_ij l_ij        (every text of every chunk)
    text_loss_c[j]  = sum_r sum_i w_ij l_ij        (every image of every rank)
No 1/B: the rank's loss is image_loss_r.sum() / B_r, and sum_r image_loss_r.sum() == sum_c text_loss_c.sum().
The kernel adds partials in 64-bit fixed point (value * 2^32); ``fixed_point_partial`` / ``fixed_point_decode`` model
that encoding for the CPU tests."""
from __future__ import annotations

import math
from typing import Dict, List

import numpy as np

from extra_images_oracle import label_blocks
from oracle.siglip_oracle import _softplus

SCALE = 2.0 ** 32
MAX_PARTIAL = 2.0 ** 16


def sample_losses(img_blocks, text_blocks, Bs, t_prime: float, bias: float, labels=None, image_weights=None,
                  text_weights=None) -> List[Dict]:
    """img_blocks[r]: [R_r, D]; text_blocks[c]: [T_c, D]; Bs: paired batches; labels / weights as closed_form_extras
    takes them. Returns per rank: image_loss [R_r], text_loss [T_r] and loss (the rank's loss, for the identities)."""
    t = math.exp(t_prime)
    imgs = [np.asarray(x, np.float64) for x in img_blocks]
    txts = [np.asarray(x, np.float64) for x in text_blocks]
    Rs = [x.shape[0] for x in imgs]
    Ts = [x.shape[0] for x in txts]
    if labels is None:
        labels = label_blocks(Bs, Rs, Ts)
    a = [np.ones(Rs[r]) if image_weights is None else np.asarray(image_weights[r], np.float64) for r in range(len(imgs))]
    cw = [np.ones(Ts[c]) if text_weights is None else np.asarray(text_weights[c], np.float64) for c in range(len(txts))]
    img_loss = [np.zeros(R) for R in Rs]
    txt_loss = [np.zeros(T) for T in Ts]
    for r, img in enumerate(imgs):
        for c, txt in enumerate(txts):
            z = t * (img @ txt.T) + bias
            L = a[r][:, None] * cw[c][None, :] * _softplus(-labels[r][c] * z)
            img_loss[r] += L.sum(axis=1)
            txt_loss[c] += L.sum(axis=0)
    return [dict(image_loss=img_loss[r], text_loss=txt_loss[r], loss=float(img_loss[r].sum() / Bs[r]))
            for r in range(len(imgs))]


def fixed_point_partial(v: float):
    """(word, poison) a partial adds: round(v * 2^32) as an integer, or a poison bit (1: too large or +inf, 2: NaN)."""
    v = np.float32(v)
    if v < MAX_PARTIAL:
        return int(np.rint(np.float64(v) * SCALE)), 0   # v * 2^32 < 2^48: rounds only below 2^-8 (fp32 ulp)
    return 0, (2 if np.isnan(v) else 1)


def fixed_point_decode(word: int, poison: int) -> np.float32:
    if poison & 2:
        return np.float32(np.nan)
    if poison & 1:
        return np.float32(np.inf)
    return np.float32(np.float64(word % (1 << 64)) / SCALE)
