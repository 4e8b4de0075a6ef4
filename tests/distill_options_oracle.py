"""Float64 oracle of distillation composed with the other options (SIGLIP_OPT_DISTILL with extras, label sets, excluded
groups, per-sample losses and top-K) — test infrastructure, never the product path. It composes the single-feature
oracles and adds no loss math of its own beyond ``closed_form_distill``'s formula:

- labels come from the ids / extras oracle (``extra_images_oracle.label_blocks``) or the label-set oracle
  (``label_sets_oracle.set_labels``), in {+1, -1}; ``exclude_groups_oracle.group_labels`` turns excluded pairs into 0;
- per pair, with m = |y| (0 for an excluded pair), y+ = [y > 0] and the teacher's p = sigma(t_T s^T + b_T) from the
  teacher rows of the images and texts (extras included):
      q = (1 - lambda) y+ + lambda p,   term = w m (softplus(z) - q z),   G = w m (sigma(z) - q) / B_r
- the loss divides by B_r, the paired batch, even with extra images (``closed_form_distill`` divides by the rows);
- per-sample losses are the row and column sums of the terms (no 1/B_r);
- top-K lists and metrics rank the student's logits (``retrieval_topk_oracle`` / ``label_sets_oracle``), unchanged.
``tests/test_distill_options_cpu.py`` checks it against float64 autograd of ``exclude_groups_oracle.torch_loss`` with
a teacher, and checks that lambda -> 0 gives the non-distillation oracles."""
from __future__ import annotations

import math
from typing import Dict, List

import numpy as np

from oracle.siglip_oracle import _sigmoid, _softplus


def closed_form_distill_options(img_blocks, text_blocks, t_prime: float, bias: float, timg_blocks, ttxt_blocks,
                                t_prime_T: float, bias_T: float, lam: float, labels: List[List[np.ndarray]], batches,
                                image_weights=None, text_weights=None) -> List[Dict]:
    """Rank r holds img_blocks[r] ([R_r, D]) and timg_blocks[r] ([R_r, D_T]); chunk c is text_blocks[c] ([T_c, D]) and
    ttxt_blocks[c] ([T_c, D_T]); labels[r][c] ([R_r, T_c]) in {+1, -1, 0}; batches[r] = B_r; weights as in
    ``closed_form_groups`` (None = ones). Returns per rank: loss, dimg [R_r, D], dt_prime, dbias, contrib[c] ([T_c, D]),
    image_loss [R_r] and text_part[c] ([T_c], this rank's column sums over chunk c; ``exclude_groups_oracle``'s
    ``dtxt_of`` / ``text_loss_of`` sum them over ranks)."""
    t, tT = math.exp(t_prime), math.exp(t_prime_T)
    imgs = [np.asarray(x, np.float64) for x in img_blocks]
    txts = [np.asarray(x, np.float64) for x in text_blocks]
    timgs = [np.asarray(x, np.float64) for x in timg_blocks]
    ttxts = [np.asarray(x, np.float64) for x in ttxt_blocks]
    a = [np.ones(x.shape[0]) if image_weights is None else np.asarray(image_weights[r], np.float64)
         for r, x in enumerate(imgs)]
    cw = [np.ones(x.shape[0]) if text_weights is None else np.asarray(text_weights[c], np.float64)
          for c, x in enumerate(txts)]
    out = []
    for r, img in enumerate(imgs):
        br = batches[r]
        res = dict(loss=0.0, dimg=np.zeros_like(img), dt_prime=0.0, dbias=0.0, contrib=[],
                   image_loss=np.zeros(img.shape[0]), text_part=[])
        for c, txt in enumerate(txts):
            s = img @ txt.T
            z = t * s + bias
            y = np.asarray(labels[r][c], np.float64)
            p = _sigmoid(tT * (timgs[r] @ ttxts[c].T) + bias_T)
            q = (1.0 - lam) * (y > 0) + lam * p
            w = a[r][:, None] * cw[c][None, :] * np.abs(y)
            term = w * (_softplus(z) - q * z)
            g = w * (_sigmoid(z) - q) / br
            res["loss"] += float(term.sum() / br)
            res["image_loss"] += term.sum(axis=1)
            res["text_part"].append(term.sum(axis=0))
            res["dimg"] += t * (g @ txt)
            res["contrib"].append(t * (g.T @ img))
            res["dt_prime"] += float(t * (g * s).sum())
            res["dbias"] += float(g.sum())
        out.append(res)
    return out
