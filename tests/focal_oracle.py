"""Float64 oracle of the focal pair loss (SIGLIP_OPT_FOCAL) — test infrastructure, never the product path. Labels in
{+1, -1, 0} come from the existing label builders (positional, sample ids, extras, label sets, excluded groups); 0 marks
an excluded pair. Pair (i, j) with weight w = a_i c_j |y|, p = sigma(z), m = -y z (the logit of the wrong answer):
    term = w a_t sigma(m)^gamma softplus(m),   a_t = alpha if y = +1 else 1 - alpha (1 without alpha),
which is torchvision's ``sigmoid_focal_loss`` term with target (y + 1) / 2. gamma = 0 without alpha gives the terms of
``exclude_groups_oracle.closed_form_groups`` (``tests/test_focal_cpu.py`` checks that, the torchvision terms and the
closed-form derivative against float64 autograd)."""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import numpy as np

from oracle.siglip_oracle import _sigmoid, _softplus


def focal_terms(z, y, gamma: float, alpha: Optional[float]):
    """(term, g) of every pair: the focal term and its derivative in z, both [R, T] float64, 0 where y = 0.
        g = y = -1:   a_t sigma(z)^gamma (gamma sigma(-z) softplus(z) + sigma(z))
            y = +1:  -a_t sigma(-z)^gamma (gamma sigma(z) softplus(-z) + sigma(-z))"""
    z = np.asarray(z, np.float64)
    y = np.asarray(y, np.float64)
    pos = y > 0
    m = np.where(pos, -z, z)
    sp = _softplus(m)
    pw = np.exp(-gamma * _softplus(-m))            # sigma(m)^gamma without a log of a rounded sigma
    a = np.ones_like(z) if alpha is None else np.where(pos, alpha, 1.0 - alpha)
    mask = np.abs(y)
    term = mask * a * pw * sp
    dm = mask * a * pw * (gamma * _sigmoid(-m) * sp + _sigmoid(m))
    return term, np.where(pos, -dm, dm)


def closed_form_focal(img_blocks, text_blocks, t_prime: float, bias: float, labels: List[List[np.ndarray]],
                      gamma: float, alpha: Optional[float] = None, batches=None, image_weights=None,
                      text_weights=None) -> List[Dict]:
    """``closed_form_groups`` with the focal terms: rank r holds img_blocks[r] ([R_r, D]), chunk c is text_blocks[c]
    ([T_c, D]), labels[r][c] in {+1, -1, 0}, weights per rank or None for ones, batches the divisors B_r (default: the
    rows of img_blocks[r]).
        L_r = (1/B_r) sum w term,   G = w g / B_r,   dimg_r = t G txt_c,  contrib_c = t G^T img_r,
        dt' = t sum G s,  dbias = sum G
    Returns per rank: loss, dimg, dt_prime, dbias, contrib[c], image_loss [R_r] and text_part[c] (no 1/B), as
    ``closed_form_groups``; ``exclude_groups_oracle.dtxt_of`` / ``text_loss_of`` combine the ranks."""
    t = math.exp(t_prime)
    imgs = [np.asarray(x, np.float64) for x in img_blocks]
    txts = [np.asarray(x, np.float64) for x in text_blocks]
    a = [np.ones(x.shape[0]) if image_weights is None else np.asarray(image_weights[r], np.float64)
         for r, x in enumerate(imgs)]
    cw = [np.ones(x.shape[0]) if text_weights is None else np.asarray(text_weights[c], np.float64)
          for c, x in enumerate(txts)]
    out = []
    for r, img in enumerate(imgs):
        br = img.shape[0] if batches is None else batches[r]
        res = dict(loss=0.0, dimg=np.zeros_like(img), dt_prime=0.0, dbias=0.0, contrib=[],
                   image_loss=np.zeros(img.shape[0]), text_part=[])
        for c, txt in enumerate(txts):
            s = img @ txt.T
            term, g = focal_terms(t * s + bias, labels[r][c], gamma, alpha)
            w = a[r][:, None] * cw[c][None, :]
            term = w * term
            G = w * g / br
            res["loss"] += float(term.sum() / br)
            res["image_loss"] += term.sum(axis=1)
            res["text_part"].append(term.sum(axis=0))
            res["dimg"] += t * (G @ txt)
            res["contrib"].append(t * (G.T @ img))
            res["dt_prime"] += float(t * (G * s).sum())
            res["dbias"] += float(G.sum())
        out.append(res)
    return out


def torch_focal_terms(img, txt, t_prime, bias, y, gamma: float, alpha: Optional[float] = None, image_w=None,
                      text_w=None, normalize: bool = False):
    """The pair terms of one rank ([R, T]) in the form the kernels evaluate, a_t exp(-gamma softplus(-m))
    softplus(m) with m = -y z, times a_i c_j |y|: torchvision's ``sigmoid_focal_loss`` terms (``tests/test_focal_cpu.py``
    checks them against it), but with the limits of the terms at z = +-inf. torchvision's own form multiplies z by the
    target, so at z = -inf for a negative its loss and gradient are NaN where the term tends to 0. Differentiable in every
    input; non-finite inputs propagate as autograd propagates them."""
    import torch

    F = torch.nn.functional
    if normalize:
        img, txt = F.normalize(img, dim=-1), F.normalize(txt, dim=-1)
    z = torch.exp(t_prime) * (img @ txt.T) + bias
    pos = y > 0
    m = torch.where(pos, -z, z)
    a = 1.0 if alpha is None else torch.where(pos, alpha, 1.0 - alpha).to(z.dtype)
    loss = a * torch.exp(-gamma * F.softplus(-m)) * F.softplus(m)
    w = y.abs()
    if image_w is not None:
        w = w * image_w[:, None]
    if text_w is not None:
        w = w * text_w[None, :]
    return w * loss


def torch_focal_loss(img, txt, t_prime, bias, y, gamma: float, alpha: Optional[float] = None, image_w=None,
                     text_w=None, normalize: bool = False, batch=None):
    """One rank's focal loss over its whole text set: the sum of ``torch_focal_terms`` / B."""
    terms = torch_focal_terms(img, txt, t_prime, bias, y, gamma, alpha, image_w, text_w, normalize)
    return terms.sum() / (img.shape[0] if batch is None else batch)


def g_bound(gamma: float, lo: float = -60.0, hi: float = 60.0, n: int = 240001) -> float:
    """max over z in [lo, hi] and y = +-1 of |g| without alpha (a_t <= 1 only shrinks it): the bound that keeps
    g * 2^14 inside the fp16 sigma operand."""
    z = np.linspace(lo, hi, n)
    return float(max(np.abs(focal_terms(z, np.full_like(z, s), gamma, None)[1]).max() for s in (-1.0, 1.0)))
