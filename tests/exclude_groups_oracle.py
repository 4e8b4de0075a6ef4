"""Float64 oracle of the loss with excluded same-group pairs (SIGLIP_OPT_EXCLUDE_GROUPS) — test infrastructure, never
the product path. Labels are in {+1, -1, 0}: 0 marks an excluded pair, which adds nothing to any output. With no 0 label
it is ``closed_form_weighted`` of ``sample_weights_oracle`` (``tests/test_exclude_groups_cpu.py`` checks both, and checks
this one against float64 autograd of a direct torch restatement)."""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import numpy as np

from oracle.siglip_oracle import _sigmoid, _softplus


def pad_rows(labels: List[List[np.ndarray]], Rs) -> List[List[np.ndarray]]:
    """Labels of ranks with extra images: rank r's [B_r, T_c] blocks grow to [R_r, T_c], the extra rows all -1 (extra
    images without ids are hard-negative images)."""
    out = []
    for r, row in enumerate(labels):
        out.append([np.concatenate([y, -np.ones((Rs[r] - y.shape[0], y.shape[1]))]) for y in row])
    return out


def group_labels(labels: List[List[np.ndarray]], image_groups, text_groups) -> List[List[np.ndarray]]:
    """labels[r][c] with every negative pair (y = -1) whose image group image_groups[r][i] equals the text group
    text_groups[c][j], both >= 0, set to 0 (excluded). Positives are never excluded."""
    out = []
    for r, row in enumerate(labels):
        gi = np.asarray(image_groups[r], np.int64)
        new = []
        for c, y in enumerate(row):
            gt = np.asarray(text_groups[c], np.int64)
            same = (gi[:, None] == gt[None, :]) & (gi[:, None] >= 0)
            new.append(np.where((y < 0) & same, 0.0, y))
        out.append(new)
    return out


def closed_form_groups(img_blocks, text_blocks, t_prime: float, bias: float, labels: List[List[np.ndarray]],
                       batches=None, image_weights=None, text_weights=None) -> List[Dict]:
    """Rank r holds img_blocks[r] ([R_r, D]) with weights image_weights[r]; text chunk c is text_blocks[c] ([T_c, D])
    with weights text_weights[c]; None = ones. labels[r][c] in {+1, -1, 0}; m = |y| masks the excluded pairs:
        L_r = (1/B_r) sum w m softplus(-y z),   G = w m (-y sigma(-y z)) / B_r
        dimg_r = t G txt_c,  contrib_c = t G^T img_r,  dt' = t sum G s,  dbias = sum G
    batches: B_r (default: the rows of img_blocks[r]). Returns per rank: loss, dimg [R_r, D], dt_prime, dbias,
    contrib[c] ([T_c, D]), image_loss [R_r] (row sums of w m softplus(-y z), no 1/B) and text_part[c] ([T_c]: this rank's
    column sums over chunk c; a text's loss is the sum over ranks, text_loss_of)."""
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
            z = t * s + bias
            y = labels[r][c]
            w = a[r][:, None] * cw[c][None, :] * np.abs(y)
            ys = np.where(y == 0, -1.0, y)   # any finite label: its terms are multiplied by m = 0
            term = w * _softplus(-ys * z)
            g = w * (-ys * _sigmoid(-ys * z)) / br
            res["loss"] += float(term.sum() / br)
            res["image_loss"] += term.sum(axis=1)
            res["text_part"].append(term.sum(axis=0))
            res["dimg"] += t * (g @ txt)
            res["contrib"].append(t * (g.T @ img))
            res["dt_prime"] += float(t * (g * s).sum())
            res["dbias"] += float(g.sum())
        out.append(res)
    return out


def dtxt_of(res: List[Dict], c: int) -> np.ndarray:
    """Text gradient of chunk c: the sum over ranks of their contributions (what rank c's step returns)."""
    return sum(x["contrib"][c] for x in res)


def text_loss_of(res: List[Dict], c: int) -> np.ndarray:
    """Per-sample losses of chunk c's texts: the sum over ranks of their column sums."""
    return sum(x["text_part"][c] for x in res)


def torch_loss(img, txt, t_prime, bias, y, image_w=None, text_w=None, normalize: bool = False, batch=None):
    """A direct torch restatement of one rank's loss over the whole text set (img [R, D], txt [T, D], y [R, T] in
    {+1, -1, 0}): sum over the pairs with |y| = 1 of a_i c_j softplus(-y z) / B. Differentiable in every input."""
    import torch

    if normalize:
        img, txt = torch.nn.functional.normalize(img, dim=-1), torch.nn.functional.normalize(txt, dim=-1)
    z = torch.exp(t_prime) * (img @ txt.T) + bias
    w = y.abs()
    if image_w is not None:
        w = w * image_w[:, None]
    if text_w is not None:
        w = w * text_w[None, :]
    ys = torch.where(y == 0, -torch.ones_like(y), y)
    return (w * torch.nn.functional.softplus(-ys * z)).sum() / (img.shape[0] if batch is None else batch)


def clustered(groups, D: int, n_clusters: int, seed: int, noise_seed: int, spread: float = 0.7) -> np.ndarray:
    """Unit embeddings [len(groups), D] around n_clusters random unit centres (drawn from `seed`, so images and texts
    made with the same seed share them), row i near centre groups[i] % n_clusters with noise of norm ~spread (from
    `noise_seed`). Rows of one group have cosine ~1 / (1 + spread^2): the pairs a group excludes carry real weight."""
    centres = np.random.default_rng(seed).standard_normal((n_clusters, D))
    centres /= np.linalg.norm(centres, axis=1, keepdims=True)
    g = np.asarray(groups, np.int64) % n_clusters
    x = centres[g] + spread / math.sqrt(D) * np.random.default_rng(noise_seed).standard_normal((len(g), D))
    return x / np.linalg.norm(x, axis=1, keepdims=True)
