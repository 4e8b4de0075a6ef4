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


def torch_terms(img, txt, t_prime, bias, y, image_w=None, text_w=None, normalize: bool = False, teacher=None):
    """The pair terms of ``torch_loss`` ([R, T]): a_i c_j |y| softplus(-y z). teacher = (timg, ttxt, t'_T, b_T, lambda)
    gives the distillation terms a_i c_j (softplus(z) - q z) instead, q = (1 - lambda) [y = 1] + lambda sigma(exp(t'_T)
    <timg_i, ttxt_j> + b_T) (normalize=True normalises the teacher rows too; no gradient flows to the teacher).
    Non-finite inputs propagate as autograd propagates them; the rows and columns of the per-sample losses are the row
    and column sums of these terms."""
    import torch

    F = torch.nn.functional
    if normalize:
        img, txt = F.normalize(img, dim=-1), F.normalize(txt, dim=-1)
    z = torch.exp(t_prime) * (img @ txt.T) + bias
    w = y.abs()
    if image_w is not None:
        w = w * image_w[:, None]
    if text_w is not None:
        w = w * text_w[None, :]
    if teacher is not None:
        timg, ttxt, ttp, tb, lam = teacher
        if normalize:
            timg, ttxt = F.normalize(timg, dim=-1), F.normalize(ttxt, dim=-1)
        p = torch.sigmoid(torch.exp(torch.as_tensor(ttp, dtype=z.dtype)) * (timg @ ttxt.T) + tb).detach()
        q = (1.0 - lam) * (y > 0).to(z.dtype) + lam * p
        return w * (F.softplus(z) - q * z)
    ys = torch.where(y == 0, -torch.ones_like(y), y)
    return w * F.softplus(-ys * z)


def torch_loss(img, txt, t_prime, bias, y, image_w=None, text_w=None, normalize: bool = False, batch=None,
               teacher=None):
    """A direct torch restatement of one rank's loss over the whole text set (img [R, D], txt [T, D], y [R, T] in
    {+1, -1, 0}): sum over the pairs with |y| = 1 of a_i c_j softplus(-y z) / B (teacher: the distillation terms of
    ``torch_terms``). Differentiable in every input."""
    terms = torch_terms(img, txt, t_prime, bias, y, image_w, text_w, normalize, teacher)
    return terms.sum() / (img.shape[0] if batch is None else batch)


def operand_values(x):
    """The values the kernels consume for an embedding tensor x, as float64: bf16 entries as they are; fp32 / fp16
    entries rounded through fp16(16 x) / 16, saturated at +-4094 (65504 / 16) outside the supported range; NaN and +-inf
    kept as they are."""
    import torch

    x64 = x.detach().double()
    if x.dtype == torch.bfloat16:
        return x64
    r = (x.detach().float() * 16.0).clamp(-65504.0, 65504.0).half().double() / 16.0
    return torch.where(torch.isfinite(x64), r, x64)


ROW_PARTIAL_COLS = 128   # a row's per-sample-loss partial: one loss tile's columns of one text chunk
COL_PARTIAL_ROWS = 16    # a column's partial: one warp's 16 rows of one loss tile
MAX_PARTIAL = 2.0 ** 16


def _partial_class(parts) -> np.ndarray:
    """Per sample (axis 0 of parts, partials along axis 1): 2 for a NaN partial, 1 for a +inf or >= 2^16 one, else 0."""
    nan = np.isnan(parts).any(axis=1)
    big = (np.nan_to_num(parts, nan=0.0, posinf=np.inf) >= MAX_PARTIAL).any(axis=1)
    return np.where(nan, 2, np.where(big, 1, 0))


def sample_loss_classes(terms, chunk_texts, rows: Optional[int] = None) -> Dict[str, np.ndarray]:
    """What the per-sample losses of one rank hold, from its pair terms ([R, sum T_c] float64, chunks side by side):
    image_loss[i] is NaN if one of its row partials (ROW_PARTIAL_COLS columns of a chunk) is NaN, +inf if one is +inf
    or not below 2^16, else the row sum; text_loss_part[j] (this rank's share of text j's loss) the same over column
    partials of COL_PARTIAL_ROWS rows. rows: the rows that belong to the step (default: all)."""
    terms = np.asarray(terms, np.float64)
    R = terms.shape[0] if rows is None else rows
    terms = terms[:R]
    rparts, lo = [], 0
    for T in chunk_texts:
        for c0 in range(lo, lo + T, ROW_PARTIAL_COLS):
            rparts.append(terms[:, c0:min(c0 + ROW_PARTIAL_COLS, lo + T)].sum(axis=1))
        lo += T
    cparts = [terms[r0:r0 + COL_PARTIAL_ROWS].sum(axis=0) for r0 in range(0, R, COL_PARTIAL_ROWS)]

    def decode(total, cls):
        return np.where(cls == 2, np.nan, np.where(cls == 1, np.inf, total))

    return dict(image_loss=decode(terms.sum(axis=1), _partial_class(np.stack(rparts, axis=1))),
                text_loss_part=decode(terms.sum(axis=0), _partial_class(np.stack(cparts, axis=1))))


def clustered(groups, D: int, n_clusters: int, seed: int, noise_seed: int, spread: float = 0.7) -> np.ndarray:
    """Unit embeddings [len(groups), D] around n_clusters random unit centres (drawn from `seed`, so images and texts
    made with the same seed share them), row i near centre groups[i] % n_clusters with noise of norm ~spread (from
    `noise_seed`). Rows of one group have cosine ~1 / (1 + spread^2): the pairs a group excludes carry real weight."""
    centres = np.random.default_rng(seed).standard_normal((n_clusters, D))
    centres /= np.linalg.norm(centres, axis=1, keepdims=True)
    g = np.asarray(groups, np.int64) % n_clusters
    x = centres[g] + spread / math.sqrt(D) * np.random.default_rng(noise_seed).standard_normal((len(g), D))
    return x / np.linalg.norm(x, axis=1, keepdims=True)
