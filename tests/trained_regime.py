"""Inputs in the regime of a trained SigLIP model, and the float64 quantities the trained-regime tests compare against —
test infrastructure, never the product path (tests/test_trained_regime_cpu.py pins what it produces).

At initialisation-like logits (independent random unit embeddings, t = 10, b = -10) the own chunk's gradients are
almost entirely the positive-pair term, which the gradient kernel adds in fp32 from g_diag; the negatives reach dimg /
dtxt only through the fp16 sigma operand G and are well under 1 % of the gradient norm. A trained model has t of order
100, large positive logits on the positives and a tail of hard negatives above z = 0: there the negatives carry most of
the gradient, slabs of the fast (series) path and of the general path sit side by side in one tile, and sigma * 2^14
reaches both ends of fp16 (16384 for hard negatives, subnormals below sigma = 3.7e-9, z < -19.4).

make_batch builds such a batch from orthogonal-ish components (every component a unit vector, weights summing to 1):
  * a modality offset, +e for images and -e for texts: -gap on every image-text logit (the "modality gap");
  * one of K cluster centroids forming a simplex (pairwise -1/(K-1)); clusters are contiguous index ranges of every
    chunk, so the 16x32 slabs between two clusters take the series path;
  * for "generic" samples (a share of every cluster, like the stock photos and captions that match many others), a
    direction of their cluster: two generic samples of a cluster are hard negatives near generic_z, and nearly every
    16x32 slab inside a cluster holds such a pair, so it takes the general path whatever the batch size or D;
  * a pair vector shared by an image and its caption (correlation rho spread so that positive logits cover the
    regime's range); a "twin" shares most of its pair vector with an earlier sample of its cluster (a near-duplicate):
    a hard negative above z = 0 with positional labels, a duplicated sample id with ids;
  * isotropic noise.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from oracle.siglip_oracle import _sigmoid

SIGMA_NORMAL_MIN = 2.0 ** -28      # 3.7e-9: sigma * 2^14 below fp16's smallest normal 2^-14 (z < -19.4)


@dataclass(frozen=True)
class Regime:
    """t, bias: the logit scale and bias of the step (bias None: the stationary bias of the batch, sum G = 0, found after
    the batch is built with design_bias). neg_z: mean logit of a negative pair inside a cluster. pos_z: the range the
    positive logits are spread over (before noise). generic_z: logit of a pair of generic samples of one cluster, a
    share `generic` of the samples. noise: weight of the isotropic component."""
    name: str
    t: float
    bias: Optional[float]
    neg_z: float
    pos_z: Tuple[float, float]
    design_bias: float = -13.0
    generic_z: float = 10.0
    clusters: int = 2
    generic: float = 0.15
    twins: float = 0.1
    noise: float = 0.1

    @property
    def t_prime(self) -> float:
        return math.log(self.t)


# t ~ 100 and b ~ -13 are where trained SigLIP models end up; t = 300 puts hard negatives at sigma * 2^14 -> 16384 and
# spreads the other negatives through fp16's subnormals; "separated" is a batch the model has learnt: most negatives
# below z = -19.4 (sigma < 3.7e-9), positives mostly well above 0.
REGIMES: Dict[str, Regime] = {
    "trained": Regime("trained", 100.0, -13.0, neg_z=-8.0, pos_z=(-5.0, 40.0)),
    "stationary": Regime("stationary", 100.0, None, neg_z=-8.0, pos_z=(-5.0, 40.0), generic_z=20.0),
    "t300": Regime("t300", 300.0, -30.0, neg_z=-8.0, pos_z=(-5.0, 40.0), design_bias=-30.0, noise=0.04),
    "separated": Regime("separated", 100.0, -10.0, neg_z=-26.0, pos_z=(0.0, 40.0), design_bias=-10.0, generic_z=0.0,
                        noise=0.05),
}


def _orthonormal(g: torch.Generator, n: int, D: int) -> torch.Tensor:
    q, _ = torch.linalg.qr(torch.randn(D, n, generator=g, dtype=torch.float64))
    return q.T.contiguous()


def _unit_rows(g: torch.Generator, n: int, D: int) -> torch.Tensor:
    return torch.nn.functional.normalize(torch.randn(n, D, generator=g, dtype=torch.float64), dim=1)


def _clusters(n: int, K: int) -> torch.Tensor:
    """Contiguous cluster ranges of a chunk of n rows."""
    return (torch.arange(n) * K) // max(n, 1)


def make_batch(regime: Regime, Bs: Sequence[int], Ks: Sequence[int], D: int, seed: int, mode: str = "pos",
               dtype: torch.dtype = torch.bfloat16):
    """A W-rank batch: images [B_r, D] and texts [B_r + K_r, D] per rank (paired texts first, then K_r extras), unit rows
    rounded to `dtype` (bf16-representable by default; fp32 for the fp32-input path). mode as in the sample-weight
    tests: pos (positional labels), ids (duplicated sample ids: a twin takes its original's id), hn (hard-negative
    extras: captions of images of their cluster, never positive), extra (extras with ids: most carry the id of the image
    they caption). Returns (imgs, texts, ids, eids); ids / eids are None for pos."""
    g = torch.Generator().manual_seed(seed)
    t, K = regime.t, regime.clusters
    W = len(Bs)
    s_same = (regime.neg_z - regime.design_bias) / t          # image . text of a negative pair inside a cluster
    p = (regime.pos_z[1] - regime.neg_z) / t                  # weight of the pair vector
    rho_lo = (regime.pos_z[0] - regime.neg_z) / (regime.pos_z[1] - regime.neg_z)
    rest = 1.0 - p - regime.noise
    a, gap = (rest + s_same) / 2, (rest - s_same) / 2           # cluster weight, modality gap
    assert min(p, rest, a, gap) >= 0.0, f"regime {regime.name} cannot be built: p={p} a={a} gap={gap}"
    q = (regime.generic_z - regime.neg_z) / t                 # weight of the generic direction
    basis = _orthonormal(g, 2 * K + 1, D)
    modality = basis[0]
    f = basis[1:K + 1]
    generic_dir = basis[K + 1:]
    centroids = (f - f.mean(0, keepdim=True)) * math.sqrt(K / (K - 1)) if K > 1 else f

    # samples: every rank's images in order; the pair vector, cluster and id of each
    n_all = sum(Bs)
    offs = np.concatenate([[0], np.cumsum(Bs)])
    cl = torch.cat([_clusters(b, K) for b in Bs])
    u = _unit_rows(g, n_all, D)
    sid = torch.arange(n_all, dtype=torch.int64)
    for i in range(n_all):
        if float(torch.rand(1, generator=g)) < regime.twins:
            earlier = torch.nonzero(cl[:i] == cl[i]).flatten()
            if len(earlier):
                j = int(earlier[torch.randint(len(earlier), (1,), generator=g)])
                fresh = _unit_rows(g, 1, D)[0]
                u[i] = torch.nn.functional.normalize(0.9 * u[j] + math.sqrt(1 - 0.81) * fresh, dim=0)
                sid[i] = sid[j]
    rho = rho_lo + (1 - rho_lo) * torch.rand(n_all, generator=g, dtype=torch.float64)
    gen = (torch.rand(n_all, generator=g) < regime.generic).double()

    def embed(sign, clus, pair, generic):
        # a generic sample's extra component comes on top of the others (the normalisation shrinks them by 1 + q)
        n = pair.shape[0]
        x = (sign * math.sqrt(gap) * modality + math.sqrt(a) * centroids[clus] + math.sqrt(p) * pair
             + math.sqrt(regime.noise) * _unit_rows(g, n, D) + math.sqrt(q) * generic[:, None] * generic_dir[clus])
        return torch.nn.functional.normalize(x, dim=1).to(dtype)

    imgs, texts, eids = [], [], []
    for r in range(W):
        rows = slice(int(offs[r]), int(offs[r + 1]))
        imgs.append(embed(1.0, cl[rows], u[rows], gen[rows]))
    for c in range(W):
        rows = slice(int(offs[c]), int(offs[c + 1]))
        r = rho[rows][:, None]
        cap = r * u[rows] + torch.sqrt(1 - r * r) * _unit_rows(g, Bs[c], D)
        parts = [embed(-1.0, cl[rows], torch.nn.functional.normalize(cap, dim=1), gen[rows])]
        e_ids = torch.empty(0, dtype=torch.int64)
        if Ks[c]:
            # extras: contiguous clusters too; each captions a random image of its cluster (any rank)
            ecl = _clusters(Ks[c], K)
            src = torch.stack([torch.nonzero(cl == k).flatten()[torch.randint(int((cl == k).sum()), (1,), generator=g)][0]
                               for k in ecl.tolist()])
            er = (rho_lo + (1 - rho_lo) * torch.rand(Ks[c], generator=g, dtype=torch.float64))[:, None]
            ecap = er * u[src] + torch.sqrt(1 - er * er) * _unit_rows(g, Ks[c], D)
            parts.append(embed(-1.0, ecl, torch.nn.functional.normalize(ecap, dim=1), gen[src]))
            # with ids, 80 % are positives of the image they caption (and its twins), the rest carry a fresh id
            fresh = torch.rand(Ks[c], generator=g) >= 0.8
            e_ids = torch.where(fresh, n_all + torch.arange(Ks[c]) + 10 * n_all * (c + 1), sid[src])
        texts.append(torch.cat(parts))
        eids.append(e_ids)
    if mode == "pos":
        return imgs, texts, None, None
    ids = [sid[int(offs[r]):int(offs[r + 1])].clone() for r in range(W)]
    return imgs, texts, ids, eids


def cold_batch(Bs: Sequence[int], Ks: Sequence[int], D: int, seed: int, mode: str = "pos"):
    """The suite's usual inputs (independent random unit embeddings, random ids), for t = 10, b = -10."""
    g = torch.Generator().manual_seed(seed)
    unit = (lambda n: torch.nn.functional.normalize(torch.randn(n, D, generator=g)).to(torch.bfloat16))  # noqa: E731
    imgs = [unit(b) for b in Bs]
    texts = [unit(b + k) for b, k in zip(Bs, Ks)]
    if mode == "pos":
        return imgs, texts, None, None
    ids = list(torch.split(torch.randint(0, max(Bs), (sum(Bs),), generator=g), list(Bs)))
    eids = [torch.randint(0, 2 * max(Bs), (k,), generator=g) for k in Ks]
    return imgs, texts, ids, eids


def random_weights(g: torch.Generator, n: int) -> torch.Tensor:
    """Weights in [0, 1] with 10 % exact zeros and 10 % exact ones (the sample-weight tests' pattern)."""
    w = torch.rand(n, generator=g)
    w[torch.rand(n, generator=g) < 0.1] = 0.0
    w[torch.rand(n, generator=g) < 0.1] = 1.0
    return w


def _f64(xs):
    return None if xs is None else [np.asarray(torch.as_tensor(x).double().numpy()) for x in xs]


def pair_terms(imgs, texts, t_prime: float, bias: float, iws=None, tws=None, labels=None):
    """Per rank r and chunk c: s [B_r, T_c], G [B_r, T_c] (as closed_form_weighted defines it) and the labels.
    labels: as label_blocks returns (default positional)."""
    from sample_weights_oracle import label_blocks

    t = math.exp(t_prime)
    I, T = _f64(imgs), _f64(texts)
    A, C = _f64(iws), _f64(tws)
    if labels is None:
        labels = label_blocks([x.shape[0] for x in I], [x.shape[0] for x in T])
    out = []
    for r, img in enumerate(I):
        row = []
        for c, txt in enumerate(T):
            s = img @ txt.T
            y = labels[r][c]
            w = np.ones_like(s)
            if A is not None:
                w = w * A[r][:, None]
            if C is not None:
                w = w * C[c][None, :]
            G = w * (-y * _sigmoid(-y * (t * s + bias))) / img.shape[0]
            row.append(dict(s=s, G=G, y=y))
        out.append(row)
    return out


def scalar_scales(imgs, texts, t_prime: float, bias: float, iws=None, tws=None, labels=None) -> List[Dict[str, float]]:
    """Per rank: the scales the scalar gradients are measured against, sum |G_ij| for dbias = sum G_ij and
    t sum |G_ij s_ij| for dt' = t sum G_ij s_ij. Near a stationary bias those sums cancel, so an error relative to
    their value means nothing; relative to these scales it is the error of the terms."""
    t = math.exp(t_prime)
    out = []
    for row in pair_terms(imgs, texts, t_prime, bias, iws, tws, labels):
        out.append(dict(dbias=float(sum(np.abs(x["G"]).sum() for x in row)),
                        dt_prime=float(t * sum(np.abs(x["G"] * x["s"]).sum() for x in row))))
    return out


def stationary_bias(imgs, texts, t_prime: float, iws=None, tws=None, labels=None, lo=-200.0, hi=200.0) -> float:
    """The bias at which sum over ranks and pairs of G_ij is 0 (where a learnt bias converges). sum G is increasing in
    the bias (sigma(z) of a negative and -sigma(-z) of a positive both grow with z), so brentq brackets one root."""
    from scipy.optimize import brentq

    t = math.exp(t_prime)
    from sample_weights_oracle import label_blocks

    I, T = _f64(imgs), _f64(texts)
    A, C = _f64(iws), _f64(tws)
    if labels is None:
        labels = label_blocks([x.shape[0] for x in I], [x.shape[0] for x in T])
    terms = []
    for r, img in enumerate(I):
        for c, txt in enumerate(T):
            w = np.ones((img.shape[0], txt.shape[0]))
            if A is not None:
                w = w * A[r][:, None]
            if C is not None:
                w = w * C[c][None, :]
            y = labels[r][c]
            keep = w != 0
            terms.append(((t * (img @ txt.T))[keep], y[keep], w[keep] / img.shape[0]))

    def total(b):
        return sum(float((w * (-y * _sigmoid(-y * (ts + b)))).sum()) for ts, y, w in terms)

    return float(brentq(total, lo, hi, xtol=1e-14, rtol=4 * np.finfo(float).eps, maxiter=500))


def split_own_diagonal(imgs, texts, t_prime: float, bias: float, iws=None, tws=None, labels=None):
    """Per rank r: the part of the own chunk's gradients that the gradient kernel adds in fp32 from g_diag — the own
    positional diagonal, dimg_i = t g_ii txt_i and contrib_i = t g_ii img_i for i < B_r — and everything else, which
    reaches dimg / the own contribution only through the 16-bit sigma operand G. Returns per rank dict(diag_dimg,
    rest_dimg, diag_contrib, rest_contrib) ([T_r, D] contributions: the extras have no diagonal term). The two parts are
    computed independently; diag + rest is the oracle's dimg / contrib[r]."""
    t = math.exp(t_prime)
    I, T = _f64(imgs), _f64(texts)
    terms = pair_terms(imgs, texts, t_prime, bias, iws, tws, labels)
    out = []
    for r, img in enumerate(I):
        txt = T[r]
        br = img.shape[0]
        G = terms[r][r]["G"].copy()
        gd = np.diagonal(G[:, :br]).copy()
        G[np.arange(br), np.arange(br)] = 0.0
        rest_dimg = t * (G @ txt)
        for c in range(len(T)):
            if c != r:
                rest_dimg += t * (terms[r][c]["G"] @ T[c])
        diag_contrib = np.zeros_like(txt)
        diag_contrib[:br] = t * gd[:, None] * img
        out.append(dict(diag_dimg=t * gd[:, None] * txt[:br], rest_dimg=rest_dimg, diag_contrib=diag_contrib,
                        rest_contrib=t * (G.T @ img)))
    return out


def slab_fast_fraction(imgs, texts, t_prime: float, bias: float, labels=None) -> Tuple[float, int]:
    """Fraction of the 16x32 slabs (kernel geometry: 16-row bands x 32 columns of each rank-by-chunk block) whose max z
    is below kFastZ, i.e. that take the series path, among the slabs whose path depends on z at all: slabs touching the
    own diagonal, crossing the border of the block, or holding a positive pair take the label-applying path whatever z
    is and are left out (tests/slab_paths.py's free slabs). Returns (fraction, number of slabs counted)."""
    from slab_paths import FREE, slab_map

    fast = total = 0
    for r, row in enumerate(pair_terms(imgs, texts, t_prime, bias, labels=labels)):
        for c, x in enumerate(row):
            m = slab_map(x["s"], x["y"], r == c, t_prime, bias)
            free = m.cls == FREE
            total += int(free.sum())
            fast += int((free & m.series).sum())
    return fast / max(total, 1), total


def logit_stats(imgs, texts, t_prime: float, bias: float, labels=None) -> Dict[str, float]:
    """Float64 logit statistics of a batch: quantiles of the positive z, the share of negatives above z = 0 and the
    share of negatives with sigma below SIGMA_NORMAL_MIN."""
    t = math.exp(t_prime)
    pos, neg = [], []
    for row in pair_terms(imgs, texts, t_prime, bias, labels=labels):
        for x in row:
            z = t * x["s"] + bias
            pos.append(z[x["y"] > 0])
            neg.append(z[x["y"] < 0])
    pos, neg = np.concatenate(pos), np.concatenate(neg)
    return dict(pos_q05=float(np.quantile(pos, 0.05)), pos_q95=float(np.quantile(pos, 0.95)),
                pos_min=float(pos.min()), pos_max=float(pos.max()), neg_above_0=float((neg > 0).mean()),
                neg_subnormal=float((_sigmoid(neg) < SIGMA_NORMAL_MIN).mean()), neg_max=float(neg.max()))


def negative_share(imgs, texts, t_prime: float, bias: float, iws=None, tws=None, labels=None) -> float:
    """||rest of dimg|| / ||dimg|| over all ranks: the share of the image gradient's norm that passes through G."""
    from sample_weights_oracle import closed_form_weighted

    ref = closed_form_weighted(_f64(imgs), _f64(texts), t_prime, bias, _f64(iws), _f64(tws), labels)
    parts = split_own_diagonal(imgs, texts, t_prime, bias, iws, tws, labels)
    rest = math.sqrt(sum(float(np.square(p["rest_dimg"]).sum()) for p in parts))
    full = math.sqrt(sum(float(np.square(x["dimg"]).sum()) for x in ref))
    return rest / full
