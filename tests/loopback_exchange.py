"""What the loopback stand-ins move between "ranks", restated from the host code, and the table of cells that runs it.

A loopback context (siglip_debug_loopback) plays one rank of a W-rank job on one GPU. The other ranks' published chunks
(text, ids, groups, label sets, weights, teacher text) sit in a stand-in of their exported allocation, from where the
step's pulls copy them into the gathered buffers the kernels read; their contributions to this rank's text gradient
sit in one block per peer, which the step's folds add into dtxt. This module restates, as plain functions of a cell:
  * folds: every read of a peer's contribution block (backward_impl, fused_impl): the split backward's in-kernel folds
    at j = 2..W (the first without a second source), its reduce-slots variant (SIGLIP_OPT_OVERLAP_REDUCE = 0), the
    fused step's remote-chunk folds at k >= 2 and G0's fold, whose second source is own_part under row panels;
  * pulls: every copy of a peer's chunk: the pull job in L(k-1) of the fused step, add_pull_job in the split forward,
    and the stream copies of SIGLIP_OPT_OVERLAP_PULL = 0, each with the kinds the cell's options move;
  * seeds: each peer's contribution, dyadic values on a coarse grid (exact in fp32 in any summation order);
  * sensitivity: what each host-side exchange bug would move a checked output by, on the oracle.
The data is option_matrix's planted data and the oracle its composed one; the gradients scale with grad_out.
tests/test_loopback_exchange_cpu.py derives coverage and sensitivity from it, tests/test_gpu_loopback_exchange.py
runs the cells on the device.
"""
from __future__ import annotations

import dataclasses
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import numpy as np

import grad_matrix as gm
import option_matrix as om

TOL = om.TOL
GRAD_OUT = 0.75      # every cell runs with an upstream gradient g != 1: a fold scaled by g again is then visible
SENSITIVITY = 20.0   # each mutation must move a checked output by more than this many tolerances


def offset(k: int, bidir: bool) -> int:
    """step_offset (csrc/siglip_capi.cu); chunk_schedule in loss.py lists (rank + offset(k)) % W."""
    if not bidir:
        return k
    return (k + 1) // 2 if (k & 1) else -(k // 2)


@dataclass(frozen=True)
class XCell:
    """An option-matrix cell (options, W, rank, schedule, panels, INPUT_F16, tiles) and the exchange options: pull
    (SIGLIP_OPT_OVERLAP_PULL), reduce (SIGLIP_OPT_OVERLAP_REDUCE), sync (SIGLIP_OPT_INKERNEL_SYNC), bf16 (GRAD_BF16)."""
    base: om.Cell
    pull: bool = True
    reduce: bool = True
    sync: bool = True
    bf16: bool = False

    @property
    def name(self) -> str:
        c, o = self.base, self.base.opts
        on = [k for k in ("ids", "xt_ids", "weights", "groups", "teacher") if getattr(o, k)]
        on += [f"M{o.labels}"] if o.labels else []
        on += ["xt"] if o.xtexts else []
        on += ["xi"] if o.ximages else []
        return (f"W{c.W}r{c.r}-{c.sched}{'-bidir' if c.bidir else ''}{'-panels' if c.panels else ''}"
                f"{'-f16' if c.f16 else ''}{'-bf16' if self.bf16 else ''}{'' if self.pull else '-nopull'}"
                f"{'' if self.reduce else '-noreduce'}{'' if self.sync else '-nosync'}-{'+'.join(on) or 'plain'}")

    def step_seed(self, step: int) -> om.Cell:
        """The cell with the seed of step `step`'s planted data: fresh data of every kind at every step."""
        return dataclasses.replace(self.base, seed=self.base.seed + 1000 * step)


def owner(c: om.Cell, k: int) -> int:
    return (c.r + offset(k, c.bidir)) % c.W


# ---------------------------------------------------------------------------------------------------------------------
# fold sites
# ---------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Fold:
    site: str               # where the read happens
    peer: int               # whose block it reads
    src2: Optional[str]     # the fold's second source: None, "acc" (dtxt_acc) or "own_part"; "slots" for the reduction


def folds(x: XCell) -> List[Fold]:
    """Every read of a peer's contribution block in the cell's step, in launch order."""
    c = x.base
    W, r = c.W, c.r
    if W == 1 or c.sched == "fwd":
        return []
    # slot j's fold reads the peer whose step j - 1 scored my chunk
    peer = [None, None] + [(r - offset(j - 1, c.bidir)) % W for j in range(2, W + 1)]
    if c.sched == "split":
        if not x.reduce:
            return [Fold("split.reduce", p, "slots") for p in range(W) if p != r]
        return [Fold("split.fold.first" if j == 2 else "split.fold.chain", peer[j], None if j == 2 else "acc")
                for j in range(2, W + 1)]
    own = "own_part" if c.panels else None
    out = [Fold("fused.fold.remote", peer[j], own if j == 2 else "acc") for j in range(2, W)]
    out.append(Fold(f"fused.G0.W{min(W, 3)}", peer[W], own if W == 2 else "acc"))
    return out


def grad_ctx(x: XCell) -> gm.Ctx:
    """The cell as tests/grad_matrix.py's step, for its launch rules."""
    c = x.base
    Bs, Rs, Ts = c.shapes()
    return gm.Ctx(Bs, Rs, Ts, om.D, r=c.r, cg=c.cg, mcast=c.mcast, f16=c.f16, bf16=x.bf16,
                  budget_mib=c.budget_mib(), sched=c.sched, grad_out=True, overlap_reduce=x.reduce)


# ---------------------------------------------------------------------------------------------------------------------
# pull sites and kinds
# ---------------------------------------------------------------------------------------------------------------------
def pull_site(x: XCell) -> str:
    if x.base.sched == "fused":
        return "fused.L"           # fused_impl: add_pull_job in L(k-1), whatever SIGLIP_OPT_OVERLAP_PULL
    return "split.L" if x.pull else "split.stream"


def kinds(x: XCell) -> List[str]:
    """What every pull of the cell moves (add_pull_job / the stream copies): the text, and with the options the ids
    slot (ids, extra-text ids, groups, label sets), the text weights and the teacher text."""
    c, o = x.base, x.base.opts
    out = ["text.f16" if c.f16 else "text.bf16"]
    if o.ids:
        out.append("ids")
    if o.xt_ids:
        out.append("xt_ids")
    if o.groups:
        out.append("groups")
    if o.labels:
        out.append(f"sets.M{o.labels}")
    if o.weights:
        out.append("weights")
    if o.teacher:
        out.append("teacher.extras" if om.distill_extras_context(c) else "teacher.distill")
    return out


def pulls(x: XCell) -> List[Tuple[str, int]]:
    """(site, chunk) of every pull of the step: the chunk of step k, pulled during step k - 1."""
    c = x.base
    if c.W == 1:
        return []
    return [(pull_site(x), owner(c, k)) for k in range(1, c.W)]


# ---------------------------------------------------------------------------------------------------------------------
# cells
# ---------------------------------------------------------------------------------------------------------------------
def _x(W, r, sched, opts=om.Options(), bidir=False, panels=False, f16=False, **kw) -> XCell:
    return XCell(om.Cell(opts, W, r, bidir, sched, panels, f16, 128, 6, 2, 1, 0), **kw)


def _cells() -> List[XCell]:
    O = om.Options
    cells = []
    hn, xi = O(xtexts=True), O(ximages=True)
    # folds, each site with the first and the last rank, fp32 and bf16 outputs, hard negatives and extra images
    for W in (2, 3):
        last = W - 1
        if W == 2:   # at W = 3 the pull cells below run these two sites from both sides
            cells += [_x(W, 0, "split", hn, bf16=True), _x(W, last, "split", xi, f16=True), _x(W, 0, "fused", xi)]
        cells += [_x(W, 0, "split", xi, reduce=False, pull=False), _x(W, last, "split", hn, f16=True, bf16=True,
                                                                      reduce=False, pull=False),
                  _x(W, last, "fused", hn, f16=True, bf16=True),
                  _x(W, 0, "fused", hn, panels=True, bf16=True), _x(W, last, "fused", xi, panels=True, f16=True),
                  _x(W, 0, "fused", xi, sync=False), _x(W, last, "fused", hn, sync=False, bf16=True)]
    # the bidirectional schedule reads other owners than the ring from W = 4 on
    cells += [_x(4, 0, "split", hn, bidir=True), _x(4, 3, "split", xi, bidir=True, bf16=True),
              _x(4, 0, "fused", xi, bidir=True, bf16=True), _x(4, 3, "fused", hn, bidir=True)]
    # every pulled kind at every pull site: ids with extra-text ids, groups and weights; label sets of 1 and of 4
    # labels (the wider one with groups); a teacher in a distillation context and in a distill-extras one
    kinds_opts = [O(ids=True, xtexts=True, xt_ids=True, groups=True, weights=True),
                  O(labels=1, xtexts=True, xt_sets=True), O(labels=4, groups=True),
                  O(teacher=True), O(teacher=True, xtexts=True, ids=True, xt_ids=True)]
    for site, (sched, pull) in enumerate((("fused", True), ("split", True), ("split", False))):
        for i, o in enumerate(kinds_opts):
            W = 2 + (site + i) % 2
            cells.append(_x(W, (i + site) % W, sched, o, pull=pull, f16=(i + site) % 2 == 1))
    # the tile width, stage count and cluster shape rotate over the cells (the exchange does not depend on them)
    return [dataclasses.replace(x, base=dataclasses.replace(x.base, tile_n=(128, 256)[i % 2], stages=(6, 4)[i // 2 % 2],
                                                            cg=(2, 1)[i // 4 % 2], seed=700 + i))
            for i, x in enumerate(cells)]


CELLS: List[XCell] = _cells()


def coverage(x: XCell) -> set:
    """What a cell reaches: each fold site with the side of the rank (first / last) and, where the bidirectional
    schedule differs from the ring, the schedule; each fold site's output format and shape features; each pull site
    with each kind it moves."""
    c = x.base
    Bs, Rs, Ts = c.shapes()
    side = "first" if c.r == 0 else "last" if c.r == c.W - 1 else "middle"
    out = set()
    for f in folds(x):
        site = f.site + ("" if x.sync else ".nosync") + (".panels" if f.src2 == "own_part" else "")
        # at W = 2 the split backward's one fold is also its last, and its one reduction reads a single peer
        site += ".W2" if c.W == 2 and c.sched == "split" else ""
        out.add(("fold", site, side, "bidir" if c.bidir and c.W >= 4 else "ring"))
        out.add(("fold", site, "bf16" if x.bf16 else "fp32"))
        if Ts[c.r] > Bs[c.r]:
            out.add(("fold", site, "T>B"))
        if Rs[c.r] > Bs[c.r]:
            out.add(("fold", site, "R>B"))
    for site, _ in pulls(x):
        for k in kinds(x):
            out.add(("pull", site, k))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# seeds and expected values
# ---------------------------------------------------------------------------------------------------------------------
def seeds(x: XCell, own: np.ndarray, step: int) -> Dict[int, np.ndarray]:
    """Each peer's seeded contribution [T_r, D]: integers in [-15, 15] times a power of two near max |own| / 16,
    distinct per peer, row and step; any sum of them is exact in fp32."""
    c = x.base
    scale = 2.0 ** np.round(np.log2(np.abs(own).max() / 16.0))
    i = np.arange(own.shape[0])[:, None]
    d = np.arange(own.shape[1])[None, :]
    return {p: (((11 * p + 3 * i + 5 * d + 7 * step) % 31) - 15) * scale for p in range(c.W) if p != c.r}


def problem(x: XCell, step: int) -> om.Problem:
    return om.planted(x.step_seed(step))


def references(x: XCell, P: om.Problem, g: float = GRAD_OUT) -> Dict:
    """Rank r's checked outputs for upstream gradient g: loss, dimg, contrib[c], dt_prime, dbias."""
    res = om.oracle(P, x.base.opts)[x.base.r]
    return dict(loss=res["loss"], dimg=g * res["dimg"], contrib=[g * a for a in res["contrib"]],
                dt_prime=g * res["dt_prime"], dbias=g * res["dbias"])


def rel(a, b) -> float:
    return om.rel(a, b)


# ---------------------------------------------------------------------------------------------------------------------
# sensitivity
# ---------------------------------------------------------------------------------------------------------------------
def fold_mutations(x: XCell, own: np.ndarray, C: Dict[int, np.ndarray], g: float = GRAD_OUT) -> Dict[str, float]:
    """The relative change of the checked dtxt - sum C (against g own) under each host-side fold bug: one peer's block
    dropped, taken from another peer's block, read one row on, cut at another chunk's T (the chunks with fewer texts),
    and the folded sum scaled by g. A mutation that cannot occur in the cell (one peer, no shorter chunk) is absent."""
    c = x.base
    Bs, Rs, Ts = c.shapes()
    T = Ts[c.r]
    out = {}
    total = sum(C.values())
    for p, blk in C.items():
        out[f"drop peer {p}"] = rel(own - blk, own)
        for q in C:
            if q != p:
                out[f"peer {q}'s block for {p}'s"] = rel(own + C[q] - blk, own)
        shifted = np.zeros_like(blk)
        shifted[:-1] = blk[1:]
        out[f"peer {p} rows shifted"] = rel(own + shifted - blk, own)
        for k in sorted({t for t in Ts if t < T}):
            cut = blk.copy()
            cut[k:] = 0.0
            out[f"peer {p} cut at T = {k}"] = rel(own + cut - blk, own)
    out["folded sum scaled by g"] = rel(own + (g - 1.0) * total, own)
    return out


KIND_FIELDS = {"text.bf16": ("txts",), "text.f16": ("txts",), "ids": ("ids",), "xt_ids": ("xt_ids",),
               "groups": ("tg",), "weights": ("tw",), "teacher.distill": ("ttxts",), "teacher.extras": ("ttxts",)}


def stale(P: om.Problem, prev: om.Problem, kind: str, chunk: int) -> om.Problem:
    """P with one pulled kind of one chunk left at the previous step's values (what a pull that did not run, or ran
    short, leaves in the gathered buffer). Label sets are the sets of chunk `chunk`'s texts: its text tags and ids."""
    fields = ("ttags", "ids", "xt_ids") if kind.startswith("sets") else KIND_FIELDS[kind]
    Q = dataclasses.replace(P, **{f: list(getattr(P, f)) for f in fields})
    for f in fields:
        getattr(Q, f)[chunk] = getattr(prev, f)[chunk]
    return Q


def checked_change(x: XCell, a: Dict, b: Dict) -> float:
    """The largest relative change over the outputs the GPU test checks: loss, dimg, every contribution, dt', dbias."""
    c = x.base
    vals = [rel(a["loss"], b["loss"])]
    if c.sched != "fwd":
        vals += [rel(a["dimg"], b["dimg"]), rel(a["dt_prime"], b["dt_prime"]), rel(a["dbias"], b["dbias"])]
        vals += [rel(u, v) for u, v in zip(a["contrib"], b["contrib"])]
    return max(vals)


def pull_mutations(x: XCell, prev: om.Problem, P: om.Problem, ref: Dict) -> Dict[str, float]:
    """The largest relative change of a checked output when one kind of one pulled chunk is the previous step's."""
    Bs, _, Ts = x.base.shapes()
    out = {}
    for _, chunk in pulls(x):
        for kind in kinds(x):
            if kind == "xt_ids" and Ts[chunk] == Bs[chunk]:
                continue   # a chunk without extra texts has no extra-text ids
            # the own-side half of a kind (a chunk's paired ids are also its images' ids) plays no part in rank r's
            # outputs: only the pulled chunk's texts are stale
            out[f"{kind} of chunk {chunk}"] = checked_change(x, references(x, stale(P, prev, kind, chunk)), ref)
    return out
