"""The loss step's options in combination: a table of cells and a composed float64 oracle — test infrastructure, never
the product path.

Every cell turns on a set of options (sample ids or label sets, extra texts / images with or without ids or sets,
weights, excluded groups, the focal terms or a teacher, per-sample losses, metrics, top-K) and picks the engine
configuration it runs under (W, bidir, schedule, row panels, INPUT_F16, gradient tile width, stages, cluster shape).
``route`` restates how ``launch_gemm`` picks the loss kernel for each launch of the step, so the table's coverage of
kernel instantiations and runtime branches is derived, not claimed. ``oracle`` composes the single-feature oracles (no
new loss math); ``retrieval`` and ``peer_stand_ins`` give the exact retrieval results and what the loopback hooks need to
stand in for the other ranks.

Planted data: every embedding entry is a small integer / 8, so the bf16 and fp16(16 x) operands are exact and every fp32
logit equals its float64 value; retrieval is compared exactly. Samples are integer cluster centres (one per group) plus
an integer vector per sample id plus sparse noise: duplicate ids are near-duplicates, captions and extras lie near their
image, and same-group negatives have sigma(z) ~ 0.12 at t = 5, bias = -6 (against ~0.003 for the other negatives), so
the excluded pairs carry weight while a flipped label still moves a step's loss by more than 20x the tolerance. A label
set holds the sample's id and a few tags of a small pool (not the groups: a positive is never excluded). The teacher's
rows are an integer vector per teacher key plus sparse noise, the key being the id except that ids 2k + 1 share 2k's:
at t_T = 6, b_T = -10 its p is ~0.97 on the pairs with one key and ~1e-4 elsewhere, a sharp teacher (a low entropy
floor under the loss) that knows matches the labels do not.

That data never votes the loss epilogue's series path (every free slab holds some z above kFastZ). COLD runs the same
rows on planted_cold's data, where most slabs do (tests/slab_paths.py models each slab's path; cell_slabs applies it)."""
from __future__ import annotations

import dataclasses
import itertools
import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import numpy as np

from distill_options_oracle import closed_form_distill_options
from exclude_groups_oracle import closed_form_groups, group_labels, text_loss_of
from extra_images_oracle import label_blocks
from focal_oracle import closed_form_focal
from label_sets_oracle import set_labels, topk_retrieval_sets
from retrieval_metrics_oracle import key_as_int64, metric_key
from retrieval_topk_oracle import recall_counts, topk_retrieval
from sample_losses_oracle import fixed_point_partial

TP, BIAS = math.log(5.0), -6.0
TTP, TBIAS, LAM = math.log(6.0), -10.0, 0.6   # the teacher's t', bias and the distillation weight lambda
TOL = 1e-3
KMAX = 10   # SIGLIP_TOPK_MAX: the width of a peer's seeded top-K column lists
D, DT = 136, 72
N_GROUPS = 10
MMAX = 4    # the widest label set a cell uses
N_TAGS = 40

MODES = ("loss", "sample_loss", "topk", "groups", "distill", "labels", "focal", "distill_opts")
CONTEXTS = ("plain", "hn", "xt", "xi", "xin", "both")
SCHEDS = ("fused", "split", "fwd")
CLUSTERS = {1: [(1, 1)], 2: [(2, 1), (1, 2)], 4: [(2, 2)]}   # cluster size -> (cta_group, mcast)
DISTILL_STAGES = 4   # kDistillStages: both teacher kernels run 4 stages whatever the request
SET_MODES = ("labels", "focal", "distill_opts")   # the modes whose steps can carry label sets
# (gamma, alpha) of the focal cells; gamma 0 without alpha is the plain step
FOCALS = tuple((g, a) for g in (0.5, 2.0, 5.0) for a in (None, 0.25))

# per-rank paired batches, extra texts and extra images of each world size (uneven, ragged past 256 at W = 1); the
# panel cells use larger batches so that a budget of a few MiB splits the rows into several panels
SHAPES = {1: ((300,), (37,), (23,)), 2: ((200, 136), (29, 41), (17, 30)),
          3: ((136, 200, 160), (19, 0, 33), (9, 27, 13)),
          # W = 4: the loopback exchange cells (tests/loopback_exchange.py), where the bidirectional schedule first
          # reads other owners than the ring
          4: ((136, 120, 160, 104), (19, 0, 33, 8), (9, 27, 0, 13))}
PANEL_SHAPES = {1: ((700,), (60,), (48,)), 2: ((600, 520), (40, 72), (24, 36)),
                3: ((520, 456, 600), (8, 40, 0), (36, 12, 20))}
# one rank with more than 960 images and texts: the gradient kernel's split-K splits (launch_impl cuts K into slices of
# at least 8 k-blocks of 64), which the shapes above never reach (the step sequences' split-K steps run these)
SPLIT_SHAPES = {1: ((1040,), (37,), (23,))}
# the multi-tile family (MULTI, MULTI_COLD): every launch over a chunk with its extra texts runs several tiles per
# cluster at every cluster size, on an H100 SXM's co-resident cluster counts (tests/tile_schedule.py). 17 520 texts are
# 137 column blocks, more than the 132 clusters of size 1: consecutive tiles of a cluster keep their row block; 520
# images are 5 row blocks, 3 row panels of 2 blocks (the last one a phantom) and 2 panels of 4 (three phantoms). At W = 2
# the family runs rank 1, whose own chunk is narrow: its launches keep the wide chunk's grid (grid_n) and leave most
# clusters without a tile. D = 136 and D_T = 72 make a tile 3 k-blocks, 5 with the teacher's: a multiple of neither 4
# nor 6 stages.
MULTI_SHAPES = {1: ((520,), (17000,), (40,)), 2: ((520, 520), (17000, 60), (40, 20))}


@dataclass(frozen=True)
class Options:
    """What a step computes. Extra-text / extra-image ids need sample ids, extra-text / extra-image sets need label sets;
    label sets take no ids, and the focal terms no teacher (the documented refusals)."""
    ids: bool = False
    xtexts: bool = False     # extra texts: hard negatives, or with xt_ids / xt_sets further captions
    ximages: bool = False    # extra images: hard negatives, or with xi_ids / xi_sets further images of a caption
    xt_ids: bool = False
    xi_ids: bool = False
    labels: int = 0          # M: label sets of M labels per sample (SIGLIP_OPT_LABEL_SETS), 0: none
    xt_sets: bool = False    # the extra texts carry sets of their own (else the empty sets of hard negatives)
    xi_sets: bool = False
    weights: bool = False
    groups: bool = False
    focal: Optional[Tuple[float, Optional[float]]] = None   # (gamma, alpha) of SIGLIP_OPT_FOCAL
    teacher: bool = False
    metrics: bool = False    # siglip_request_metrics (top-1)
    losses: bool = False     # siglip_request_sample_losses
    topk: int = 0            # siglip_request_topk's K; K = 1 runs the metrics path

    @property
    def context(self) -> str:
        if self.xtexts and self.ximages:
            return "both"
        if self.xtexts:
            return "xt" if (self.xt_ids or self.xt_sets) else "hn"
        if self.ximages:
            return "xi" if (self.xi_ids or self.xi_sets) else "xin"
        return "plain"

    @property
    def keys(self) -> bool:
        """The step reduces argmax keys (row_keys): a metrics request or a K = 1 top-K request."""
        return self.metrics or self.topk == 1

    def valid(self) -> bool:
        if (self.xt_ids and not (self.ids and self.xtexts)) or (self.xi_ids and not (self.ids and self.ximages)):
            return False
        if (self.xt_sets and not (self.labels and self.xtexts)) or (self.xi_sets and not (self.labels and
                                                                                           self.ximages)):
            return False
        if not 0 <= self.labels <= MMAX or (self.labels and self.ids):
            return False
        return not (self.focal is not None and self.teacher)

    def removals(self) -> Dict[str, "Options"]:
        """Each option this step turns on that changes its labels, weights or targets, switched off on its own (with
        what depends on it: ids take the extras' ids along, label sets the extras' sets)."""
        r = dataclasses.replace
        out = {}
        if self.xtexts:
            out["extra texts"] = r(self, xtexts=False, xt_ids=False, xt_sets=False)
        if self.ximages:
            out["extra images"] = r(self, ximages=False, xi_ids=False, xi_sets=False)
        if self.ids:
            out["ids"] = r(self, ids=False, xt_ids=False, xi_ids=False)
        if self.xt_ids:
            out["extra text ids"] = r(self, xt_ids=False)
        if self.xi_ids:
            out["extra image ids"] = r(self, xi_ids=False)
        if self.labels:
            out["label sets"] = r(self, labels=0, xt_sets=False, xi_sets=False)
        if self.xt_sets:
            out["extra text sets"] = r(self, xt_sets=False)
        if self.xi_sets:
            out["extra image sets"] = r(self, xi_sets=False)
        if self.weights:
            out["weights"] = r(self, weights=False)
        if self.groups:
            out["groups"] = r(self, groups=False)
        if self.focal is not None:
            out["focal"] = r(self, focal=None)
        if self.teacher:
            out["teacher"] = r(self, teacher=False)
        return out


@dataclass(frozen=True)
class Cell:
    opts: Options
    W: int
    r: int
    bidir: bool
    sched: str
    panels: bool
    f16: bool
    tile_n: int
    stages: int
    cg: int
    mcast: int
    seed: int
    cold: bool = False   # planted_cold's data: the series path's family
    splitk: bool = False  # SPLIT_SHAPES instead of SHAPES / PANEL_SHAPES
    multi: bool = False   # MULTI_SHAPES: the multi-tile family

    @property
    def mode(self) -> str:
        return mode_of(self.opts)

    @property
    def cluster(self) -> int:
        return self.cg * self.mcast

    @property
    def name(self) -> str:
        o = self.opts
        on = [k for k in ("ids", "xt_ids", "xi_ids", "xt_sets", "xi_sets", "weights", "groups", "teacher", "metrics",
                          "losses") if getattr(o, k)]
        on += [f"M{o.labels}"] if o.labels else []
        on += [f"g{o.focal[0]:g}" + (f"a{o.focal[1]:g}" if o.focal[1] is not None else "")] if o.focal else []
        on += [f"k{o.topk}"] if o.topk else []
        return (f"{self.seed:03d}-{self.mode}-{o.context}-{'+'.join(on) or 'none'}-W{self.W}r{self.r}"
                f"{'-bidir' if self.bidir else ''}-{self.sched}{'-panels' if self.panels else ''}"
                f"{'-f16' if self.f16 else ''}-t{self.tile_n}-s{self.stages}-cg{self.cg}m{self.mcast}"
                f"{'-cold' if self.cold else ''}{'-splitk' if self.splitk else ''}{'-multi' if self.multi else ''}")

    def shapes(self):
        """(Bs, Rs, Ts) of every rank, as the step sees them."""
        Bs, K, E = shape_table(self)[self.W]
        Ts = tuple(b + (k if self.opts.xtexts else 0) for b, k in zip(Bs, K))
        Rs = tuple(b + (e if self.opts.ximages else 0) for b, e in zip(Bs, E))
        return Bs, Rs, Ts

    def budget_mib(self, cluster: Optional[int] = None) -> int:
        """The smallest SIGLIP_OPT_SIGMA_BUDGET_MIB that runs the fused step in more than one row panel (0: no panels),
        for the cell's cluster size or another one (siglip_ctx_sigma_panels: panels of whole 128-row cluster blocks)."""
        if not self.panels:
            return 0
        Bs, Rs, Ts = self.shapes()
        rp, tp = _round_up(max(Rs), 256), _round_up(max(Ts), 256)
        nbuf, unit = (2 if self.W > 1 else 1), 128 * (cluster or self.cluster)
        for mib in range(1, 64):
            rows = mib * 2 ** 20 // (nbuf * tp * 2) // unit * unit
            if rows and rp * nbuf * tp * 2 > mib * 2 ** 20 and Rs[self.r] > rows:
                return mib
        raise AssertionError(f"{self.name}: no budget splits the rows into panels")

    def panel_rows(self) -> int:
        """The rows of the step's panels under budget_mib() (sigma_panels): all R_r rows without panels."""
        Bs, Rs, Ts = self.shapes()
        if not self.panels:
            return Rs[self.r]
        unit = 128 * self.cluster
        P = self.budget_mib() * 2 ** 20 // ((2 if self.W > 1 else 1) * _round_up(max(Ts), 256) * 2) // unit * unit
        return min(P, Rs[self.r])


def shape_table(cell: Cell):
    return MULTI_SHAPES if cell.multi else SPLIT_SHAPES if cell.splitk else PANEL_SHAPES if cell.panels else SHAPES


def _round_up(x, m):
    return (x + m - 1) // m * m


def mode_of(o: Options) -> str:
    """The loss kernel launch_gemm selects (csrc/siglip_kernels.cu): a teacher with per-sample losses, top-K (K > 1),
    groups or label sets runs kModeDistillOpts, any other teacher kModeDistill; then the focal terms, label sets, groups,
    top-K, per-sample losses, and otherwise the plain loss kernel."""
    if o.teacher:
        return "distill_opts" if (o.losses or o.topk > 1 or o.groups or o.labels) else "distill"
    if o.focal is not None:
        return "focal"
    if o.labels:
        return "labels"
    if o.groups:
        return "groups"
    if o.topk > 1:
        return "topk"
    if o.losses:
        return "sample_loss"
    return "loss"


def route(cell: Cell):
    """The loss-kernel launches of the cell's step, one per text chunk: (instantiation, runtime options) pairs.
    An instantiation is (mode, stages, cluster size[, ids, metrics, weights]) — kModeLoss compiles its three options in,
    the other modes take them at run time. ids is on for a chunk whose labels come from ids: True for every chunk with
    sample ids, "iota" for the own chunk of a rank that holds extras of both kinds (run_loss_chunk's own_pos_ids: the
    positional pairs as iota ids, the same branch fed differently; under label sets the label-set pre-pass folds them into
    the positives). sets is on for every chunk of a label-set step. A teacher step also records the context it runs in
    (distill_extras_context): the distill-extras workspace puts the gathered teacher text, and what follows it, at other
    offsets, so the same kModeDistill branch reads different addresses there."""
    return {chunk_route(cell, c) for c in range(cell.W)}


def own_pos_ids(cell: Cell) -> bool:
    """The rank holds extras of both kinds: its own chunk takes its positional positives from iota ids."""
    Bs, Rs, Ts = cell.shapes()
    return Rs[cell.r] > Bs[cell.r] and Ts[cell.r] > Bs[cell.r]


def chunk_route(cell: Cell, c: int):
    """The (instantiation, runtime options) of the loss launches over text chunk c (route)."""
    o = cell.opts
    mode = mode_of(o)
    stages = DISTILL_STAGES if mode in ("distill", "distill_opts") else cell.stages
    ids = True if o.ids else ("iota" if c == cell.r and own_pos_ids(cell) else False)
    if mode == "loss":
        return (mode, stages, cell.cluster, ids, o.keys, o.weights), ()
    rt = dict(ids=ids, weights=o.weights, metrics=o.keys)
    if mode in ("topk", "groups") + SET_MODES:
        rt["losses"] = o.losses
    if mode in ("groups",) + SET_MODES:
        rt["topk"] = o.topk > 1
    if mode in SET_MODES:
        rt["groups"] = o.groups
    if mode in ("focal", "distill_opts"):
        rt["sets"] = bool(o.labels)
    if o.teacher:
        rt["extras_ctx"] = distill_extras_context(cell)
    return (mode, stages, cell.cluster), tuple(sorted(rt.items()))


def distill_extras_context(cell: Cell) -> bool:
    """A teacher cell runs in a siglip_ctx_create_distill_extras context (distill_options=True) when it has extras or
    kModeDistillOpts's options, and in a siglip_ctx_create_distill one otherwise."""
    Bs, Rs, Ts = cell.shapes()
    return cell.opts.teacher and (Rs != Bs or Ts != Bs or cell.mode == "distill_opts")


def runtime_options(mode: str) -> List[str]:
    """The runtime options a mode's kernel branches on. The label source of kModeFocal and kModeDistillOpts is ids or
    sets (positions: neither); kModeLabels always has sets, and its iota ids are part of them."""
    return {"loss": [], "sample_loss": ["ids", "metrics", "weights"], "topk": ["ids", "losses", "metrics", "weights"],
            "groups": ["ids", "losses", "metrics", "topk", "weights"],
            "labels": ["groups", "losses", "metrics", "topk", "weights"],
            "focal": ["groups", "ids", "losses", "metrics", "sets", "topk", "weights"],
            "distill": ["ids", "metrics", "weights"],
            "distill_opts": ["groups", "ids", "losses", "metrics", "sets", "topk", "weights"]}[mode]


def runtime_combos(mode: str) -> List[Dict[str, bool]]:
    """Every combination of the mode's runtime options a step can reach: no ids with sets, and a teacher step without
    sets, groups, per-sample losses and top-K runs kModeDistill instead."""
    names = runtime_options(mode)
    out = []
    for v in itertools.product((False, True), repeat=len(names)):
        f = dict(zip(names, v))
        if f.get("ids") and f.get("sets"):
            continue
        if mode == "distill_opts" and not (f["sets"] or f["groups"] or f["losses"] or f["topk"]):
            continue
        out.append(f)
    return out


def instantiations(mode: str):
    """Every loss-kernel instantiation launch_gemm can select for a mode."""
    if mode in ("distill", "distill_opts"):
        return {(mode, DISTILL_STAGES, cs) for cs in CLUSTERS}
    base = {(mode, st, cs) for st in (4, 6) for cs in CLUSTERS}
    if mode != "loss":
        return base
    return {b + f for b in base for f in itertools.product((False, True), repeat=3)}


def axis_values(mode: str) -> Dict[str, tuple]:
    """The values of every other axis a mode can be paired with: the set width M for the modes that carry sets, and
    (gamma, alpha) for the focal terms."""
    out = dict(context=CONTEXTS, W=(1, 2, 3), bidir=(False, True), sched=SCHEDS, panels=(False, True),
               f16=(False, True), tile_n=(128, 256), stages=(4, 6), cluster=(1, 2, 4))
    if mode in SET_MODES:
        out["M"] = tuple(range(1, MMAX + 1))
    if mode == "focal":
        out["focal"] = FOCALS
    return out


def axis_of(cell: Cell, axis: str):
    if axis == "context":
        return cell.opts.context
    if axis == "M":
        return cell.opts.labels
    if axis == "focal":
        return cell.opts.focal
    return getattr(cell, axis)


# ---------------------------------------------------------------------------------------------------------------------
# the table
# ---------------------------------------------------------------------------------------------------------------------
def _mode_rows():
    """(mode, runtime options, stages, cluster) of every cell: the 48 kModeLoss instantiations, and for every other mode
    each combination of its runtime options once, cycling through its instantiations. kModeDistill's combinations run
    without extras (the cells the table had before a teacher took extras); one cell per other context follows them."""
    rows = []
    for f in runtime_combos("sample_loss"):   # ids, metrics, weights: kModeLoss's compiled-in options
        for st in (4, 6):
            for cs in (1, 2, 4):
                rows.append(("loss", f, st, cs))
    for mode in MODES[1:]:
        combos = runtime_combos(mode)
        if mode == "distill":
            combos += [dict(ids=True, metrics=k % 2 == 1, weights=k // 2 % 2 == 1) for k in range(len(CONTEXTS) - 1)]
        for i, f in enumerate(combos):
            rows.append((mode, f, (4, 6)[(i // 3) % 2], (1, 2, 4)[i % 3]))
    return rows


def _lru_pick(order, ok):
    """The least recently picked value of `order` that satisfies ok; it moves to the back."""
    v = next(x for x in order if ok(x))
    order.remove(v)
    order.append(v)
    return v


def build_table(cold: bool = False, multi: bool = False) -> List[Cell]:
    """The cells of every row of _mode_rows. cold: the same rows on planted_cold's data (seeds from COLD_SEED), without
    kModeDistill's rows for the other contexts: they run its branches again, and the cold family is the minimal cover of
    the instantiations and runtime combinations. multi: the multi-tile family on MULTI_SHAPES (seeds from MULTI_SEED),
    every cell with extra texts (the wide chunk), at W = 1 and 2 without row panels, and only the rows that add an item
    of multi_items to the rows before them and to the rows after them (the minimal cover of what the tile schedule has
    to reach)."""
    cells, counters = [], {}
    for seed, (mode, f, stages, cs) in enumerate(_mode_rows()):
        j = counters.setdefault(mode, [0, {}])
        i, cyc = j[0], j[1]
        j[0] += 1
        if cold and mode == "distill" and i >= len(runtime_combos(mode)):
            continue
        ids = f.get("ids", False)
        sets = mode == "labels" or f.get("sets", False)
        W = (1, 2)[i // 2 % 2] if multi else (1, 2, 3)[i % 3]
        # xt / xi: extras with ids or sets of their own; both at W = 1 under positional labels would run iota ids only
        # (which the multi-tile family wants of every mode with an ids option: every context of it has the wide chunk's
        # extra texts; a kModeLoss row would run the kIds instantiation instead of its own)
        if multi:
            ctx = _lru_pick(cyc.setdefault("ctx", list(MULTI_CONTEXTS)),
                            lambda c: ids or sets or (c != "xt" and not (c == "both" and W == 1 and mode == "loss")))
        elif mode == "distill":   # its runtime combinations without extras, then every other context once
            ctx = "plain" if i < len(runtime_combos(mode)) else CONTEXTS[1 + i - len(runtime_combos(mode))]
        else:
            ctx = _lru_pick(cyc.setdefault("ctx", list(CONTEXTS)),
                            lambda c: (ids or sets or c not in ("xt", "xi")) and (ids or sets or W > 1 or c != "both"))
        panels = i % 4 == 3 and not multi
        # the loss alone can move by less than 20x the tolerance when a label-set step has extras (the tag positives
        # raise it, the same-id positives lower it, and the extras' pairs are few) or a teacher's step has sets or
        # extras with ids (its soft targets): those cells check gradients too
        own = ctx in ("xt", "xi", "both")
        loss_only = not ((sets and ctx != "plain") or (mode in ("distill", "distill_opts") and (sets or (ids and own))))
        sched = "fused" if panels else _lru_pick(cyc.setdefault("sched", list(SCHEDS)), lambda s: loss_only or s != "fwd")
        cg, mcast = CLUSTERS[cs][(i // 2) % len(CLUSTERS[cs])]
        metrics = f.get("metrics", False)
        M = _lru_pick(cyc.setdefault("M", list(range(1, MMAX + 1))), lambda m: True) if sets else 0
        focal = _lru_pick(cyc.setdefault("focal", list(FOCALS)), lambda x: True) if mode == "focal" else None
        if cold and focal is not None:
            # gamma >= 2 leaves a series slab's terms below 2e-4 of every output and its sigma * 2^14 among fp16's
            # subnormals, where the 16-bit operand, not the path, sets the error: the cold family runs gamma = 0.5
            focal = (0.5, focal[1])
        o = Options(ids=ids, xtexts=ctx in ("hn", "xt", "both"), ximages=ctx in ("xi", "xin", "both"),
                    xt_ids=ids and ctx in ("xt", "both"), xi_ids=ids and ctx in ("xi", "both"),
                    labels=M, xt_sets=sets and ctx in ("xt", "both"), xi_sets=sets and ctx in ("xi", "both"),
                    weights=f.get("weights", False), groups=mode == "groups" or f.get("groups", False),
                    focal=focal, teacher=mode in ("distill", "distill_opts"),
                    # a metrics cell of the modes without a top-K option asks for it as a K = 1 top-K request every
                    # other time: the same keys, a second set of outputs
                    metrics=metrics and not (mode in ("loss", "sample_loss") and i % 2),
                    losses=f.get("losses", False) or mode == "sample_loss",
                    topk=(5 if mode == "topk" else 3 if f.get("topk") else
                          1 if metrics and mode in ("loss", "sample_loss") and i % 2 else 0))
        assert o.valid() and mode_of(o) == mode, o
        cells.append(Cell(o, W, W - 1 if multi else i % W, W > 1 and (i // 3) % 2 == 1, sched, panels, (i + i // 4) % 2 == 1,
                          (128, 256)[(i // 2 + i // 8) % 2], stages, cg, mcast,
                          seed + COLD_SEED * cold + MULTI_SEED * multi, cold, multi=multi))
    if not multi:
        return cells
    items = [multi_items(c) for c in cells]
    keep, seen = [], set()
    for k in range(len(cells)):   # forward: the rows that add something; backward: drop the ones the rest cover
        if items[k] - seen:
            keep.append(k)
            seen |= items[k]
    for k in reversed(list(keep)):
        rest = set().union(*(items[j] for j in keep if j != k))
        if items[k] <= rest:
            keep.remove(k)
    return [cells[k] for k in keep]


COLD_SEED = 500
MULTI_SEED = 1000
MULTI_CONTEXTS = ("hn", "xt", "both")


# ---------------------------------------------------------------------------------------------------------------------
# the tile schedule of a cell's loss launches (tests/tile_schedule.py)
# ---------------------------------------------------------------------------------------------------------------------
def cell_launches(cell: Cell, clusters=None, num_sms: Optional[int] = None):
    """(chunk_route, chunk, window, tile_schedule.Launch) of every loss launch of rank r's step (slab_paths.windows), on
    clusters[(mode, stages, cluster size)] co-resident clusters of each instantiation and num_sms SMs (an H100 SXM's by
    default). The
    grid counts the step's widest chunk (grid_n = Tmax); a tile is D / 64 k-blocks, plus D_T / 64 under a teacher."""
    import slab_paths
    import tile_schedule as ts

    Bs, Rs, Ts = cell.shapes()
    r = cell.r
    kb = ts.num_kb(D, DT if cell.opts.teacher else 0)
    out = []
    for c in range(cell.W):
        rt = chunk_route(cell, c)
        mode, stages, cs = rt[0][:3]
        n = ts.H100_CLUSTERS[cs] if clusters is None else clusters[(mode, stages, cs)]
        for win in slab_paths.windows(Rs[r], Bs[r], Ts[c], c == r, own_pos_ids(cell), cell.panel_rows()):
            out.append((rt, c, win, ts.launch(win[1], win[3], cs, stages, kb, n, max(Ts), num_sms or ts.NUM_SMS)))
    return out


def multi_items(cell: Cell, clusters=None, num_sms: Optional[int] = None) -> set:
    """What a cell's launches reach of the tile schedule: per instantiation a launch where some cluster runs 3 tiles or
    more and the last wave is ragged ("waves"), and consecutive tiles that keep / change the row block, a tile that
    starts mid-ring and one at phase 1; per mode every runtime option on in such a multi-wave launch (ids "iota" apart);
    per cluster size > 1 a CTA that scores a real block and then a phantom, in a cluster that goes on after a phantom;
    and at W > 1 chunks that give a cluster different tile counts (the grid_n grid)."""
    out = set()
    counts = {}
    for (inst, rt), _, _, L in cell_launches(cell, clusters, num_sms):
        mode = inst[0]
        opts = dict(ids=inst[3], metrics=inst[4], weights=inst[5]) if mode == "loss" else dict(rt)
        inst = tuple(bool(v) if k >= 3 else v for k, v in enumerate(inst))
        if L.max_tiles() >= 3 and L.ragged():
            out.add(("waves", inst))
            out.update(("option", mode, k if v is True else f"{k}={v}") for k, v in opts.items() if v)
        for what, ok in (("keep", L.keeps_row_block()), ("change", L.changes_row_block()), ("stage", L.mid_ring()),
                         ("phase", L.phase_one())):
            if ok:
                out.add((what, inst))
        if L.cs > 1 and L.phantom_after_real() and L.phantom_then_more():
            out.add(("phantom", L.cs))
        counts.setdefault(L.clusters, set()).add(tuple(len(x) for x in L.per_cluster))
    if cell.W > 1 and any(len(v) > 1 for v in counts.values()):
        out.add(("grid_n",))
    return out


TABLE = build_table()
COLD = build_table(cold=True)
MULTI = build_table(multi=True)
MULTI_COLD = build_table(cold=True, multi=True)


# ---------------------------------------------------------------------------------------------------------------------
# planted data
# ---------------------------------------------------------------------------------------------------------------------
@dataclass
class Problem:
    """Every rank's embeddings and per-sample inputs for the cell's shapes with all extras present (float64 values of
    integers / 8); an Options picks which of them a step uses."""
    Bs: tuple
    Rs: tuple
    Ts: tuple
    imgs: list        # [R_r, D]
    txts: list        # [T_r, D]
    ids: list         # [B_r] int64
    xt_ids: list      # [T_r - B_r]
    xi_ids: list      # [R_r - B_r]
    iw: list          # [R_r] fp32 values
    tw: list          # [T_r]
    ig: list          # [R_r] int64, -1: no group
    tg: list          # [T_r]
    itags: list       # [R_r, MMAX] int64 tags of the label sets, -1: an empty slot
    ttags: list       # [T_r, MMAX]
    timgs: list       # [R_r, DT] teacher
    ttxts: list       # [T_r, DT]

    def view(self, o: Options):
        """(Bs, Rs, Ts, imgs, txts) of the step: the extras a step without them does not have are cut off."""
        Rs = self.Rs if o.ximages else self.Bs
        Ts = self.Ts if o.xtexts else self.Bs
        return (self.Bs, Rs, Ts, [x[:n] for x, n in zip(self.imgs, Rs)], [x[:n] for x, n in zip(self.txts, Ts)])

    def teacher(self, o: Options):
        """(timgs [R_r, DT], ttxts [T_r, DT]) of the step."""
        Bs, Rs, Ts, _, _ = self.view(o)
        return [x[:n] for x, n in zip(self.timgs, Rs)], [x[:n] for x, n in zip(self.ttxts, Ts)]

    def sets(self, o: Options):
        """(image sets [R_r, M], text sets [T_r, M]) of a label-set step: the first M tag slots with the row's id
        (sample id, then the extra's id) in slot row % M, and the empty sets that siglip_set_label_sets writes for
        extras without sets of their own. A paired text's set is its image's."""
        Bs, Rs, Ts, _, _ = self.view(o)
        M = o.labels

        def build(tags, ids, extra_ids, b, n, own):
            s = tags[:n, :M].copy()
            s[np.arange(n), np.arange(n) % M] = np.concatenate([ids, extra_ids])[:n]
            if not own:
                s[b:] = -1
            return s

        return ([build(*a, o.xi_sets) for a in zip(self.itags, self.ids, self.xi_ids, Bs, Rs)],
                [build(*a, o.xt_sets) for a in zip(self.ttags, self.ids, self.xt_ids, Bs, Ts)])


def planted(cell: Cell) -> Problem:
    if cell.cold:
        return planted_cold(cell)
    Bs, K, E = shape_table(cell)[cell.W]
    Rs = tuple(b + e for b, e in zip(Bs, E))
    Ts = tuple(b + k for b, k in zip(Bs, K))
    g = np.random.default_rng(1000 + cell.seed)
    centres = g.choice([-1, 0, 1], (N_GROUPS, D), p=[0.2, 0.6, 0.2])
    n_ids = max(8, sum(Bs) // 2)                       # duplicates within and across ranks
    id_vec = g.choice([-1, 0, 1], (n_ids, D), p=[0.3, 0.4, 0.3])
    id_grp = g.integers(0, N_GROUPS, n_ids)
    tkey_vec = g.integers(-2, 3, (n_ids, DT))   # the teacher's vector of each key

    def near(idv):
        idv = np.asarray(idv, np.int64)
        return (centres[id_grp[idv]] + id_vec[idv] + g.choice([-1, 0, 1], (len(idv), D), p=[0.1, 0.8, 0.1])) / 8.0

    def tnear(idv):
        idv = np.asarray(idv, np.int64)
        return (tkey_vec[idv - (idv % 2 == 1)] + g.choice([-1, 0, 1], (len(idv), DT), p=[0.1, 0.8, 0.1])) / 8.0

    def groups_of(idv):
        gr = id_grp[np.asarray(idv, np.int64)].astype(np.int64)
        gr[g.random(len(gr)) < 0.2] = -1
        return gr

    def weights(n):
        w = g.random(n).astype(np.float32)
        w[g.random(n) < 0.2] = 0.0
        return w

    def tags(n):
        return np.where(g.random((n, MMAX)) < 0.15, 10 ** 7 + g.integers(0, N_TAGS, (n, MMAX)), -1).astype(np.int64)

    P = dict(imgs=[], txts=[], ids=[], xt_ids=[], xi_ids=[], iw=[], tw=[], ig=[], tg=[], itags=[], ttags=[], timgs=[],
             ttxts=[])
    for b, r_, t_ in zip(Bs, Rs, Ts):
        ids = g.integers(0, n_ids, b)
        # extras: a text (image) near a sample of the global id pool; a fifth of the extra images carry a fresh id
        xt = g.integers(0, n_ids, t_ - b)
        xi = g.integers(0, n_ids, r_ - b)
        xi_content = xi.copy()
        fresh = g.random(r_ - b) < 0.2
        xi[fresh] = 10 ** 6 + g.integers(0, 10 ** 6, int(fresh.sum()))
        P["ids"].append(ids.astype(np.int64))
        P["xt_ids"].append(xt.astype(np.int64))
        P["xi_ids"].append(xi.astype(np.int64))
        P["imgs"].append(np.concatenate([near(ids), near(xi_content)]))
        P["txts"].append(np.concatenate([near(ids), near(xt)]))
        P["iw"].append(weights(r_))
        P["tw"].append(weights(t_))
        P["ig"].append(np.concatenate([groups_of(ids), groups_of(xi_content)]))
        P["tg"].append(np.concatenate([groups_of(ids), groups_of(xt)]))
        ti = tags(r_)
        P["itags"].append(ti)
        P["ttags"].append(np.concatenate([ti[:b], tags(t_ - b)]))
        P["timgs"].append(np.concatenate([tnear(ids), tnear(xi_content)]))
        P["ttxts"].append(np.concatenate([tnear(ids), tnear(xt)]))
    if cell.multi and cell.opts.topk > 1:
        # rank r's first row block at 8x (integers, still exact): its rows' K-th best over any one tile lies above the
        # top-K keys of the next row blocks, so a CTA whose next tile kept the previous rows' top-K floor would lose
        # keys of its new rows' lists
        P["imgs"][cell.r][:TOPK_FLOOR_ROWS] *= TOPK_FLOOR_SCALE
    return Problem(Bs, Rs, Ts, **P)


TOPK_FLOOR_ROWS, TOPK_FLOOR_SCALE = 128, 8


# Cold data: integer rows / 8, so U = 64 <img, txt> is an integer and z = 5 U / 64 - 6 (U < 23.04: z < kFastZ).
COLD_BAND = 32                   # the first rows of each paired batch: duplicate ids, shared tags and groups
COLD_POOL = 24                   # the ids of the bands
COLD_SIG, COLD_COMMON = 96, 104  # dims [0, 96): a sample's signature, [96, 104): common to all, [104, D): planted pairs
COLD_TSIG = 56                   # teacher dims [0, 56): signature, [56, DT): planted slabs
COLD_TARGETS = (24, 36, 23)      # U of the planted pairs: just above kFastZ (-4.125), warm (-3.19), just below (-4.203)
COLD_TEACHER_U = 96              # added to U_T over a planted teacher slab: z_T ~ -1, p ~ 0.27


def planted_cold(cell: Cell) -> Problem:
    """The cold family's data: most negatives at z ~ -6.2 .. -4.6, so that the series slabs carry a large part of the
    loss, the gradients and each sample's loss. A sample is a signature of 32 entries +-1 over 96 dims (the one of its id,
    so positives and extras with a band id have U = 40, z = -2.9) plus 8 common dims (U = 8 between all rows). Duplicate
    ids, label-set tags and groups lie in the first COLD_BAND rows of each paired batch only, every other sample has an
    id of its own; a half of the extras caption a band id. Then, against each chunk, rank r gets planted negatives of
    U in COLD_TARGETS off the bands (one dim of their own each): general slabs off the diagonal and series slabs whose
    max z lies 3e-3 below kFastZ, where the series truncation is largest. The teacher's rows are a signature of 6 entries
    +-4 (z_T = -1 on pairs of one id, below -5.5 elsewhere) and, on some whole slabs of rank r, U_T + COLD_TEACHER_U:
    a teacher that knows matches the labels do not, in slabs whose student votes either way. Weights as planted's."""
    Bs, K, E = shape_table(cell)[cell.W]
    Rs = tuple(b + e for b, e in zip(Bs, E))
    Ts = tuple(b + k for b, k in zip(Bs, K))
    g = np.random.default_rng(1000 + cell.seed)
    sig, tsig = {}, {}
    fresh = iter(range(10 ** 5, 10 ** 6))

    def rows(idv):
        out = np.zeros((len(idv), D), np.int64)
        for n, k in enumerate(idv):
            if k not in sig:
                v = np.zeros(COLD_SIG, np.int64)
                v[g.choice(COLD_SIG, 32, replace=False)] = g.choice([-1, 1], 32)
                sig[k] = v
            out[n, :COLD_SIG] = sig[k]
        out[:, COLD_SIG:COLD_COMMON] = 1
        return out

    def trows(idv):
        out = np.zeros((len(idv), DT), np.int64)
        for n, k in enumerate(idv):
            if k not in tsig:
                v = np.zeros(COLD_TSIG, np.int64)
                v[g.choice(COLD_TSIG, 6, replace=False)] = g.choice([-4, 4], 6)
                tsig[k] = v
            out[n, :COLD_TSIG] = tsig[k]
        return out

    def weights(n):
        w = g.random(n).astype(np.float32)
        w[g.random(n) < 0.2] = 0.0
        return w

    def band_or_fresh(n):
        return np.array([g.integers(0, COLD_POOL) if g.random() < 0.5 else next(fresh) for _ in range(n)], np.int64)

    P = dict(imgs=[], txts=[], ids=[], xt_ids=[], xi_ids=[], iw=[], tw=[], ig=[], tg=[], itags=[], ttags=[], timgs=[],
             ttxts=[])
    for b, r_, t_ in zip(Bs, Rs, Ts):
        nb = min(COLD_BAND, b)
        ids = np.concatenate([g.integers(0, COLD_POOL, nb), [next(fresh) for _ in range(b - nb)]]).astype(np.int64)
        xt, xi_content = band_or_fresh(t_ - b), band_or_fresh(r_ - b)
        xi = xi_content.copy()
        new = g.random(r_ - b) < 0.2
        xi[new] = 10 ** 6 + g.integers(0, 10 ** 6, int(new.sum()))
        band = np.arange(b) < nb
        grp = np.where(band, ids % 3, -1)
        tags = np.where(band[:, None] & (g.random((b, MMAX)) < 0.3), 10 ** 7 + g.integers(0, 3, (b, MMAX)), -1)
        P["ids"].append(ids)
        P["xt_ids"].append(xt)
        P["xi_ids"].append(xi)
        P["imgs"].append(rows(np.concatenate([ids, xi_content])))
        P["txts"].append(rows(np.concatenate([ids, xt])))
        P["iw"].append(weights(r_))
        P["tw"].append(weights(t_))
        P["ig"].append(np.concatenate([grp, np.full(r_ - b, -1)]).astype(np.int64))
        P["tg"].append(np.concatenate([grp, np.full(t_ - b, -1)]).astype(np.int64))
        P["itags"].append(np.concatenate([tags, np.full((r_ - b, MMAX), -1)]).astype(np.int64))
        P["ttags"].append(np.concatenate([tags, np.full((t_ - b, MMAX), -1)]).astype(np.int64))
        P["timgs"].append(trows(np.concatenate([ids, xi_content])))
        P["ttxts"].append(trows(np.concatenate([ids, xt])))
    r, R = cell.r, Rs[cell.r]
    img, timg = P["imgs"][r], P["timgs"][r]
    n, nt = (D - COLD_COMMON) // cell.W, (DT - COLD_TSIG) // cell.W

    def off_diagonal(c, i0, j0):   # not a slab on the own diagonal (slab_paths.classes)
        return c != r or i0 // 128 != j0 // 128 or not (i0 < j0 + 32 and j0 < i0 + 16)

    for c in range(cell.W):
        txt, ttxt, T = P["txts"][c], P["ttxts"][c], Ts[c]
        pairs = []
        for k in range(n):
            i = COLD_BAND + (k * (R - COLD_BAND)) // n + int(g.integers(0, (R - COLD_BAND) // n))
            j = int(g.integers(COLD_BAND, T))
            while not off_diagonal(c, i // 16 * 16, j // 32 * 32):
                j = int(g.integers(COLD_BAND, T))
            d = COLD_COMMON + c * n + k
            img[i, d], txt[j, d] = 1, COLD_TARGETS[k % 3] - int(img[i] @ txt[j])
            pairs.append((i // 16 * 16, j // 32 * 32))
        for k in range(nt):
            if k % 2 == 0:   # the slab of a planted pair: the student's vote goes either way
                i0, j0 = pairs[k]
            else:
                i0, j0 = 16 * int(g.integers(COLD_BAND // 16, R // 16)), 32 * int(g.integers(COLD_BAND // 32, T // 32))
                while not off_diagonal(c, i0, j0):
                    j0 = 32 * int(g.integers(COLD_BAND // 32, T // 32))
            d = COLD_TSIG + c * nt + k
            timg[i0:i0 + 16, d], ttxt[j0:j0 + 32, d] = 8, COLD_TEACHER_U // 8
    for key in ("imgs", "txts", "timgs", "ttxts"):
        P[key] = [x / 8.0 for x in P[key]]
    return Problem(Bs, Rs, Ts, **P)


def cell_slabs(cell: Cell, P: Problem) -> List[Tuple[Tuple, "slab_paths.SlabMap"]]:
    """(chunk_route, SlabMap) of every loss launch of rank r's step (slab_paths.windows): the slabs' classes from the
    oracle's labels and the fp32 votes of the student (and of a teacher) on the planted logits."""
    import slab_paths

    o, r = cell.opts, cell.r
    Bs, Rs, Ts, imgs, txts = P.view(o)
    lab = labels(P, o)[r]
    timgs, ttxts = P.teacher(o) if o.teacher else (None, None)
    out = []
    for c in range(cell.W):
        route_c = chunk_route(cell, c)
        for r0, rows, c0, cols, own in slab_paths.windows(Rs[r], Bs[r], Ts[c], c == r, own_pos_ids(cell),
                                                          cell.panel_rows()):
            win = (slice(r0, r0 + rows), slice(c0, c0 + cols))
            s = imgs[r][win[0]] @ txts[c][win[1]].T
            ts = timgs[r][win[0]] @ ttxts[c][win[1]].T if o.teacher else None
            out.append((route_c, slab_paths.slab_map(s, lab[c][win], own, TP, BIAS, cell.f16, ts, TTP, TBIAS, c, r0,
                                                      c0)))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# the composed oracle
# ---------------------------------------------------------------------------------------------------------------------
def labels(P: Problem, o: Options):
    Bs, Rs, Ts, _, _ = P.view(o)
    if o.labels:
        lab = set_labels(*P.sets(o), Bs)
    else:
        lab = label_blocks(Bs, Rs, Ts, P.ids if o.ids else None, P.xt_ids if o.xt_ids else None,
                           P.xi_ids if o.xi_ids else None)
    if o.groups:
        lab = group_labels(lab, [x[:n] for x, n in zip(P.ig, Rs)], [x[:n] for x, n in zip(P.tg, Ts)])
    return lab


def oracle(P: Problem, o: Options, tp: float = TP, bias: float = BIAS, lam: float = LAM) -> List[Dict]:
    """Per rank: loss, dimg [R_r, D], contrib[c] [T_c, D], dt_prime, dbias, image_loss [R_r], text_part[c] (this rank's
    column sums over chunk c) and text_loss [T_r] (every rank's column sums of its chunk), at t' = tp, bias and the
    distillation weight lam (the cells' TP, BIAS and LAM by default)."""
    Bs, Rs, Ts, imgs, txts = P.view(o)
    iw = [x[:n].astype(np.float64) for x, n in zip(P.iw, Rs)] if o.weights else None
    tw = [x[:n].astype(np.float64) for x, n in zip(P.tw, Ts)] if o.weights else None
    lab = labels(P, o)
    if o.teacher:
        res = closed_form_distill_options(imgs, txts, tp, bias, *P.teacher(o), TTP, TBIAS, lam, lab, Bs, iw, tw)
    elif o.focal is not None:
        res = closed_form_focal(imgs, txts, tp, bias, lab, o.focal[0], o.focal[1], Bs, iw, tw)
    else:
        res = closed_form_groups(imgs, txts, tp, bias, lab, Bs, iw, tw)
    for r, x in enumerate(res):
        x["text_loss"] = text_loss_of(res, r)
    return res


def retrieval(P: Problem, o: Options, k: int) -> List[Dict]:
    """Per rank: top-K lists and recall (topk_retrieval, or topk_retrieval_sets under label sets), and the top-1 outputs
    they contain: i2t_index / t2i_index (column 0) and top1 = (i2t, t2i) rates as the kernels count them. Weights, groups,
    the focal terms and a teacher play no part; i2t ranks all R_r images only under extra-image ids or label sets, t2i
    all T_r texts only under extra-text ids or label sets."""
    Bs, Rs, Ts, imgs, txts = P.view(o)
    if o.labels:
        out = topk_retrieval_sets(imgs, txts, Bs, max(k, 1), *P.sets(o))
    else:
        img_ids = txt_ids = None
        if o.ids:
            img_ids = [np.concatenate([a, b]) if o.xi_ids else a for a, b in zip(P.ids, P.xi_ids)]
            txt_ids = [np.concatenate([a, b]) if o.xt_ids else a for a, b in zip(P.ids, P.xt_ids)]
        out = topk_retrieval(imgs, txts, Bs, max(k, 1), img_ids, txt_ids, rank_all_images=o.xi_ids,
                             rank_all_texts=o.xt_ids)
    for x in out:
        x["i2t_index"], x["t2i_index"] = x["i2t_topk"][:, 0].copy(), x["t2i_topk"][:, 0].copy()
        x["top1"] = np.array([recall_counts(x["i2t_first"], 1)[0], recall_counts(x["t2i_first"], 1)[0]], np.float32)
        x["recall_f32"] = np.concatenate([recall_counts(x["i2t_first"], max(k, 1)),
                                          recall_counts(x["t2i_first"], max(k, 1))])
    return out


def peer_stand_ins(P: Problem, o: Options, r: int, res: Optional[List[Dict]], ret: Optional[List[Dict]],
                   f16: bool = False):
    """What each peer p != r publishes for rank r's chunk: metric_keys (its column argmax keys, [B_r], [T_r] under
    extra-text ids or label sets), topk_keys ([T_r, KMAX] sorted, 0-padded), partials (fixed-point words of its column
    sums, [T_r]), xi_ids (its extra-image ids, under extra-image ids) and under label sets tsets (its text chunk's sets)
    and xi_sets (its extra images' sets). The keys hold the loss kernel's accumulator: <img, txt>, or 2^8 <img, txt> for
    fp16(16 x) operands (f16), as every rank of an INPUT_F16 job computes them."""
    acc = 256.0 if f16 else 1.0
    Bs, Rs, Ts, _, _ = P.view(o)
    isets, tsets = P.sets(o) if o.labels else (None, None)
    out = {}
    for p in range(len(Bs)):
        if p == r:
            continue
        d = {}
        if ret is not None:
            S, off, toff = ret[r]["S"], ret[r]["off"], ret[r]["toff"]
            keys = np.zeros((Ts[r], KMAX), np.int64)
            for j in range(Ts[r]):
                col = S[off[p]:off[p + 1], toff[r] + j]
                order = np.lexsort((np.arange(len(col)), -col))[:KMAX]
                keys[j, :len(order)] = [key_as_int64(metric_key(acc * col[i], off[p] + i)) for i in order]
            d["topk_keys"] = keys
            d["metric_keys"] = keys[:Ts[r] if (o.xt_ids or o.labels) else Bs[r], 0].copy()
        if res is not None:
            d["partials"] = np.array([fixed_point_partial(v)[0] for v in res[p]["text_part"][r]], np.int64)
        if o.xi_ids:
            d["xi_ids"] = P.xi_ids[p][:Rs[p] - Bs[p]]
        if o.labels:
            d["tsets"] = tsets[p]
            d["xi_sets"] = isets[p][Bs[p]:]
        out[p] = d
    return out


def rel(a, b) -> float:
    """The suite's norm-and-max relative error (test_gpu_exclude_groups._rel) in numpy."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return max(float(np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-300)),
               float(np.abs(a - b).max() / (np.abs(b).max() + 1e-300)))
