"""Step sequences on one long-lived context: the per-context state a step leaves behind, and the sequences that test it
— test infrastructure, never the product path.

A training job runs thousands of steps on one siglip_ctx, with fresh data, t' and bias at every step, options changed
between steps (siglip_ctx_set_option accepts almost every option at any time) and evaluation forwards and metric
requests in between. Several pieces of the context carry from one step to the next; STATE restates, for each, which
step kinds write it whole, which write part of it, which read it, and the rule that keeps a step from reading an
earlier step's values (with the csrc/siglip_capi.cu lines that implement it). A SEQUENCE is one context (W, rank,
shapes, context kind) and its steps; each step gives its options (option_matrix.Options: what it computes and which
requests it arms), its engine knobs (every siglip_ctx_set_option value), its schedule, a fresh data seed and its own
t', bias, distillation weight and upstream gradient. Some steps are refused on purpose (REFUSALS): each is followed by
a step that is checked against the oracle.

The oracle, data and stand-ins are option_matrix's (planted, oracle at the step's t' / bias / lambda, retrieval,
peer_stand_ins) and loopback_exchange's (the peers' contributions); there is no new loss math here.
tests/test_step_sequences_cpu.py derives from this model that every option changes both ways between two checked
steps, that every state item sees a transition in which a leak would show, and that such a leak moves a checked output
by more than 20x the tolerance; tests/test_gpu_step_sequences.py runs the sequences on the device."""
from __future__ import annotations

import dataclasses
import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import grad_matrix as gm
import option_matrix as om

SENSITIVITY = 20.0   # a claimed leak must move a checked output by more than this many tolerances
NUM_SMS = 132        # H100 SXM: the loss kernel's persistent grid is at most this many CTAs

# Two regimes of the scalars: "hot" steps (large loss, dt' and dbias) and the option matrix's regime. A stale fraction
# of a scalar only shows when the earlier step's value is the larger one, so every scalar transition runs hot -> cold.
HOT = (math.log(20.0), -2.0)
COLD = (om.TP, om.BIAS)

# siglip_ctx_set_option's options a sequence must change both ways between two checked steps, and the ones exempt
# because they change no output (timing events, the launch trace, the peer-wait bound, the accepted no-op sleeps)
EXEMPT = ("KERNEL_TIMING", "AUX_TRACE", "PEER_TIMEOUT_MS", "EPI_SLEEP_GRAD_NS", "EPI_SLEEP_LOSS_NS")
# the context's values at creation (siglip_ctx, csrc/siglip_capi.cu:190-300), with SigmoidLossEngine's cta_group = 2
DEFAULTS = dict(CTA_GROUP=2, MCAST=1, STAGES_LOSS=0, STAGES_GRAD=0, GRAD_TILE_N=0, SPLIT_K=0, OVERLAP_PULL=1,
                OVERLAP_REDUCE=1, INKERNEL_SYNC=1, PDL=1, BIDIR=0, SYNC_SCALAR_GRADS=0, SIGMA_BUDGET_MIB=0,
                INPUT_F16=0, TPRIME_F64=0, GRAD_BF16=0, SAMPLE_IDS=0, EXTRA_TEXT_IDS=0, EXTRA_IMAGE_IDS=0,
                LABEL_SETS=0, SAMPLE_WEIGHTS=0, EXCLUDE_GROUPS=0, FOCAL=0, DISTILL=0)
# the options that follow from a step's Options, operands and t' (the engine sets INPUT_F16 / TPRIME_F64 / GRAD_BF16
# from the tensors' dtypes); the rest are knobs a step sets directly
DERIVED = ("SAMPLE_IDS", "EXTRA_TEXT_IDS", "EXTRA_IMAGE_IDS", "LABEL_SETS", "SAMPLE_WEIGHTS", "EXCLUDE_GROUPS", "FOCAL",
           "DISTILL", "INPUT_F16", "TPRIME_F64", "GRAD_BF16", "SIGMA_BUDGET_MIB")
KNOBS = tuple(k for k in DEFAULTS if k not in DERIVED)

SCHEDS = ("fused", "scaled", "split", "fwd", "eval")
# fused: siglip_fwd_bwd; scaled: siglip_fwd_bwd_scaled with grad_out; split: siglip_forward(save) + siglip_backward with
# grad_out; fwd: siglip_fwd; eval: siglip_forward(save), siglip_fwd of other data, then the backward of the saved one

# the refusals a sequence provokes; each returns before the step counters advance
REFUSALS = ("ids", "extra_text_ids", "extra_image_ids", "weights", "groups", "sets", "teacher", "focal",
            "distill_losses", "distill_topk", "budget_below_panel", "split_over_budget", "backward_unsaved")


@dataclass(frozen=True)
class Step:
    opts: om.Options
    sched: str = "fused"
    knobs: Tuple[Tuple[str, int], ...] = ()   # every KNOBS value (make fills them in)
    budget: bool = False                      # SIGLIP_OPT_SIGMA_BUDGET_MIB at the sequence's smallest splitting budget
    budget_mib: int = 0                       # an explicit budget instead (a refusal's)
    f16: bool = False                         # fp16 (16 x) operands: INPUT_F16
    tp64: bool = False                        # t' as an fp64 tensor: TPRIME_F64
    bf16: bool = False                        # bf16 gradients: GRAD_BF16
    tp: float = COLD[0]
    bias: float = COLD[1]
    lam: float = om.LAM
    grad_out: float = 1.0
    seed: int = 0
    refuse: Optional[str] = None              # a REFUSALS kind: the call returns an error and computes nothing

    def knob(self, name: str) -> int:
        return dict(self.knobs)[name]

    @property
    def cluster(self) -> int:
        return self.knob("CTA_GROUP") * self.knob("MCAST")

    @property
    def backward(self) -> bool:
        return self.sched != "fwd"

    @property
    def requests(self) -> bool:
        return self.opts.metrics or self.opts.losses or self.opts.topk > 0


@dataclass
class Seq:
    name: str
    W: int
    r: int
    panel_shapes: bool = False             # option_matrix.PANEL_SHAPES (a budget can split the rows) or SHAPES
    split_shapes: bool = False             # option_matrix.SPLIT_SHAPES (the gradient kernel's split-K splits)
    xtexts: bool = False
    ximages: bool = False
    M: int = 0                             # label-set width of the context (siglip_ctx_create_labels), 0: none
    teacher: str = ""                      # "", "distill" (siglip_ctx_create_distill) or "extras" (..._distill_extras)
    steps: List[Step] = field(default_factory=list)

    def cell(self, st: Step) -> om.Cell:
        """The step as an option-matrix cell: its shapes, seed, schedule and configuration."""
        sched = {"scaled": "fused", "eval": "split"}.get(st.sched, st.sched)
        return om.Cell(st.opts, self.W, self.r, bool(st.knob("BIDIR")), sched, self.panel_shapes, st.f16,
                       st.knob("GRAD_TILE_N") or 128, st.knob("STAGES_LOSS") or 6, st.knob("CTA_GROUP"),
                       st.knob("MCAST"), st.seed, splitk=self.split_shapes)

    def budget_of(self, st: Step) -> int:
        if st.budget_mib:
            return st.budget_mib
        return self.cell(st).budget_mib(st.cluster) if st.budget else 0

    def options(self, st: Step) -> Dict[str, int]:
        """Every siglip_ctx_set_option value the context holds while the step runs."""
        o = st.opts
        out = dict(st.knobs)
        out.update(SAMPLE_IDS=int(o.ids), EXTRA_TEXT_IDS=int(o.xt_ids), EXTRA_IMAGE_IDS=int(o.xi_ids),
                   LABEL_SETS=int(o.labels > 0), SAMPLE_WEIGHTS=int(o.weights), EXCLUDE_GROUPS=int(o.groups),
                   FOCAL=int(o.focal is not None), DISTILL=int(o.teacher), INPUT_F16=int(st.f16),
                   TPRIME_F64=int(st.tp64), GRAD_BF16=int(st.bf16), SIGMA_BUDGET_MIB=self.budget_of(st))
        return out


def make(name, W, r, steps, panel_shapes=False, xtexts=False, ximages=False, M=0, teacher="", seed=0,
         split_shapes=False, **base):
    """A sequence from step deltas: each step is a dict of Step fields and knobs (by option name) that differ from the
    previous step; the first starts from DEFAULTS and `base`. Options is given whole (`o`), or defaults to the previous
    step's with its requests off; every step draws fresh data (seed) unless it is a refusal."""
    out, prev = [], None
    knobs = {k: DEFAULTS[k] for k in KNOBS}
    knobs.update(base)
    ctx = dict(xtexts=xtexts, ximages=ximages)
    for i, d in enumerate(steps):
        d = dict(d)
        knobs.update({k: d.pop(k) for k in list(d) if k in KNOBS})
        if "o" in d:
            o = om.Options(**ctx, **d.pop("o"))
        else:
            o = dataclasses.replace(prev.opts, metrics=False, losses=False, topk=0) if prev else om.Options(**ctx)
        kw = dict(sched="fused", f16=False, tp64=False, bf16=False, tp=COLD[0], bias=COLD[1], lam=om.LAM,
                  grad_out=1.0, budget=False)
        if prev is not None:   # dtypes, regime, budget and grad_out carry over unless the delta changes them
            kw.update(sched=prev.sched, f16=prev.f16, tp64=prev.tp64, bf16=prev.bf16, tp=prev.tp, bias=prev.bias,
                      lam=prev.lam, grad_out=prev.grad_out, budget=prev.budget)
        if d.pop("hot", False):
            kw.update(tp=HOT[0], bias=HOT[1])
        if d.pop("cold", False):
            kw.update(tp=COLD[0], bias=COLD[1])
        kw.update(d)
        if kw["sched"] in ("fused", "fwd"):   # siglip_fwd_bwd and siglip_fwd take no upstream gradient
            kw["grad_out"] = 1.0
        kw.setdefault("refuse", None)
        if kw["refuse"] is None:
            kw.pop("budget_mib", None)
        st = Step(o, knobs=tuple(sorted(knobs.items())), seed=seed * 100 + i, **kw)
        assert o.valid(), (name, i, o)
        out.append(st)
        prev = st if st.refuse is None else (prev or st)
    return Seq(name, W, r, panel_shapes, split_shapes, xtexts, ximages, M, teacher, out)


# ---------------------------------------------------------------------------------------------------------------------
# the loss launch's grid (slab_paths / option_matrix.route's model: 128-row tiles per cluster rank, 128-column tiles,
# row-panel windows, a persistent grid of at most NUM_SMS CTAs)
# ---------------------------------------------------------------------------------------------------------------------
def panel_rows(seq: Seq, st: Step) -> int:
    """Rows of the step's row panels (all R_r rows without a budget): option_matrix's sigma_panels restatement."""
    Bs, Rs, Ts = seq.cell(st).shapes()
    mib = seq.budget_of(st)
    if not mib or st.sched != "fused" and st.sched != "scaled":
        return Rs[seq.r]
    unit = 128 * st.cluster
    P = mib * 2 ** 20 // ((2 if seq.W > 1 else 1) * om._round_up(max(Ts), 256) * 2) // unit * unit
    return min(P, Rs[seq.r])


def panels(seq: Seq, st: Step) -> int:
    Bs, Rs, Ts = seq.cell(st).shapes()
    return -(-Rs[seq.r] // panel_rows(seq, st))


def loss_grid(seq: Seq, st: Step, rows: int) -> int:
    """CTAs of a loss launch over `rows` rows: the grid of the largest chunk (grid_n = Tmax), in whole clusters."""
    Bs, Rs, Ts = seq.cell(st).shapes()
    cs = st.cluster
    tiles = -(-rows // (128 * cs)) * -(-max(Ts) // 128)
    return min(NUM_SMS // cs, tiles) * cs


def first_grid(seq: Seq, st: Step) -> int:
    """The grid of the forward's first loss launch, which overwrites its CTAs' partial slots: the own chunk's panel 0
    (W > 1), or at W = 1 under panels the last, shortest panel (preceded by the memset of every slot)."""
    Bs, Rs, Ts = seq.cell(st).shapes()
    P = panel_rows(seq, st)
    n = panels(seq, st)
    rows = Rs[seq.r] - (n - 1) * P if (seq.W == 1 and n > 1) else min(P, Rs[seq.r])
    return loss_grid(seq, st, rows)


def split_launches(seq: Seq, st: Step) -> Tuple:
    """(cluster size, S, split tiles) of every gradient launch of the step that splits K (grad_matrix.split_rule, the
    restatement of launch_impl's rule: S is cut back until every slice has 8 k-blocks, so a launch splits only when
    both of its problems' K are at least 961); empty: the split-K workspace is neither written nor read."""
    Bs, Rs, Ts = seq.cell(st).shapes()
    sched = "split" if st.sched in ("split", "eval") else "fused"
    c = gm.Ctx(Bs, Rs, Ts, om.D, r=seq.r, cg=st.knob("CTA_GROUP"), mcast=st.knob("MCAST"), stages=st.knob("STAGES_GRAD"),
               tile_n=st.knob("GRAD_TILE_N"), split_k=st.knob("SPLIT_K"), f16=st.f16, bf16=st.bf16,
               budget_mib=seq.budget_of(st) if sched == "fused" else 0, sched=sched, grad_out=st.sched != "fused",
               overlap_reduce=bool(st.knob("OVERLAP_REDUCE")))
    return tuple((st.cluster, L.split.S, L.split.rem) for L in gm.launches(c) if L.split.S > 1)


# ---------------------------------------------------------------------------------------------------------------------
# the state table
# ---------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Item:
    name: str
    fields: str        # the siglip_ctx members
    whole: str         # step kinds that write it whole
    part: str          # step kinds that write part of it
    reads: str         # step kinds that read it
    reset: str         # what keeps a step from reading an earlier step's values, restated from the code
    leak: str          # the smallest leak the model allows (test_step_sequences_cpu measures it on the oracle)


STATE = [
    Item("partials", "partials [num_sms][4], fin_counter",
         "every forward: the own chunk's first loss launch over its grid",
         "the later loss launches of the forward add into the slots of their CTAs",
         "the forward's last loss launch (its last CTA sums every slot into loss, dt', dbias)",
         "the first launch overwrites the slots of its grid (run_loss_chunk, siglip_capi.cu:1716); every launch of a "
         "forward keeps the grid of its largest chunk (grid_n = Tmax, siglip_kernels.cu:2840); at W = 1 under row "
         "panels the shortest panel runs first, so every slot is zeroed first (siglip_capi.cu:1731)",
         "one CTA's partial of the previous step (one 128-row block's share of loss, dt' and dbias)"),
    Item("sigma", "G[i] with g_rows, gen, saved_f16",
         "a saving forward (all W operands), the fused step (buffers 0 and 1, panel by panel)",
         "a row panel writes its rows of the buffer", "the gradient kernels of the split backward and the fused step",
         "gen = 0 on a saving or multi-rank forward (siglip_capi.cu:1444), on the fused step (1639), on a budget change "
         "(2245, which also releases the operands) and on SIGLIP_OPT_BIDIR (2276); the backward refuses gen = 0 (1517)",
         "one stale 128-row block of dimg"),
    Item("diag_and_16bit", "g_diag, img16 / txt16",
         "the conversion jobs of the step's first loss launch (add_cvt_jobs, siglip_capi.cu:1118)",
         "a panel's loss launch writes g_diag for its rows", "the gradient kernels (the positive-pair term)",
         "written by every forward that saves, in its loss launches (add_cvt_jobs before run_loss_chunk, siglip_capi.cu:1466, "
         "1696, 1727), before any gradient launch reads them; INPUT_F16 picks the conversion",
         "one stale 128-row block of dimg or dtxt"),
    Item("accumulators", "dimg_acc, dtxt_acc, slots",
         "the first gradient launch of a step (dimg_add = null at j = 1, siglip_capi.cu:1537, 1814)",
         "later launches add; own panels past 0 sum into own_part (slot r or dtxt_acc, siglip_capi.cu:1649)",
         "the last gradient launch, the folds and debug_get_slot",
         "the first gradient launch of every backward writes without an add source (siglip_capi.cu:1537, 1814, 1854)",
         "one stale 128-row block of dimg, dtxt or a peer slot"),
    Item("split_k", "splitk_ws, splitk_counters",
         "a gradient launch that splits K (SIGLIP_OPT_SPLIT_K, mcast 1, both K >= 961: split_launches)",
         "the tiles of the ragged last wave", "the same launch's last K-slice",
         "the counters return to 0 when a tile's last slice has added (siglip_capi.cu:887 zeroes them once)",
         "one stale 128-row block of dimg or dtxt"),
    Item("saved_scalars", "scalars[8], scalars[9]", "a saving forward and the fused step (fin.dt_prime, 1459, 1654)",
         "", "the split backward (dt' and dbias times grad_out)",
         "a forward without save writes no saved scalar (fin.dt_prime = null, siglip_capi.cu:1459)",
         "the previous step's dt' and dbias"),
    Item("parity_blocks", "mkeys[2], lsum[2], tk_cols[2] / tk_rows[2]",
         "an armed step of that parity (memsets in take_metrics 634, take_sample_losses 585, take_topk 736)",
         "the loss kernels of an armed step", "the finalisation kernels of an armed step",
         "memset at the start of every armed step of the parity (siglip_capi.cu:585, 634, 736); an unarmed step neither "
         "writes nor reads them",
         "one stale key, list entry or fixed-point word"),
    Item("step_inputs", "ids_in, rids, lrows, w_in, ids_all / w_all / ttxt_all, and their *_set flags",
         "siglip_set_* before the step; the pulls of the step (add_pull_job, 1316)",
         "the ids copies move the chunk's ids (or the whole slot under groups or label sets)",
         "the loss kernels and the finalisations",
         "take_ids (siglip_capi.cu:444) refuses a step whose inputs were not given since the previous step and clears "
         "the flags (473-479); set_option clears the flag of the option it changes (2200, 2222, 2232, 2285-2308)",
         "one stale pulled chunk of each kind (text, ids, weights, groups, sets, teacher text)"),
    Item("teacher_focal", "t_img / t_txt / teacher scalars and lambda, gamma / alpha",
         "siglip_set_teacher (teacher_set, cleared by take_ids 475), siglip_set_focal (focal_set, 2659)", "",
         "the loss kernels of a distillation or focal step",
         "the teacher is given before every step (take_ids clears teacher_set, siglip_capi.cu:475); the focal terms hold "
         "until the next siglip_set_focal (2659)",
         "the previous step's lambda, gamma or alpha"),
    Item("counters", "n_fwd / n_bwd / prewait3",
         "", "every forward (++n_fwd, 1438, 1632), every backward (++n_bwd, 1522, 1633)",
         "the flag values of a multi-rank step, and the parity of the request blocks",
         "a refused call returns before the counters advance (siglip_capi.cu:1434-1438, 1626-1632)", "the previous step's request block parity"),
]
ITEMS = tuple(i.name for i in STATE)


def writes(seq: Seq, st: Step) -> Dict[str, object]:
    """What the step writes of each state item: an extent (larger is more) or a content tag; None: nothing."""
    o = st.opts
    Bs, Rs, Ts = seq.cell(st).shapes()
    fwd = st.refuse is None
    saves = fwd and st.sched in ("fused", "scaled", "split", "eval")
    grads = fwd and st.backward
    return {
        "partials": first_grid(seq, st) if fwd else None,
        "sigma": (panel_rows(seq, st), st.f16) if saves else None,
        "diag_and_16bit": ("f16" if st.f16 else "bf16", panel_rows(seq, st)) if saves else None,
        "accumulators": (panels(seq, st), st.sched) if grads else None,
        "split_k": split_launches(seq, st) if grads else None,
        "saved_scalars": (st.tp, st.bias) if saves else None,
        "parity_blocks": (o.keys, o.losses, o.topk) if fwd and st.requests else None,
        "step_inputs": tuple(k for k in ("ids", "xt_ids", "xi_ids", "weights", "groups", "teacher") if getattr(o, k))
        + ((f"M{o.labels}",) if o.labels else ()) if fwd else None,
        "teacher_focal": (o.focal, st.lam if o.teacher else None) if fwd and (o.teacher or o.focal) else None,
        "counters": fwd,
    }


def transitions(seq: Seq) -> Dict[str, List[Tuple[int, int]]]:
    """(earlier, later) step indices per state item where the earlier successful step wrote more of the item than the
    later one reads, or different content: grid or panel shrink, panels off after on, fp16 -> bf16, requests armed ->
    unarmed -> armed on one parity, K up, inputs off and on again, a lambda or (gamma, alpha) change, a cluster change
    under split-K, and the hot -> cold scalar regime for the scalar-carrying items."""
    ok = [i for i, st in enumerate(seq.steps) if st.refuse is None]
    out = {k: [] for k in ITEMS}
    for a, b in zip(ok, ok[1:]):
        A, B = seq.steps[a], seq.steps[b]
        wa, wb = writes(seq, A), writes(seq, B)
        hot_cold = A.tp > B.tp and A.bias > B.bias
        # slots past the later step's first grid: a smaller grid, or at W = 1 the shortest panel running first
        if hot_cold and (wa["partials"] > wb["partials"] or (seq.W == 1 and panels(seq, B) > 1)):
            out["partials"].append((a, b))
        if wa["sigma"] and wb["sigma"] and (wa["sigma"][0] > wb["sigma"][0] or wa["sigma"][1] != wb["sigma"][1]):
            out["sigma"].append((a, b))
        if wa["diag_and_16bit"] and wb["diag_and_16bit"] and wa["diag_and_16bit"] != wb["diag_and_16bit"]:
            out["diag_and_16bit"].append((a, b))
        if wa["accumulators"] and wb["accumulators"] and wa["accumulators"] != wb["accumulators"]:
            out["accumulators"].append((a, b))
        if wa["split_k"] and wb["split_k"] and wa["split_k"] != wb["split_k"]:   # two splitting steps, other splits
            out["split_k"].append((a, b))
        if wa["saved_scalars"] and B.sched in ("split", "eval") and hot_cold:
            out["saved_scalars"].append((a, b))
        if wa["step_inputs"] != wb["step_inputs"] and wa["step_inputs"] and wb["step_inputs"]:
            out["step_inputs"].append((a, b))
        if (A.opts.teacher and B.opts.teacher and A.lam != B.lam) or \
                (A.opts.focal and B.opts.focal and A.opts.focal != B.opts.focal):
            out["teacher_focal"].append((a, b))
        if b > a + 1:   # a refused call between two successful steps
            out["counters"].append((a, b))
    # the request blocks: armed at step a, then the same parity (two forwards later) armed again with less or other
    # requests, one unarmed step between
    for i, a in enumerate(ok):
        for b in ok[i + 2:i + 3]:
            A, M_, B = seq.steps[a], seq.steps[ok[i + 1]], seq.steps[b]
            if A.requests and B.requests and not M_.requests:
                out["parity_blocks"].append((a, b))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# the sequences
# ---------------------------------------------------------------------------------------------------------------------
O = dict   # Options fields (the context's extras are added by make)


def _sequences() -> List[Seq]:
    S = []
    # W = 1, plain context: panels on -> off -> on (the panel-slot memset), requests armed -> unarmed -> armed on one
    # parity, K up, hot -> cold scalars, grid shrink through the cluster shape
    S.append(make("w1-plain-panels", 1, 0, [
        dict(o=O(metrics=True, topk=3), budget=True, hot=True),
        dict(budget=False, cold=True, CTA_GROUP=1),
        dict(o=O(topk=7, losses=True), budget=True, hot=True, CTA_GROUP=2, MCAST=2),
        dict(cold=True, MCAST=1, sched="split", budget=False),
        dict(o=O(metrics=True), sched="fwd", hot=True),
        dict(sched="fused", cold=True, f16=True),
        dict(o=O(losses=True, topk=2), f16=False, hot=True),
        dict(cold=True, sched="scaled", grad_out=0.5),
    ], panel_shapes=True, seed=1))
    # W = 1, hard negatives: the eval schedule (a forward without save between a saving forward and its backward),
    # saved scalars hot -> cold, split-K under a cluster change, t' in fp64, bf16 gradients
    S.append(make("w1-hn-eval-splitk", 1, 0, [
        dict(hot=True, SPLIT_K=-1, GRAD_TILE_N=128),
        dict(sched="eval", cold=True, tp64=True, CTA_GROUP=1),
        dict(sched="split", hot=True, bf16=True, SPLIT_K=2, CTA_GROUP=2),
        dict(sched="split", cold=True, tp64=False, bf16=False, SPLIT_K=0, GRAD_TILE_N=256),
        dict(o=O(metrics=True, losses=True), sched="fused", hot=True, STAGES_LOSS=4, STAGES_GRAD=4),
        dict(sched="eval", cold=True, SPLIT_K=-1, STAGES_LOSS=0, STAGES_GRAD=0, GRAD_TILE_N=128),
    ], xtexts=True, seed=2))
    # W = 1, extras with ids: ids / extra ids off and on again, weights and groups, and the take_ids refusals of ids
    S.append(make("w1-xt-ids", 1, 0, [
        dict(o=O(ids=True, xt_ids=True, metrics=True), hot=True),
        dict(o=O(ids=True, xt_ids=True, weights=True, metrics=True), refuse="extra_text_ids"),
        dict(o=O(ids=True, weights=True, topk=4), cold=True),
        dict(o=O(ids=True, xt_ids=True, groups=True, losses=True), hot=True, PDL=0),
        dict(o=O(ids=True, xt_ids=True, groups=True), refuse="groups"),
        dict(o=O(groups=True, weights=True, metrics=True), cold=True, PDL=1),
        dict(o=O(ids=True, groups=True), refuse="ids"),
        dict(o=O(ids=True, xt_ids=True, metrics=True, losses=True), hot=True, f16=True),
        dict(o=O(), cold=True, f16=False),
    ], xtexts=True, seed=3))
    # W = 1, extra images with ids: extra-image ids, weights refused, both ways
    S.append(make("w1-xi-ids", 1, 0, [
        dict(o=O(ids=True, xi_ids=True, topk=5, losses=True), hot=True),
        dict(o=O(ids=True, xi_ids=True), refuse="extra_image_ids"),
        dict(o=O(ids=True, weights=True, metrics=True), cold=True),
        dict(o=O(ids=True, weights=True), refuse="weights"),
        dict(o=O(ids=True, xi_ids=True, weights=True), hot=True, sched="split"),
        dict(o=O(topk=3), cold=True, sched="fused"),
    ], ximages=True, seed=4))
    # W = 1, label sets: sets off and on (ids in between), the refusal of missing sets, focal on and off with its own
    # refusal (set_focal never called), (gamma, alpha) changed
    S.append(make("w1-labels-focal", 1, 0, [
        dict(o=O(labels=3, metrics=True), hot=True),
        dict(o=O(labels=3, topk=3), refuse="sets"),
        dict(o=O(ids=True, topk=4), cold=True),
        dict(o=O(labels=3, focal=(2.0, 0.25)), refuse="focal"),
        dict(o=O(labels=3, focal=(2.0, 0.25), losses=True), hot=True),
        dict(o=O(labels=3, focal=(0.5, None), topk=3), cold=True),
        dict(o=O(labels=3, groups=True, losses=True)),
        dict(o=O(focal=(5.0, 0.25)), hot=True),
    ], panel_shapes=True, M=3, seed=5))
    # W = 1, a distillation context: lambda changes, DISTILL off and on, the teacher refusal, and the two refusals of
    # a request the context cannot serve under DISTILL (per-sample losses, top-K), each followed by a checked step
    S.append(make("w1-distill", 1, 0, [
        dict(o=O(teacher=True, metrics=True), hot=True, lam=0.9),
        dict(o=O(teacher=True, losses=True), refuse="distill_losses"),
        dict(o=O(teacher=True), cold=True, lam=0.3),
        dict(o=O(teacher=True, topk=3), refuse="distill_topk"),
        dict(o=O(ids=True, metrics=True), hot=True),
        dict(o=O(teacher=True, ids=True), refuse="teacher"),
        dict(o=O(teacher=True, ids=True, weights=True), cold=True, lam=0.6, sched="split"),
        dict(o=O(topk=2, losses=True), sched="fused"),
    ], teacher="distill", seed=6))
    # W = 1, a distill-extras context: a teacher with extras, sets, focal excluded; teacher on -> off -> on
    S.append(make("w1-distill-extras", 1, 0, [
        dict(o=O(teacher=True, ids=True, xt_ids=True, xi_ids=True, losses=True, topk=3), hot=True, lam=0.8),
        dict(o=O(ids=True, xt_ids=True, metrics=True), cold=True),
        dict(o=O(teacher=True, labels=2, xt_sets=True, groups=True, topk=4), hot=True, lam=0.4),
        dict(o=O(teacher=True, labels=2, xi_sets=True, losses=True), cold=True, f16=True),
        dict(o=O(focal=(2.0, None), labels=2), hot=True, f16=False),
        dict(o=O(teacher=True), cold=True, lam=0.6),
    ], xtexts=True, ximages=True, M=2, teacher="extras", seed=7))
    # W = 1: the budget refusals (a saving forward over the budget, backward without a saved forward) and the
    # refusals' requests left unconsumed
    S.append(make("w1-budget-refusals", 1, 0, [
        dict(o=O(metrics=True, losses=True), budget=True, hot=True),
        dict(o=O(topk=3, losses=True), sched="split", refuse="split_over_budget"),
        dict(sched="fused", cold=True),
        dict(sched="split", refuse="backward_unsaved"),
        dict(o=O(metrics=True), sched="split", budget=False, hot=True),
        dict(sched="fused", budget=True, cold=True, CTA_GROUP=1),
    ], panel_shapes=True, seed=8))

    # W = 2 and 3: fresh peers, contributions and mailboxes every step; exchange options both ways
    S.append(make("w2-plain-exchange", 2, 0, [
        dict(o=O(metrics=True), hot=True),
        dict(cold=True, INKERNEL_SYNC=0, OVERLAP_REDUCE=0),
        dict(sched="split", hot=True, OVERLAP_PULL=0),
        dict(o=O(losses=True, topk=3), sched="split", cold=True, OVERLAP_PULL=1, OVERLAP_REDUCE=1),
        dict(sched="fused", hot=True, INKERNEL_SYNC=1, SYNC_SCALAR_GRADS=1),
        dict(o=O(metrics=True, losses=True), sched="split", cold=True, grad_out=0.75),
        dict(sched="scaled", hot=True, SYNC_SCALAR_GRADS=0, grad_out=2.0),
        dict(sched="fwd", cold=True),
    ], seed=9))
    S.append(make("w2-panels", 2, 1, [
        dict(o=O(topk=4, losses=True), budget=True, hot=True),
        dict(budget=False, cold=True),
        dict(o=O(topk=6, losses=True), budget=True, hot=True, BIDIR=1),
        dict(cold=True, CTA_GROUP=1, bf16=True),
        dict(o=O(metrics=True), budget=False, hot=True, BIDIR=0, CTA_GROUP=2, bf16=False, sched="split"),
        dict(sched="fused", cold=True, budget=True, MCAST=2),
        dict(o=O(losses=True), refuse="budget_below_panel", budget_mib=1),
        dict(sched="fused", hot=True, MCAST=1),
        dict(cold=True),
    ], panel_shapes=True, seed=10))
    S.append(make("w2-hn-ids", 2, 1, [
        dict(o=O(ids=True, xt_ids=True, weights=True, metrics=True), hot=True, f16=True),
        dict(o=O(ids=True, weights=True, groups=True, topk=3), cold=True, f16=False),
        dict(o=O(ids=True, groups=True), refuse="groups"),
        dict(o=O(groups=True, losses=True), hot=True, sched="split"),
        dict(o=O(ids=True, xt_ids=True, metrics=True), cold=True, sched="fused"),
        dict(o=O(ids=True, xt_ids=True), refuse="ids"),
        dict(o=O(weights=True), hot=True),
        dict(o=O(ids=True, xt_ids=True, weights=True, losses=True), cold=True),
    ], xtexts=True, seed=11))
    S.append(make("w2-xi-labels", 2, 0, [
        dict(o=O(labels=2, xi_sets=True, metrics=True), hot=True),
        dict(o=O(labels=2, xi_sets=True, weights=True, topk=3), cold=True),
        dict(o=O(ids=True, xi_ids=True, losses=True), hot=True),
        dict(o=O(labels=2, focal=(2.0, 0.25), groups=True, metrics=True), cold=True),
        dict(o=O(labels=2, focal=(0.5, 0.25), losses=True), hot=True),
        dict(o=O(labels=2, xi_sets=True), cold=True, sched="split"),
    ], ximages=True, M=2, seed=12))
    S.append(make("w2-distill-extras", 2, 1, [
        dict(o=O(teacher=True, ids=True, xt_ids=True, losses=True), hot=True, lam=0.9),
        dict(o=O(teacher=True, ids=True, xt_ids=True, topk=3), cold=True, lam=0.2, sched="split"),
        dict(o=O(ids=True, xt_ids=True), refuse="ids"),
        dict(o=O(ids=True, metrics=True), hot=True, sched="fused"),
        dict(o=O(teacher=True, labels=3, xt_sets=True, groups=True), cold=True, lam=0.6),
        dict(o=O(teacher=True, labels=3), refuse="teacher"),
        dict(o=O(teacher=True, labels=3, losses=True), hot=True, f16=True),
    ], xtexts=True, M=3, teacher="extras", seed=13))
    S.append(make("w3-plain", 3, 1, [
        dict(o=O(metrics=True, losses=True), hot=True, BIDIR=1),
        dict(cold=True, sched="split", tp64=True),
        dict(o=O(topk=5), hot=True, BIDIR=0, sched="fused", tp64=False),
        dict(cold=True, sched="split", SYNC_SCALAR_GRADS=1),
        dict(o=O(losses=True), hot=True, sched="split", OVERLAP_REDUCE=0),
        dict(cold=True, sched="fused", SYNC_SCALAR_GRADS=0, OVERLAP_REDUCE=1, INKERNEL_SYNC=0),
        dict(o=O(metrics=True), sched="fwd", hot=True),
        dict(cold=True, sched="scaled", grad_out=0.25, INKERNEL_SYNC=1),
    ], seed=14))
    S.append(make("w3-panels-hn", 3, 2, [
        dict(o=O(ids=True, topk=3), budget=True, hot=True),
        dict(o=O(ids=True), budget=False, cold=True),
        dict(o=O(ids=True, losses=True, topk=5), budget=True, hot=True, CTA_GROUP=1),
        dict(o=O(weights=True), cold=True, CTA_GROUP=2, SPLIT_K=-1),
        dict(o=O(weights=True, metrics=True), hot=True, MCAST=2),
        dict(o=O(), cold=True, MCAST=1, SPLIT_K=0, budget=False),
    ], xtexts=True, panel_shapes=True, seed=15))
    # W = 1 at SPLIT_SHAPES, where the gradient launches split K: a cluster change and a split count change between
    # splitting steps (the counters must be back at 0, the workspace rewritten), split-K off and on again
    S.append(make("w1-splitk", 1, 0, [
        dict(hot=True, SPLIT_K=-1, GRAD_TILE_N=128),
        dict(cold=True, CTA_GROUP=1),
        dict(o=O(metrics=True), hot=True, sched="split", SPLIT_K=2),
        dict(cold=True, sched="fused", SPLIT_K=0),
        dict(hot=True, SPLIT_K=-1, CTA_GROUP=2, bf16=True),
        dict(o=O(losses=True), cold=True, sched="scaled", grad_out=0.5, bf16=False, CTA_GROUP=1),
    ], split_shapes=True, seed=16))
    return S


SEQUENCES: List[Seq] = _sequences()
