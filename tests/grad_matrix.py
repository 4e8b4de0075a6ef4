"""The gradient kernel's (kModeOut) launch rules, restated from the host code, and the table of cells that runs them.

Every gradient launch of a step contracts two problems in one persistent kernel: dimg (M = panel rows, K = the chunk's
texts, the sigma operand K-major) and dtxt (M = the chunk's texts, K = panel rows, the operand MN-major), N = D for
both. This module restates, as plain functions of the context's options and shapes:
  * grad_tile_cols (csrc/siglip_capi.cu): 128 or 256 columns; split-K with mcast = 1 forces 128;
  * launch_gemm's dispatch (csrc/siglip_kernels.cu): 128 columns x {4, 6} stages x clusters {1, 2, 4}, and 256 columns
    (always kWideStages = 4) x clusters {1, 2, 4} — the 9 production instantiations;
  * launch_impl's split-K of the ragged last wave: rem = tiles % clusters, S = clusters // rem (capped at 4 for -1 and at
    an explicit request), slices of at least 8 k blocks, at most kSplitKMaxTiles split tiles, the workspace, mcast = 1;
  * run_grad_chunk's per-problem epilogue branches for every launch of a fused (siglip_fwd_bwd) or split
    (siglip_forward + siglip_backward) step, with row panels, W >= 1, extras, own_pos_ids, INPUT_F16 and GRAD_BF16.
tests/test_grad_matrix_cpu.py derives from it that the cells reach every instantiation, every branch and split-K with
S = 2, 3 and 4 at cluster sizes 1 and 2 on both problems; tests/test_gpu_grad_matrix.py runs the cells against the
float64 oracle. The co-resident cluster counts are inputs: H100 SXM values here, the device's own on the GPU.
"""
from __future__ import annotations

import itertools
import math
from dataclasses import dataclass, replace
from typing import Dict, List, Optional, Tuple

import numpy as np

NUM_SMS = 132                           # H100 SXM
H100_CLUSTERS = {1: 132, 2: 66, 4: 30}  # co-resident clusters of the out kernel per cluster size (4: never split)
BLOCK_M, BLOCK_K = 128, 64
TILE, WIDE_TILE, WIDE_STAGES = 128, 256, 4
SPLIT_K_MAX_TILES = 160                 # kSplitKMaxTiles
X_SCALE = 16.0                          # INPUT_F16 operands hold fp16(16 x)


def ceil_div(a: int, b: int) -> int:
    return -(-a // b)


def splitk_ws_bytes(num_sms: int = NUM_SMS) -> int:
    """ensure_splitk: (SMs + 2) fp32 partials of 128 x 128."""
    return (num_sms + 2) * 128 * TILE * 4


@dataclass(frozen=True)
class Ctx:
    """One rank's context and step. Bs / Rs / Ts: batch, images and texts per rank (Rs > Bs: extra images, Ts > Bs:
    hard-negative texts). stages / tile_n / split_k / budget_mib: SIGLIP_OPT_STAGES_GRAD, GRAD_TILE_N, SPLIT_K,
    SIGMA_BUDGET_MIB. sched: "fused" (siglip_fwd_bwd) or "split" (siglip_forward with save, then siglip_backward).
    grad_out: an upstream gradient tensor is passed. overlap_reduce: SIGLIP_OPT_OVERLAP_REDUCE (split backward, W > 1)."""
    Bs: Tuple[int, ...]
    Rs: Tuple[int, ...]
    Ts: Tuple[int, ...]
    D: int
    r: int = 0
    cg: int = 2
    mcast: int = 1
    stages: int = 0
    tile_n: int = 0
    split_k: int = 0
    f16: bool = False
    bf16: bool = False
    budget_mib: int = 0
    sched: str = "fused"
    grad_out: bool = False
    overlap_reduce: bool = True

    @property
    def W(self) -> int:
        return len(self.Bs)

    @property
    def cs(self) -> int:
        return self.cg * self.mcast

    @property
    def own_pos_ids(self) -> bool:
        """Extra images and extra texts: the positives of the own chunk are iota ids in G, no fp32 term."""
        return self.Rs[self.r] > self.Bs[self.r] and self.Ts[self.r] > self.Bs[self.r]

    def owner(self, k: int) -> int:
        return (self.r + k) % self.W


def round_up(x: int, m: int) -> int:
    return ceil_div(x, m) * m


def sigma_panels(c: Ctx) -> Tuple[int, int]:
    """(panel rows, panels) of the fused step (sigma_panels with fused_buffers; the budget must hold one panel)."""
    R, Rp, Tp = c.Rs[c.r], round_up(max(c.Rs), 256), round_up(max(c.Ts), 256)
    nbuf = 2 if c.W > 1 else 1
    row_bytes = nbuf * Tp * 2
    budget = c.budget_mib * 1024 * 1024
    if c.budget_mib <= 0 or Rp * row_bytes <= budget:
        return R, 1
    unit = 128 * c.cs
    P = budget // row_bytes // unit * unit
    assert P > 0, "budget below one minimal panel"
    rows = min(P, R)
    return rows, ceil_div(R, rows)


def grad_tile_cols(c: Ctx, M0: int, M1: int, num_sms: int = NUM_SMS) -> int:
    if c.split_k != 0 and c.mcast == 1:
        return TILE
    if c.tile_n != 0:
        return c.tile_n
    units = max(num_sms // c.cs, 1)

    def waves(w):
        return ceil_div((ceil_div(M0, 128 * c.cs) + ceil_div(M1, 128 * c.cs)) * ceil_div(c.D, w), units)

    return WIDE_TILE if 18 * waves(WIDE_TILE) <= 10 * waves(TILE) else TILE


def instantiation(c: Ctx, tile_n: int) -> Tuple[int, int, int]:
    """(columns, stages, cluster size) of the kernel launch_gemm runs."""
    if tile_n == WIDE_TILE:
        return WIDE_TILE, WIDE_STAGES, c.cs
    return TILE, 4 if c.stages == 4 else 6, c.cs


ALL_INSTANTIATIONS = sorted({(TILE, s, cs) for s in (4, 6) for cs in (1, 2, 4)} |
                            {(WIDE_TILE, WIDE_STAGES, cs) for cs in (1, 2, 4)})


@dataclass(frozen=True)
class Split:
    S: int                 # K-slices per split tile (0: not split)
    rem: int = 0           # tiles of the ragged last wave
    first: int = 0         # first split tile
    dimg: bool = False     # some dimg tile is split
    dtxt: bool = False


def split_rule(c: Ctx, tile_n: int, probs: List[Tuple[int, int]], clusters: int,
               num_sms: int = NUM_SMS) -> Split:
    """launch_impl's split-K for problems [(M, K)] (N = D) and the grid's cluster count."""
    if not (tile_n == TILE and c.split_k != 0 and c.mcast == 1 and clusters > 1):
        return Split(0)
    tiles = [ceil_div(M, BLOCK_M * c.cs) * ceil_div(c.D, tile_n) for M, _ in probs]
    total = sum(tiles)
    rem = total % clusters
    if rem == 0:
        return Split(0)
    num_kb = ceil_div(min(K for _, K in probs), BLOCK_K)
    S = clusters // rem
    if c.split_k > 1:
        S = min(S, c.split_k)
    if c.split_k < 0:
        S = min(S, 4)
    while S > 1 and num_kb // S < 8:
        S -= 1
    need = rem * (S - 1) * c.cs * BLOCK_M * TILE * 4
    if S < 2 or rem > SPLIT_K_MAX_TILES or need > splitk_ws_bytes(num_sms):
        return Split(0)
    first = total - rem
    return Split(S, rem, first, dimg=first < tiles[0], dtxt=True)


# per-problem epilogue branches of one launch: pos (the fp32 positive-pair term, fix_vec / fix_mat), f16 (fix_f16 with
# fix_mat_scale), short (fix_rows < M: rows without the term), add (add_src), bf16 (bf16 output, else fp32)
PROBLEM_FLAGS = ("pos", "f16", "short", "add", "bf16")
# launch-wide: grad_out folded in, sc (sc_saved: dt' / dbias written), wait (dtxt waits for the in-kernel fold's flag),
# fold (an auxiliary fold job of a peer's contribution runs in the launch)
LAUNCH_FLAGS = ("grad_out", "sc", "wait", "fold")


@dataclass(frozen=True)
class Launch:
    chunk: int             # owner of the text chunk
    r0: int                # first row of the panel
    M: int                 # panel rows (dimg M, dtxt K)
    Bn: int                # the chunk's texts (dimg K, dtxt M)
    flags: Tuple[str, ...]  # "dimg.pos", ..., "dtxt.add", "grad_out", ...
    tile_n: int = 0
    inst: Tuple[int, int, int] = (0, 0, 0)
    split: Split = Split(0)


def _launch(c: Ctx, chunk, r0, M, Bn, own, fix_dtxt, dimg_add, dimg_bf16, dtxt_add, dtxt_bf16, sc, wait, fold,
            clusters: Dict[int, int], num_sms: int) -> Launch:
    B = c.Bs[c.r]
    pos = own and not c.own_pos_ids
    fix_rows = max(B - r0, 0)
    f = []
    for name, p, rows, add, bf in (("dimg", pos, M, dimg_add, dimg_bf16), ("dtxt", pos and fix_dtxt, Bn, dtxt_add,
                                                                             dtxt_bf16)):
        if p:
            f.append(f"{name}.pos")
            if c.f16:
                f.append(f"{name}.f16")
            if fix_rows < rows:
                f.append(f"{name}.short")
        if add:
            f.append(f"{name}.add")
        if bf:
            f.append(f"{name}.bf16")
    for name, on in (("grad_out", c.grad_out), ("sc", sc), ("wait", wait), ("fold", fold)):
        if on:
            f.append(name)
    tn = grad_tile_cols(c, M, Bn, num_sms)
    inst = instantiation(c, tn)
    sp = split_rule(c, tn, [(M, Bn), (Bn, M)], clusters[c.cs], num_sms)
    return Launch(chunk, r0, M, Bn, tuple(f), tn, inst, sp)


def launches(c: Ctx, clusters: Optional[Dict[int, int]] = None, num_sms: int = NUM_SMS) -> List[Launch]:
    """Every gradient launch of the step, in launch order (fused_impl / backward_impl)."""
    cl = H100_CLUSTERS if clusters is None else clusters
    W, r, R, T = c.W, c.r, c.Rs[c.r], c.Ts[c.r]
    bf = c.bf16
    out = []
    if c.sched == "split":
        assert c.budget_mib == 0, "the split step keeps whole operands"
        for j in range(1, W + 1):
            k = j if j < W else 0
            last = j == W
            out.append(_launch(c, c.owner(k), 0, R, c.Ts[c.owner(k)], k == 0, True, j > 1, last and bf, False,
                               W == 1 and bf, last, False, W > 1 and c.overlap_reduce and j >= 2, cl, num_sms))
        return out
    P, n = sigma_panels(c)
    prow = [min(P, R - p * P) for p in range(n)]
    for p in range(n - 1, 0, -1):       # own panels past 0
        out.append(_launch(c, r, p * P, prow[p], T, True, False, False, W == 1 and bf, p != n - 1, False, False,
                           False, False, cl, num_sms))
    for k in range(1, W):               # remote chunks, panel by panel; the last one runs its panel 0 last
        ck = c.owner(k)
        order = list(range(1, n)) + [0] if k == W - 1 else list(range(n))
        for q, p in enumerate(order):
            rows_final = p > 0 and k == W - 1
            out.append(_launch(c, ck, p * P, prow[p], c.Ts[ck], False, True, k > 1 or p > 0, rows_final and bf,
                               q > 0, False, False, False, k >= 2 and q == 0, cl, num_sms))
    out.append(_launch(c, r, 0, prow[0], T, True, True, W > 1, bf, W > 1 or n > 1, bf, True, W > 1, W > 1, cl,
                       num_sms))
    return out


def problem_combos(flags: Tuple[str, ...]) -> List[Tuple[str, Tuple[str, ...]]]:
    """The epilogue branches of each problem of a launch: ("dimg", its flags), ("dtxt", its flags and wait)."""
    return [(p, tuple(f for f in flags if f.startswith(p + ".") or (p == "dtxt" and f == "wait")))
            for p in ("dimg", "dtxt")]


def step_grid() -> List[Ctx]:
    """Steps over every option that chooses a gradient branch, at shapes where each option is live (a budget below the
    whole operands panels the step): W, schedule, extra images, hard negatives, INPUT_F16, GRAD_BF16, row panels,
    grad_out and, for the split backward, the in-kernel fold against the reduce-slots variant."""
    out = []
    for W, sched, E, K, f16, bf16, panels, grad_out, reduce in itertools.product(
            (1, 2, 3), ("fused", "split"), (0, 40), (0, 70), (False, True), (False, True), (False, True),
            (False, True), (True, False)):
        if (sched == "split" and panels) or (sched == "fused" and not reduce):
            continue
        B = 700 if W > 1 else 600
        out.append(Ctx((B,) * W, (B + E,) + (B,) * (W - 1), (B + K,) * W, 136, f16=f16, bf16=bf16,
                       budget_mib=(2 if W > 1 else 1) if panels else 0, sched=sched, grad_out=grad_out,
                       overlap_reduce=reduce))
    return out


def edges(L: Launch, c: Ctx) -> Tuple[str, ...]:
    """Tile edges of a launch: a 4-CTA cluster tile over at most 384 rows (CTAs of padding only), N = D below one
    tile, K below one k block, a split problem whose last slice ends inside a k block."""
    e = []
    for name, M, K, split in (("dimg", L.M, L.Bn, L.split.dimg), ("dtxt", L.Bn, L.M, L.split.dtxt)):
        if c.cs == 4 and M <= 384:
            e.append(f"{name}.pad_ctas")
        if K < BLOCK_K:
            e.append(f"{name}.k_below_block")
        if split and K % BLOCK_K:
            e.append(f"{name}.split_partial_kb.S{L.split.S}")
    if c.D < L.tile_n:
        e.append("n_below_tile")
    return tuple(e)


# ---------------------------------------------------------------------------------------------------------------------
# cells
# ---------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Cell:
    name: str
    ctx: Ctx
    regime: str = "trained"
    seed: int = 0


def _c(name, B, D, cg=2, mcast=1, regime="trained", W=1, E=0, K=0, **kw) -> Cell:
    """A cell of W ranks of batch B (rank 0 with E extra images and K hard-negative texts; every rank's chunk has K)."""
    Bs = (B,) * W
    Rs = (B + E,) + (B,) * (W - 1)
    Ts = (B + K,) * W
    return Cell(name, Ctx(Bs, Rs, Ts, D, cg=cg, mcast=mcast, **kw), regime, seed=len(name) * 1009 + B + D)


def _cells() -> List[Cell]:
    cells = []
    # the smallest batch the engine accepts, M around one, two, three and four 128-row blocks, at each cluster size
    for cg, mc in ((1, 1), (2, 1), (2, 2)):
        cs = cg * mc
        for B in (1, 17, 127, 128, 129, 255, 256, 257, 383, 511, 512, 513, 1000):
            cells.append(_c(f"M{B}-cs{cs}", B, 136 if B % 2 else 120, cg, mc,
                            regime="t300" if B % 3 == 0 else "trained", tile_n=0 if B > 500 else 128,
                            stages=4 if B in (17, 255, 513) else 0))
    # D below, at and past one tile, 8 valid columns of a 256-wide tile, at each width
    for D in (8, 16, 120, 136, 248, 264, 392):
        for tn, cg, mc in ((128, 1, 1), (256, 2, 1), (256, 2, 2)):
            cells.append(_c(f"D{D}-tn{tn}-cs{cg * mc}", 200, D, cg, mc, tile_n=tn, regime="t300" if D > 200 else
                            "trained"))
    # K = T_c or R below, at and just past one k block (dtxt K = panel rows, dimg K = the chunk's texts)
    for B in (40, 64, 65):
        for cg, mc, tn in ((1, 1, 128), (2, 2, 256), (1, 2, 128)):
            cells.append(_c(f"K{B}-cs{cg * mc}-tn{tn}", B, 136, cg, mc, tile_n=tn))
    # every branch at every instantiation: W = 2 and 3 loopback steps, extras, panels, f16, bf16 outputs, grad_out
    for tn, st in ((128, 4), (128, 6), (256, 0)):
        for cg, mc in ((1, 1), (2, 1), (2, 2)):
            tag = f"tn{tn}-st{st}-cs{cg * mc}"
            cells.append(_c(f"W3-fused-panels-xi-f16-bf16-{tag}", 700, 136, cg, mc, W=3, E=40, tile_n=tn, stages=st,
                            f16=True, bf16=True, budget_mib=2, grad_out=True))
            cells.append(_c(f"W2-fused-hn-{tag}", 300, 136, cg, mc, W=2, K=70, tile_n=tn, stages=st,
                            regime="t300"))
            cells.append(_c(f"W1-panels-xi-f16-{tag}", 600, 136, cg, mc, E=50, tile_n=tn, stages=st, f16=True,
                            budget_mib=1, bf16=True))
            cells.append(_c(f"W3-split-xi-hn-{tag}", 200, 136, cg, mc, W=3, E=30, K=20, tile_n=tn, stages=st,
                            sched="split", grad_out=True, bf16=True))
            cells.append(_c(f"W2-split-noreduce-f16-{tag}", 200, 136, cg, mc, W=2, K=20, tile_n=tn, stages=st,
                            sched="split", f16=True, overlap_reduce=False))
    # every per-problem branch combination a step can produce: the first configuration of step_grid that adds one,
    # on the instantiations in turn
    seen = {pc for cell in cells for L in launches(cell.ctx) for pc in problem_combos(L.flags)}
    insts = [(128, 4, 1, 1), (128, 6, 2, 1), (256, 0, 2, 2), (128, 4, 2, 1), (256, 0, 1, 1), (128, 6, 2, 2),
             (128, 4, 2, 2), (128, 6, 1, 1), (256, 0, 2, 1)]
    for c0 in step_grid():
        for i in range(len(insts)):   # the next instantiation whose panels give this step something new
            tn, st, cg, mc = insts[(len(cells) + i) % len(insts)]
            c = replace(c0, tile_n=tn, stages=st, cg=cg, mcast=mc)
            new = {pc for L in launches(c) for pc in problem_combos(L.flags)} - seen
            if new:
                break
        if not new:
            continue
        seen |= new
        tag = (f"W{c.W}-{c.sched}-E{c.Rs[0] - c.Bs[0]}-K{c.Ts[0] - c.Bs[0]}-f16{int(c.f16)}-bf16{int(c.bf16)}"
               f"-P{int(c.budget_mib > 0)}-g{int(c.grad_out)}-red{int(c.overlap_reduce)}")
        cells.append(Cell(f"branches-{tag}-tn{tn}-st{st}-cs{cg * mc}", c, "trained", seed=len(cells)))
    # split-K: S = 2, 3, 4 at cluster sizes 1 and 2 on the dimg and dtxt problems, slices ending inside a k block
    for name, B, D, cg, sk in (("S4-cs1", 2000, 128, 1, -1), ("S4-cs1-kb", 2048, 128, 1, 4),
                               ("S2-cs1", 1000, 264, 1, -1), ("S3-cs1", 2100, 120, 1, -1),
                               ("S2-cs2", 1100, 264, 2, 2),
                               ("S3-cs2", 2200, 120, 2, -1), ("S4-cs2", 2000, 120, 2, -1),
                               ("S1-cs1", 520, 264, 1, -1)):
        cells.append(_c(f"splitk-{name}", B, D, cg, 1, split_k=sk, regime="t300" if B % 3 == 0 else "trained"))
    return cells


CELLS: List[Cell] = _cells()


# ---------------------------------------------------------------------------------------------------------------------
# the float64 oracle of one rank's step: closed_form_weighted / split_own_diagonal generalised to extra images (rows
# past B_r, never positive, divisor B_r)
# ---------------------------------------------------------------------------------------------------------------------
def oracle(imgs: List[np.ndarray], texts: List[np.ndarray], Bs, r: int, t_prime: float, bias: float,
           grad_out: float = 1.0) -> Dict:
    """Rank r's loss, dimg [R_r, D], contrib[c] [T_c, D], dt', dbias, and the parts through G: rest_dimg, rest_contrib (own
    chunk) — everything but the fp32 own-diagonal term t g_ii of the first B_r rows."""
    from oracle.siglip_oracle import _sigmoid

    t = math.exp(t_prime)
    img, B = np.asarray(imgs[r], np.float64), Bs[r]
    res = dict(loss=0.0, dimg=np.zeros_like(img), contrib=[], dt_prime=0.0, dbias=0.0, sum_abs_g=0.0, sum_abs_gs=0.0)
    for c, txt in enumerate(texts):
        txt = np.asarray(txt, np.float64)
        s = img @ txt.T
        y = -np.ones_like(s)
        if c == r:
            y[np.arange(B), np.arange(B)] = 1.0
        res["loss"] += float(np.logaddexp(0.0, -y * (t * s + bias)).sum() / B)
        G = grad_out * (-y * _sigmoid(-y * (t * s + bias))) / B
        res["dimg"] += t * (G @ txt)
        if c != r:
            res["rest_dimg"] = res.get("rest_dimg", 0.0) + t * (G @ txt)
        res["contrib"].append(t * (G.T @ img))
        res["dt_prime"] += float(t * (G * s).sum())
        res["dbias"] += float(G.sum())
        res["sum_abs_g"] += float(np.abs(G).sum())
        res["sum_abs_gs"] += float(t * np.abs(G * s).sum())
        if c == r:
            gd = np.diagonal(G[:, :B]).copy()
            Gr = G.copy()
            Gr[np.arange(B), np.arange(B)] = 0.0
            res["rest_contrib"] = t * (Gr.T @ img)
            res["rest_dimg"] = res.get("rest_dimg", 0.0) + t * (Gr @ txt)
            res["diag_dimg"] = np.zeros_like(img)
            res["diag_dimg"][:B] = t * gd[:, None] * txt[:B]
    return res


def cell_inputs(cell: Cell):
    """(imgs [R_p, D], texts [T_p, D]) per rank from tests/trained_regime.py (bf16-representable unit rows), t', bias.
    Extra images are further images of the same regime; without ids every pair they form is a negative."""
    import torch

    from trained_regime import REGIMES, make_batch

    c = cell.ctx
    R = REGIMES[cell.regime]
    E = [rp - bp for rp, bp in zip(c.Rs, c.Bs)]
    K = [tp - bp for tp, bp in zip(c.Ts, c.Bs)]
    imgs, texts, _, _ = make_batch(R, [b + e for b, e in zip(c.Bs, E)], K, c.D, cell.seed, "pos")
    # make_batch pairs every image with a text: drop the texts of the extra images (the paired B come first)
    texts = [torch.cat([t[:b], t[b + e:]]) for t, b, e in zip(texts, c.Bs, E)]
    imgs = [x.float().numpy().astype(np.float64) for x in imgs]
    texts = [x.float().numpy().astype(np.float64) for x in texts]
    if c.f16:   # the operands are fp16(16 x): the oracle sees exactly what the kernels read
        imgs = [(x * X_SCALE).astype(np.float16).astype(np.float64) / X_SCALE for x in imgs]
        texts = [(x * X_SCALE).astype(np.float16).astype(np.float64) / X_SCALE for x in texts]
    return imgs, texts, float(np.float32(R.t_prime)), float(np.float32(R.bias))
