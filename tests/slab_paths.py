"""Which path each 16x32 slab of the loss kernel's epilogue takes, restated from csrc/siglip_kernels.cu — test
infrastructure, never the product path (tests/test_option_matrix_cpu.py pins it and derives the option matrix's
coverage of the series path from it; trained_regime.slab_fast_fraction counts with it).

The loss kernel scores 128 x 128 tiles; each consumer warp walks a 16-row band of its tile in 4 slabs of 32 columns
(the kModeLoss epilogue, sample_loss_epilogue and distill_epilogue). A slab is
  edge  when it crosses the launch's last row or column (slab_edge: the elements past the matrix are masked),
  diag  when it overlaps the own positional diagonal inside a diagonal tile (slab_diag: own_chunk and row0 == col_base),
  pos   when it holds a positive of sample ids, extra ids or label sets (slab_pos, the lpos pre-pass),
  excl  when it holds an excluded same-group pair (slab_excl),
  free  otherwise.
A free slab takes the series path (loss_slab_fast, focal_slab_fast) when the warp vote fmaf(max s, t_eff, bias) <
kFastZ holds in fp32, the general path (loss_slab<false>, focal_slab) when it does not; the other classes take the
masked general path whatever z is. The teacher modes vote in every slab, whatever its class (distill_slab_series): the
student on its accumulator and the teacher on its own in the pre-pass. Elements past the matrix hold s = 0 there (the
TMA fills them with zeros). t_eff is t for bf16 operands and t / 256 on the 2^8 s accumulator of fp16(16 x) operands:
the same product in fp32, so the vote does not depend on the operand format.

Metrics and top-K keys are taken from the raw accumulator before the path choice (tile_metrics, tile_topk), so
retrieval does not depend on the path.

One loss launch scores rows [r0, r0 + rows) of the rank against columns [c0, c0 + cols) of a text chunk
(run_loss_chunk's Window): the whole chunk, or under row panels each panel's rows, the own chunk's panels past 0 in
two launches split at column p0 (the diagonal window from p0 on, the columns before it without a diagonal). Local
coordinates start at the window's origin, a multiple of 128, so the slab grid is the global one."""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import numpy as np

SLAB_ROWS, SLAB_COLS, TILE = 16, 32, 128
FAST_Z = float(np.float32(-4.2))   # kFastZ
MARGIN = 1e-5                      # a counted vote is this far from kFastZ: the model is exact away from the boundary
EDGE, DIAG, POS, EXCL, FREE = "edge", "diag", "pos", "excl", "free"
CLASSES = (EDGE, DIAG, POS, EXCL, FREE)


def t_eff(t_prime: float, f16: bool = False) -> float:
    """The fp32 scale of the vote: expf(t') (x 2^-8 on the fp16(16 x) accumulator)."""
    t = float(np.float32(math.exp(float(np.float32(t_prime)))))
    return t / 256.0 if f16 else t


def vote(smax, t_prime: float, bias: float, f16: bool = False):
    """fmaf(max acc, t_eff, bias) in fp32 for the slabs' max <img, txt> (float64 exact): one rounding of the exact
    product and sum. acc = 256 s for fp16(16 x) operands, t_eff = t / 256: the same product."""
    acc = np.asarray(smax, np.float64) * (256.0 if f16 else 1.0)
    return (acc * t_eff(t_prime, f16) + float(np.float32(bias))).astype(np.float32)


@dataclass
class SlabMap:
    """The slabs of one launch: cls [nb, nc] (CLASSES), z [nb, nc] the student's vote value, zt the teacher's (teacher
    modes), series / tseries whether the student's / teacher's vote passes, and the window the launch scores."""
    cls: np.ndarray
    z: np.ndarray
    zt: Optional[np.ndarray]
    chunk: int
    r0: int
    c0: int
    rows: int
    cols: int

    @property
    def series(self):
        return self.z < FAST_Z

    @property
    def tseries(self):
        return None if self.zt is None else self.zt < FAST_Z

    def student_path(self, teacher: bool):
        """'series' / 'general' per slab: a free slab's vote outside the teacher modes; the vote of every slab in them."""
        ser = self.series if teacher else self.series & (self.cls == FREE)
        return np.where(ser, "series", "general")

    def min_margin(self, teacher: bool) -> float:
        """The smallest |z - kFastZ| over the votes that decide a path (and the teacher's)."""
        m = np.abs(self.z.astype(np.float64) - FAST_Z)
        m = m if teacher else m[self.cls == FREE]
        out = float(m.min()) if m.size else math.inf
        if self.zt is not None:
            out = min(out, float(np.abs(self.zt.astype(np.float64) - FAST_Z).min()))
        return out

    def elements(self, slabs: np.ndarray) -> np.ndarray:
        """[rows, cols] mask of the launch's elements that lie in the given slabs ([nb, nc] bool)."""
        full = np.repeat(np.repeat(slabs, SLAB_ROWS, axis=0), SLAB_COLS, axis=1)
        return full[:self.rows, :self.cols]


def _slab_max(s: np.ndarray) -> np.ndarray:
    """Max over each 16x32 slab of s, the elements past the matrix read as 0."""
    M, N = s.shape
    nb, nc = -(-M // SLAB_ROWS), -(-N // SLAB_COLS)
    pad = np.zeros((nb * SLAB_ROWS, nc * SLAB_COLS))
    pad[:M, :N] = s
    return pad.reshape(nb, SLAB_ROWS, nc, SLAB_COLS).max(axis=(1, 3))


def _slab_any(mask: np.ndarray) -> np.ndarray:
    M, N = mask.shape
    nb, nc = -(-M // SLAB_ROWS), -(-N // SLAB_COLS)
    pad = np.zeros((nb * SLAB_ROWS, nc * SLAB_COLS), bool)
    pad[:M, :N] = mask
    return pad.reshape(nb, SLAB_ROWS, nc, SLAB_COLS).any(axis=(1, 3))


def classes(M: int, N: int, own_chunk: bool, y: np.ndarray) -> np.ndarray:
    """[nb, nc] class of every slab of an M x N launch; y [M, N] the launch's labels (+1 positive, 0 excluded, -1
    negative). The own positional diagonal is the geometry's, not y's: own_chunk is off for an own chunk that takes its
    positives from (iota) ids."""
    nb, nc = -(-M // SLAB_ROWS), -(-N // SLAB_COLS)
    band = (np.arange(nb) * SLAB_ROWS)[:, None]
    col0 = (np.arange(nc) * SLAB_COLS)[None, :]
    edge = (band + SLAB_ROWS > M) | (col0 + SLAB_COLS > N)
    diag = own_chunk & (band // TILE == col0 // TILE) & (band < col0 + SLAB_COLS) & (col0 < band + SLAB_ROWS)
    pos, excl = _slab_any(y > 0), _slab_any(y == 0)
    cls = np.full((nb, nc), FREE, dtype=object)
    cls[excl] = EXCL
    cls[pos] = POS
    cls[diag] = DIAG
    cls[edge] = EDGE
    return cls


def windows(R: int, B: int, T: int, own: bool, own_pos_ids: bool, panel_rows: int):
    """(r0, rows, c0, cols, own_chunk) of the loss launches over one text chunk of T columns (run_fwd_bwd /
    run_loss_chunk): one launch per row panel of panel_rows rows; the own chunk's panels past 0 that hold paired rows
    twice, at column p0 with the diagonal and before it without. own_chunk is off where the own chunk takes its
    positives from iota ids (extras of both kinds, own_pos_ids)."""
    out = []
    for p0 in range(0, R, panel_rows):
        rows = min(panel_rows, R - p0)
        if own and p0 > 0 and p0 < B and not own_pos_ids:
            out += [(p0, rows, p0, T - p0, True), (p0, rows, 0, p0, False)]
        else:
            out.append((p0, rows, 0, T, own and p0 < B and not own_pos_ids))
    return out


def slab_map(s, y, own_chunk: bool, t_prime: float, bias: float, f16: bool = False, ts=None, t_prime_T=None,
             bias_T=None, chunk: int = 0, r0: int = 0, c0: int = 0) -> SlabMap:
    """The slabs of one launch: s [M, N] its <img, txt> (float64), y its labels, ts the teacher's <timg, ttxt>."""
    M, N = s.shape
    zt = None if ts is None else vote(_slab_max(ts), t_prime_T, bias_T, f16)
    return SlabMap(classes(M, N, own_chunk, y), vote(_slab_max(s), t_prime, bias, f16), zt, chunk, r0, c0, M, N)
