"""The loss kernel's persistent tile schedule, restated from csrc/siglip_kernels.cu (launch_impl, decode_tile and the
producer / consumer loops of siglip_gemm_kernel) — test infrastructure, never the product path.

One loss launch scores a rows x cols window (slab_paths.windows) in cluster tiles: kCS vertically adjacent 128-row
blocks against one 128-column block, in row-panel order (tile t: row panel t / tiles_n, column block t % tiles_n, CTA
crank of the cluster on row block (t / tiles_n) kCS + crank). A row block at or past the window's last row is a phantom:
fully masked, but its CTA still streams its share of the B tile and releases the ring for the cluster. The grid is
min(co-resident clusters, num_sms / kCS, grid tiles), where the grid tiles count grid_n columns when the step's largest
chunk is wider than the launch (KernelParams::grid_n: every chunk of a forward launches the same grid, so a narrower
chunk leaves clusters with fewer tiles or none). Cluster c runs tiles c, c + clusters, c + 2 clusters, ...

The producer and the consumers step one ring of `stages` stages through every k-block of every tile of the CTA (the
teacher's k-blocks first in the teacher modes), stage and phase running on across tiles: the tile of ordinal j of a
CTA starts at ring position g = j num_kb, stage g % stages, phase (g / stages) % 2."""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Tuple

TILE, KBLK = 128, 64
NUM_SMS = 132                            # H100 SXM
H100_CLUSTERS = {1: 132, 2: 66, 4: 30}   # co-resident clusters per cluster size (loss and gradient kernels alike)


def num_kb(d: int, d_teacher: int = 0) -> int:
    """k-blocks of one tile: ceil(D / 64), plus ceil(D_T / 64) of the teacher pass in the teacher modes."""
    return -(-d // KBLK) + (-(-d_teacher // KBLK) if d_teacher else 0)


@dataclass(frozen=True)
class Tile:
    """One cluster tile of a cluster's list: its row panel and column block, and where the ring stands at its first
    k-block."""
    mrow: int
    n_blk: int
    stage: int
    phase: int


@dataclass
class Launch:
    rows: int
    cols: int
    cs: int
    stages: int
    num_kb: int
    clusters: int
    tiles_m: int
    tiles_n: int
    per_cluster: List[List[Tile]]

    def m_blk(self, tile: Tile, crank: int) -> int:
        return tile.mrow * self.cs + crank

    def phantom(self, tile: Tile, crank: int) -> bool:
        return self.m_blk(tile, crank) * TILE >= self.rows

    def cta_tiles(self, cluster: int, crank: int) -> List[Tuple[int, int, int, int, bool]]:
        """(m_blk, n_blk, stage, phase, phantom) of every tile CTA crank of the cluster scores, in order."""
        return [(self.m_blk(t, crank), t.n_blk, t.stage, t.phase, self.phantom(t, crank))
                for t in self.per_cluster[cluster]]

    @property
    def total(self) -> int:
        return self.tiles_m * self.tiles_n

    def max_tiles(self) -> int:
        return max(len(x) for x in self.per_cluster)

    def ragged(self) -> bool:
        """The last wave leaves clusters idle: not every cluster runs the same number of tiles."""
        return len({len(x) for x in self.per_cluster}) > 1

    def keeps_row_block(self) -> bool:
        """Some cluster's consecutive tiles lie in one row panel (its CTAs keep their rows)."""
        return any(a.mrow == b.mrow for x in self.per_cluster for a, b in zip(x, x[1:]))

    def changes_row_block(self) -> bool:
        return any(a.mrow != b.mrow for x in self.per_cluster for a, b in zip(x, x[1:]))

    def later_tiles(self):
        """(ordinal, previous tile, tile) of every tile after a cluster's first."""
        return [(j, x[j - 1], x[j]) for x in self.per_cluster for j in range(1, len(x))]

    def mid_ring(self) -> bool:
        """Some tile starts at a stage other than 0."""
        return any(t.stage for x in self.per_cluster for t in x)

    def phase_one(self) -> bool:
        return any(t.phase for x in self.per_cluster for t in x)

    def phantom_after_real(self) -> bool:
        """Some CTA scores a real block and then a phantom one."""
        return any(not self.phantom(a, k) and self.phantom(b, k)
                   for x in self.per_cluster for a, b in zip(x, x[1:]) for k in range(self.cs))

    def phantom_then_more(self) -> bool:
        """Some cluster scores a tile that holds a phantom block and then another tile: the phantom CTA keeps streaming
        its share of B and releasing the ring for its siblings."""
        return any(any(self.phantom(a, k) for k in range(self.cs)) for x in self.per_cluster for a in x[:-1])

    def phantom_before_real(self) -> bool:
        """Some CTA scores a phantom block and then a real one: never, the last row panel comes last in the order."""
        return any(self.phantom(a, k) and not self.phantom(b, k)
                   for x in self.per_cluster for a, b in zip(x, x[1:]) for k in range(self.cs))


def launch(rows: int, cols: int, cs: int, stages: int, kb: int, co_resident: int, grid_n: Optional[int] = None,
           num_sms: int = NUM_SMS) -> Launch:
    """The schedule of one loss launch of rows x cols at cluster size cs with `stages` ring stages and kb k-blocks per
    tile (num_kb), on a device with co_resident clusters of the instantiation; grid_n the step's widest chunk."""
    tiles_m = -(-rows // (TILE * cs))
    tiles_n = -(-cols // TILE)
    total = tiles_m * tiles_n
    clusters = min(co_resident, num_sms // cs)
    grid_tiles = total
    if grid_n is not None and grid_n > cols:
        grid_tiles = tiles_m * -(-grid_n // TILE)
    clusters = max(1, min(clusters, grid_tiles))
    per = []
    for c in range(clusters):
        tiles = []
        for j, t in enumerate(range(c, total, clusters)):
            g = j * kb
            tiles.append(Tile(t // tiles_n, t % tiles_n, g % stages, (g // stages) % 2))
        per.append(tiles)
    return Launch(rows, cols, cs, stages, kb, clusters, tiles_m, tiles_n, per)
