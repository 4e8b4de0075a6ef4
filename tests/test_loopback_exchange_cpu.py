"""The loopback exchange cells (tests/loopback_exchange.py): they reach every fold and pull site with every pulled kind,
none is redundant, and every host-side exchange bug the GPU test is meant to catch moves a checked output by more than
20x the tolerance on the oracle.

Every mutation of every cell meets the bound. Some mutations cannot occur in some cells, and are not counted there: at
W = 2 there is one peer, so no other peer's block to read instead; a rank whose chunk has the fewest texts has no
shorter chunk to be cut at (W = 2 at rank 1, W = 4 at rank 3); and a chunk without extra texts (chunk 1 at W = 3) has
no extra-text ids to leave stale. The other cells meet each of those mutations."""
import pytest

import grad_matrix as gm
import loopback_exchange as lx

FOLD_SITES = ("split.fold.first", "split.fold.first.W2", "split.fold.chain", "split.reduce", "split.reduce.W2",
              "fused.fold.remote", "fused.G0.W2",
              "fused.G0.W3", "fused.fold.remote.panels", "fused.G0.W2.panels", "fused.fold.remote.nosync",
              "fused.G0.W2.nosync", "fused.G0.W3.nosync")
BIDIR_SITES = ("split.fold.first", "split.fold.chain", "fused.fold.remote", "fused.G0.W3")
PULL_KINDS = ("text.bf16", "text.f16", "ids", "xt_ids", "groups", "sets.M1", "sets.M4", "weights", "teacher.distill",
              "teacher.extras")
PULL_SITES = ("fused.L", "split.L", "split.stream")


def _all():
    return set().union(*(lx.coverage(x) for x in lx.CELLS))


def test_fold_sites_match_the_gradient_launch_rules():
    """The in-kernel folds restated here are the launches grad_matrix.launches gives a fold flag, in the same number."""
    for x in lx.CELLS:
        if x.base.sched == "fwd":
            continue
        n = sum("fold" in L.flags for L in gm.launches(lx.grad_ctx(x)))
        in_kernel = [f for f in lx.folds(x) if f.src2 != "slots"]
        assert n == len(in_kernel), (x.name, n, in_kernel)
        # every peer is folded exactly once
        assert sorted(f.peer for f in lx.folds(x)) == [p for p in range(x.base.W) if p != x.base.r], x.name


def test_every_fold_site_is_reached_from_both_sides():
    cov = _all()
    missing = [(s, side) for s in FOLD_SITES for side in ("first", "last")
               if ("fold", s, side, "ring") not in cov]
    missing += [(s, side, "bidir") for s in BIDIR_SITES for side in ("first", "last")
                if ("fold", s, side, "bidir") not in cov]
    for feature in ("fp32", "bf16", "T>B", "R>B"):
        if not any(k[0] == "fold" and k[-1] == feature for k in cov):
            missing.append(feature)
    for s in ("split.fold.first", "split.reduce", "fused.G0.W2", "fused.G0.W3"):
        missing += [(s, f) for f in ("fp32", "bf16", "T>B", "R>B") if ("fold", s, f) not in cov]
    assert not missing, missing


def test_every_pull_site_moves_every_kind():
    cov = _all()
    missing = [(s, k) for s in PULL_SITES for k in PULL_KINDS if ("pull", s, k) not in cov]
    assert not missing, missing
    # the teacher kinds run in the two context types
    assert {lx.om.distill_extras_context(x.base) for x in lx.CELLS if x.base.opts.teacher} == {False, True}


def test_no_cell_is_redundant():
    covs = [lx.coverage(x) for x in lx.CELLS]
    assert len({x.name for x in lx.CELLS}) == len(lx.CELLS)
    for i, x in enumerate(lx.CELLS):
        others = set().union(*(c for j, c in enumerate(covs) if j != i))
        assert covs[i] - others, f"{x.name} reaches nothing the other cells do not"


@pytest.mark.parametrize("x", lx.CELLS, ids=lambda x: x.name)
def test_every_exchange_bug_moves_a_checked_output(x):
    """Per step (the second, whose data the first step's would stand in for): each fold mutation moves dtxt - sum C
    against g own, and each pulled kind of each pulled chunk left at the first step's values moves some checked output,
    by more than 20x the tolerance."""
    bound = lx.SENSITIVITY * lx.TOL
    prev, P = lx.problem(x, 0), lx.problem(x, 1)
    ref = lx.references(x, P)
    own = ref["contrib"][x.base.r]
    C = lx.seeds(x, own, 1)
    for p, blk in C.items():
        assert blk.shape == own.shape and (blk[1:] != blk[:-1]).any(axis=1).all(), "neighbouring rows must differ"
        assert all((blk != C[q]).any(axis=1).all() for q in C if q != p), "peers' rows must differ"
    weak = {k: v for k, v in lx.fold_mutations(x, own, C).items() if v <= bound}
    weak.update({k: v for k, v in lx.pull_mutations(x, prev, P, ref).items() if v <= bound})
    assert not weak, f"{x.name}: below {bound:.2f}: {weak}"
