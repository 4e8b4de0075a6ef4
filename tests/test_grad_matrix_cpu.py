"""The gradient kernel's coverage, derived on the CPU from tests/grad_matrix.py with H100 SXM constants (132 SMs; 132
and 66 co-resident clusters at cluster sizes 1 and 2): the cells reach every kModeOut instantiation, every reachable
combination of run_grad_chunk's epilogue branches, each branch at every instantiation, split-K with S = 2, 3 and 4 at
cluster sizes 1 and 2 on the dimg and the dtxt problem, and the tile edges. `pytest -s` prints what it derives."""
import ctypes
import os
import re

import pytest

import grad_matrix as gm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNELS = os.path.join(ROOT, "distributed_sigmoid_loss_b200", "csrc", "siglip_kernels.cu")


def _rowclass(M, cs):
    """Where M ends in a CTA's 128-row block, and how many such blocks (capped)."""
    u = gm.BLOCK_M
    r = M % u
    return min(gm.ceil_div(M, u), 8), {0: "full", 1: "one", u - 1: "minus1"}.get(r, "mid")


def _kclass(K):
    """k blocks of a contraction (capped) and whether the last one is whole."""
    return min(gm.ceil_div(K, gm.BLOCK_K), 3), K % gm.BLOCK_K == 0


def _keys(cell, clusters=gm.H100_CLUSTERS):
    """The fine coverage of a cell: per launch its instantiation, branch flags, split and tile edges, with the shape
    classes of its two problems."""
    c = cell.ctx
    out = set()
    for L in gm.launches(c, clusters):
        out.add((L.inst, L.flags, (L.split.S, L.split.dimg), gm.edges(L, c), _rowclass(L.M, c.cs),
                 _rowclass(L.Bn, c.cs), _kclass(L.M), _kclass(L.Bn), c.D % L.tile_n, c.D // L.tile_n))
    return out


def coverage(cells, clusters=gm.H100_CLUSTERS):
    """(instantiations, branch combinations per instantiation, (instantiation, flag) pairs, split facts, edges)."""
    insts, combos, pairs, splits, edges = set(), set(), set(), set(), set()
    for cell in cells:
        c = cell.ctx
        for L in gm.launches(c, clusters):
            insts.add(L.inst)
            combos.update((L.inst, fs) for fs in problem_combos(L.flags))
            pairs.update((L.inst, f) for f in L.flags)
            if L.split.S:
                if L.split.dimg:
                    splits.add((L.split.S, c.cs, "dimg"))
                splits.add((L.split.S, c.cs, "dtxt"))
            edges.update(gm.edges(L, c))
    return insts, combos, pairs, splits, edges


problem_combos = gm.problem_combos


def reachable_flag_sets():
    """Every branch combination some step of gm.step_grid produces."""
    return {L.flags for c in gm.step_grid() for L in gm.launches(c)}


ALL_FLAGS = tuple(f"{p}.{f}" for p in ("dimg", "dtxt") for f in gm.PROBLEM_FLAGS) + gm.LAUNCH_FLAGS


def _derive(clusters=gm.H100_CLUSTERS):
    insts, combos, pairs, splits, edges = coverage(gm.CELLS, clusters)
    missing = []
    missing += [f"instantiation {i}" for i in gm.ALL_INSTANTIATIONS if i not in insts]
    got = {f for _, f in combos}
    want = {pc for f in reachable_flag_sets() for pc in problem_combos(f)}
    missing += [f"branch combination {f}" for f in sorted(want) if f not in got]
    used = {f for fs in reachable_flag_sets() for f in fs}
    missing += [f"flag {f} at {i}" for i in gm.ALL_INSTANTIATIONS for f in sorted(used) if (i, f) not in pairs]
    missing += [f"split-K S={S} cluster size {cs} on {p}" for S in (2, 3, 4) for cs in (1, 2) for p in ("dimg", "dtxt")
                if (S, cs, p) not in splits]
    want_edges = {"dimg.pad_ctas", "dtxt.pad_ctas", "dimg.k_below_block", "dtxt.k_below_block", "n_below_tile"}
    want_edges |= {f"{p}.split_partial_kb.S{S}" for p in ("dimg", "dtxt") for S in (2, 3, 4)}
    missing += [f"edge {e}" for e in sorted(want_edges - edges)]
    return missing, (insts, combos, pairs, splits, edges)


def test_model_flags_are_the_known_branches():
    for f in reachable_flag_sets():
        assert set(f) <= set(ALL_FLAGS), f
    assert {f for fs in reachable_flag_sets() for f in fs} == set(ALL_FLAGS)


def test_cells_cover_every_instantiation_branch_and_split():
    missing, (insts, combos, pairs, splits, edges) = _derive()
    print(f"\ngrad matrix: {len(gm.CELLS)} cells, {sum(len(gm.launches(c.ctx)) for c in gm.CELLS)} launches")
    print(f"  instantiations (columns, stages, cluster): {sorted(insts)}")
    want = {pc for f in reachable_flag_sets() for pc in problem_combos(f)}
    print(f"  per-problem branch combinations: {len({f for _, f in combos})} of {len(want)} reachable; "
          f"(instantiation, combination) pairs {len(combos)}; (instantiation, flag) pairs {len(pairs)}")
    print(f"  split-K (S, cluster size, problem): {sorted(splits)}")
    print(f"  edges: {sorted(edges)}")
    assert not missing, "not covered: " + "; ".join(missing)


def test_no_cell_is_redundant():
    keys = [_keys(c) for c in gm.CELLS]
    for k, cell in enumerate(gm.CELLS):
        rest = set().union(*(keys[:k] + keys[k + 1:]))
        assert not keys[k] <= rest, f"{cell.name} covers nothing no other cell covers"
    assert len({c.name for c in gm.CELLS}) == len(gm.CELLS)


def test_every_split_cell_splits_and_the_control_does_not():
    for cell in gm.CELLS:
        if cell.ctx.split_k == 0:
            continue
        S = [L.split.S for L in gm.launches(cell.ctx)]
        if cell.name.startswith("splitk-S1"):
            assert S == [0], cell.name
        else:
            assert all(s == int(cell.name.split("-")[1][1]) for s in S), (cell.name, S)


def test_kernel_list_matches_launch_gemm():
    """The out-kernel instantiations launch_gemm dispatches to (the 8-bit measurement path apart) are exactly the ones
    the matrix knows: a new gradient instantiation fails here until the matrix covers it."""
    src = open(KERNELS).read()
    body = src[src.index("int launch_gemm("):]
    body = body[:body.index("\n}\n")]
    stages = {"kWideStages": gm.WIDE_STAGES}
    found = set()
    for m in re.finditer(r"launch_impl<kModeOut,\s*(\w+),\s*(\d)((?:,\s*\w+)*)>", body):
        extra = [a.strip() for a in m.group(3).split(",") if a.strip()]
        if extra and extra[0] == "true":       # kF8: the fp8 measurement path
            continue
        tile = gm.WIDE_TILE if extra and extra[-1] == "kWideTileN" else gm.TILE
        found.add((tile, int(stages.get(m.group(1), m.group(1))), int(m.group(2))))
    for m in re.finditer(r"SIGLIP_LAUNCH_STAGES\(kModeOut,\s*(\d)\)", body):
        found.update({(gm.TILE, 4, int(m.group(1))), (gm.TILE, 6, int(m.group(1)))})
    assert re.search(r"if \(stages == 4\) SIGLIP_LAUNCH\(MODE, 4, CS\);\s*\\\s*SIGLIP_LAUNCH\(MODE, 6, CS\);", src)
    assert re.search(r"constexpr int kWideStages = %d;" % gm.WIDE_STAGES, src)
    assert found == set(gm.ALL_INSTANTIATIONS), sorted(found)


def test_panel_rule_matches_the_library():
    """The matrix's row panels against siglip_sigma_panel_rows (host code of the built library)."""
    from distributed_sigmoid_loss_b200 import _capi

    L = _capi.lib()
    for cell in gm.CELLS:
        c = cell.ctx
        if c.sched != "fused":
            continue
        P, n = gm.sigma_panels(c)
        buf = ctypes.c_int()
        got = L.siglip_sigma_panel_rows(c.Rs[c.r], gm.round_up(max(c.Rs), 256), gm.round_up(max(c.Ts), 256),
                                        2 if c.W > 1 else 1, 128 * c.cs, c.budget_mib, ctypes.byref(buf))
        assert got == P, (cell.name, got, P)
        if c.budget_mib:
            assert n > 1, f"{cell.name}: the budget does not panel the step"


@pytest.mark.parametrize("counts", [{1: 132, 2: 66, 4: 32}, {1: 132, 2: 60, 4: 30}])
def test_split_rule_is_monotone_in_the_request(counts):
    """An explicit request never splits more than S = clusters // rem, and -1 never more than 4."""
    for cell in gm.CELLS:
        c = cell.ctx
        for L in gm.launches(c, counts):
            if L.split.S:
                assert 2 <= L.split.S <= (4 if c.split_k < 0 else c.split_k)
                assert L.split.S * L.split.rem <= counts[c.cs]
                assert gm.ceil_div(min(L.M, L.Bn), gm.BLOCK_K) // L.split.S >= 8


def test_oracle_is_the_suites_float64_oracle():
    """gm.oracle against closed_form_weighted / split_own_diagonal (hard negatives, W = 2) and closed_form_extras
    (extra images, whose rows have no positive and divide by B)."""
    import numpy as np
    import torch

    from extra_images_oracle import closed_form_extras
    from sample_weights_oracle import closed_form_weighted
    from trained_regime import split_own_diagonal

    cell = gm._c("oracle-hn", 150, 136, W=2, K=30)
    imgs, texts, tp, bias = gm.cell_inputs(cell)
    for r in range(2):
        ref = gm.oracle(imgs, texts, cell.ctx.Bs, r, tp, bias)
        cf = closed_form_weighted(imgs, texts, tp, bias)[r]
        part = split_own_diagonal([torch.from_numpy(x) for x in imgs], [torch.from_numpy(x) for x in texts], tp, bias)[r]
        np.testing.assert_allclose(ref["dimg"], cf["dimg"], rtol=1e-12, atol=1e-15)
        for k in range(2):
            np.testing.assert_allclose(ref["contrib"][k], cf["contrib"][k], rtol=1e-12, atol=1e-15)
        np.testing.assert_allclose(ref["rest_contrib"], part["rest_contrib"], rtol=1e-12, atol=1e-15)
        np.testing.assert_allclose(ref["rest_dimg"], part["rest_dimg"], rtol=1e-12, atol=1e-15)
        assert abs(ref["dbias"] - cf["dbias"]) < 1e-12 and abs(ref["dt_prime"] - cf["dt_prime"]) < 1e-10
    cell = gm._c("oracle-xi", 150, 136, W=2, E=20, f16=True)
    imgs, texts, tp, bias = gm.cell_inputs(cell)
    ref = gm.oracle(imgs, texts, cell.ctx.Bs, 0, tp, bias, 0.5)
    cf = closed_form_extras(imgs, texts, list(cell.ctx.Bs), tp, bias)[0]
    np.testing.assert_allclose(ref["dimg"], 0.5 * cf["dimg"], rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(ref["contrib"][1], 0.5 * cf["contrib"][1], rtol=1e-12, atol=1e-15)
    assert np.all(ref["diag_dimg"][150:] == 0)
