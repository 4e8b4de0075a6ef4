"""Row panels (SIGLIP_OPT_SIGMA_BUDGET_MIB) without a device: the panel-size rule of siglip_sigma_panel_rows and the
module's argument checks."""
import ctypes

import pytest

from distributed_sigmoid_loss_b200 import _capi
from distributed_sigmoid_loss_b200.loss import _sigma_budget_mib

MIB = 1 << 20


def _rows(R, Rp, Tp, nbuf, unit, budget_mib):
    buf = ctypes.c_int(-1)
    P = _capi.lib().siglip_sigma_panel_rows(R, Rp, Tp, nbuf, unit, budget_mib, ctypes.byref(buf))
    return P, buf.value


def test_unbounded_and_whole_operand_give_one_panel():
    # budget 0, or one that holds nbuf whole [Rp, Tp] operands: one panel of R rows in Rp-row buffers
    assert _rows(3000, 3072, 3072, 1, 256, 0) == (3000, 3072)
    need = 2 * 3072 * 3072 * 2
    assert _rows(3000, 3072, 3072, 2, 256, -(-need // MIB)) == (3000, 3072)


def test_panels_are_multiples_of_the_cluster_rows():
    Tp = 3072
    for nbuf in (1, 2):
        for unit in (128, 256, 512):
            for mib in range(1, 40):
                P, buf = _rows(3000, 3072, Tp, nbuf, unit, mib)
                if P == 0:
                    assert nbuf * unit * Tp * 2 > mib * MIB   # refused only below one minimal panel
                    continue
                assert nbuf * buf * Tp * 2 <= mib * MIB or buf == 3072
                if P < 3000:
                    assert P % unit == 0 and P == buf
                    # the largest such multiple
                    assert nbuf * (P + unit) * Tp * 2 > mib * MIB


def test_ragged_last_panel():
    # B = 3000, Tp = 3072, one buffer, 3 MiB: 512-row panels, 5 full and a last one of 440 rows
    P, buf = _rows(3000, 3072, 3072, 1, 256, 3)
    assert (P, buf) == (512, 512)
    assert 3000 - 5 * P == 440


def test_refusal_below_one_minimal_panel():
    assert _rows(3000, 3072, 3072, 1, 256, 1)[0] == 0     # 256 x 3072 x 2 B = 1.5 MiB > 1 MiB
    assert _rows(3000, 3072, 3072, 2, 256, 2)[0] == 0     # two buffers: 3 MiB
    assert _rows(3000, 3072, 3072, 2, 256, 3)[0] == 256


def test_invalid_arguments():
    L = _capi.lib()
    assert L.siglip_sigma_panel_rows(0, 256, 256, 1, 256, 1, None) == -_capi.SIGLIP_ERR_INVALID
    assert L.siglip_sigma_panel_rows(300, 256, 256, 1, 256, 1, None) == -_capi.SIGLIP_ERR_INVALID
    assert L.siglip_sigma_panel_rows(256, 256, 256, 1, 256, -1, None) == -_capi.SIGLIP_ERR_INVALID


def test_option_number_and_budget_rounding():
    assert _capi.SIGLIP_OPT_SIGMA_BUDGET_MIB == 26
    assert _sigma_budget_mib(None) == 0
    assert _sigma_budget_mib(0) == 0
    assert _sigma_budget_mib(4 * MIB + 123) == 4
    for bad in (-1, 1.5, True, MIB - 1):
        with pytest.raises(ValueError):
            _sigma_budget_mib(bad)


# ---- the panelled fused step on the CPU protocol model of tests/test_protocol_model.py ----
# Launch sequence of a W > 1 step with np panels (csrc/siglip_capi.cu `fused_impl`):
#   L0.0  [L0.p G0.p] p = np-1..1  [Lk.p Gk.p] p = 0..np-1 for k = 1..W-1  G0.0
# The own panels past 0 write a local partial into slot `rank` (no peer reads it), which the first fold reads as its
# second source. A remote chunk's slot is written by all its panels; flag 1 is raised by the last one. Flag 2 is the
# end signal of the last loss launch, L(W-1).(np-1).
import random  # noqa: E402

from test_protocol_model import Rank, build_actions, producer_of  # noqa: E402


def build_panel_actions(rk, bidir, np_, flag_after_first=False):
    acts = build_actions(rk, bidir)
    W, r, n = rk.W, rk.r, rk.step
    base = (n - 1) * W
    if W == 1:
        return acts

    def own_partial(p):
        def eff(ranks):
            if p == np_ - 1:
                rk.slots[r] = (n, "writing")
            if p == 1:
                rk.slots[r] = (n, "ok")
        return eff

    def first_fold_check(ranks):
        ver, state = rk.slots[r]
        assert (ver, state) == (n, "ok"), f"rank {r} bwd {n}: first fold read the own partial in state {ver, state}"

    def signal1(j):
        def eff(ranks):
            for q in ranks:
                q.flags[1][r] = max(q.flags[1][r], base + j)
        return eff

    out, deferred_end2 = [], None
    for name, guard, eff in acts:
        if name == "L(W-1).end":
            deferred_end2 = (name, guard, eff)
            continue
        if ".fold(" in name:
            pr = int(name[name.index("(") + 1:-1])
            assert pr != r, "a fold never reads the slot a rank keeps its own partial in"
            # with one panel there is no own partial: the first fold has no second source, as in the unbounded step
            first = np_ > 1 and (name.startswith("G2.") or (W == 2 and name.startswith("G0.")))
            if first:
                out.append((name + ".own", lambda ranks: True, lambda ranks: first_fold_check(ranks)))
            out.append((name, guard, eff))
            continue
        if name.startswith("G") and name.endswith(".end") and name != "G0.end":
            j = int(name[1:name.index(".")])
            c = rk.sched[j]
            for p in range(np_):
                last = p == np_ - 1
                if p > 0:
                    out.append((f"L{j}.{p}.mma", lambda ranks, o=c: True,
                                lambda ranks, o=c, j=j: _model_check(rk.gathered.get(o) == n,
                                                                     f"rank {r}: L{j} scores stale text of {o}")))
                    if last and j == W - 1:
                        out.append(deferred_end2)
                        deferred_end2 = None
                ok = (lambda ranks, c=c: rk.slots.__setitem__(c, (n, "ok"))) if last else (lambda ranks: None)
                signal = (last and not flag_after_first) or (p == 0 and flag_after_first)
                sig = signal1(j) if signal else (lambda ranks: None)
                out.append((f"G{j}.{p}.end", lambda ranks: True,
                            lambda ranks, ok=ok, sig=sig: (ok(ranks), sig(ranks))))
            continue
        out.append((name, guard, eff))
        if name.startswith("L0.pull("):
            for p in range(np_ - 1, 0, -1):
                out.append((f"L0.{p}", lambda ranks: True, lambda ranks: None))
                out.append((f"G0.{p}.partial", lambda ranks: True, own_partial(p)))
    if deferred_end2 is not None:   # np == 1: where the unbounded step raises it
        out.insert([a[0] for a in out].index(f"G{W - 1}.write.begin"), deferred_end2)
    return out


def _model_check(cond, msg):
    assert cond, msg


def simulate_panels(world, steps, bidir, seed, np_, lag_rank=None, flag_after_first=False):
    rng = random.Random(seed)
    ranks = [Rank(r, world, bidir) for r in range(world)]
    build = lambda rk: build_panel_actions(rk, bidir, np_, flag_after_first)  # noqa: E731
    for rk in ranks:
        rk.actions = build(rk)
    while any(rk.done_steps < steps for rk in ranks):
        enabled = [rk for rk in ranks if rk.done_steps < steps and rk.actions[rk.pc][1](ranks)]
        assert enabled, "deadlock: " + "; ".join(
            f"rank {rk.r} step {rk.step} at {rk.actions[rk.pc][0]}" for rk in ranks if rk.done_steps < steps)
        weights = [0.05 if (lag_rank is not None and rk.r == lag_rank) else 1.0 for rk in enabled]
        rk = rng.choices(enabled, weights)[0]
        rk.actions[rk.pc][2](ranks)
        rk.pc += 1
        if rk.pc == len(rk.actions):
            rk.done_steps += 1
            rk.step += 1
            rk.pc = 0
            rk.actions = build(rk)


def test_panel_schedule_is_what_the_model_runs():
    rk = Rank(0, 3, False)
    names = [a[0] for a in build_panel_actions(rk, False, 3)]
    assert names.index("L0.pull(1)") < names.index("L0.2") < names.index("G0.1.partial") < names.index("L1.pull(2)")
    assert names.index("G2.fold(2).own") < names.index("G2.fold(2)")
    assert names.index("L2.2.mma") < names.index("L(W-1).end") < names.index("G2.2.end") < names.index("G0.fold(1)")
    assert [n for n in names if n.startswith("G1.") and n.endswith(".end")] == ["G1.0.end", "G1.1.end", "G1.2.end"]


@pytest.mark.parametrize("np_", [1, 2, 3, 5])
@pytest.mark.parametrize("bidir", [False, True])
@pytest.mark.parametrize("world", [2, 3, 4])
def test_panelled_protocol_under_random_interleavings(world, bidir, np_):
    for seed in range(30):
        simulate_panels(world, steps=4, bidir=bidir, seed=seed, np_=np_)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_panelled_protocol_with_a_rank_that_is_always_late(world):
    for lag in range(world):
        for seed in range(8):
            simulate_panels(world, steps=3, bidir=(seed % 2 == 1), seed=100 * lag + seed, np_=3, lag_rank=lag)


def test_the_model_catches_flag1_after_the_first_panel():
    """Control: raising "contribution complete" after a chunk's FIRST panel lets the owner fold a slot that later
    panels are still writing; the model must see that stale read."""
    hits = 0
    for seed in range(60):
        try:
            simulate_panels(3, steps=3, bidir=(seed % 2 == 1), seed=seed, np_=3, lag_rank=seed % 3,
                            flag_after_first=True)
        except AssertionError as ex:
            assert "deadlock" not in str(ex)
            assert "folded slot" in str(ex) or "last fold read slot" in str(ex)
            hits += 1
    assert hits > 0
