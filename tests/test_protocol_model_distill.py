"""The CPU protocol model of tests/test_protocol_model.py with the job placement of a distillation step (csrc/siglip_capi.cu
`fused_impl`, `l0_work_in_l1`): L0 publishes the teacher text right before the student text (same flag-2 wait, covered
by the same flag-0 signal), every text pull is followed by the pull of the same chunk's teacher text, and the flag-3 wait
runs in L1 (after L0's pull, before L1's pull) instead of L0. At W = 2 L1 is also the last loss launch, so its flag-2
end signal now comes after the flag-3 wait. Under random interleavings (and with one rank always late) the model checks
that no rank deadlocks, that every student and teacher pull reads the owner's slot while it holds THIS step's data, and
every check of the base model (folds, the last fold before the dtxt epilogue)."""
import random

import pytest

from test_protocol_model import Rank, build_actions


def build_distill_actions(rk, bidir):
    acts = build_actions(rk, bidir)
    if rk.W == 1:
        return acts
    r, s = rk.r, rk.step
    if not hasattr(rk, "tslot"):
        rk.tslot = (0, "ok")      # my exported teacher-text slot
        rk.tgathered = {}
    out = []
    wait3 = None
    for name, guard, eff in acts:
        if name == "L0.wait3":
            wait3 = (name.replace("L0", "L1"), guard, eff)
            continue
        if name == "L0.copy.begin":
            # teacher publish job: the same wait on flag 2 as the text publish job behind it
            out.append(("L0.tcopy.begin", guard, lambda ranks: setattr(rk, "tslot", (s, "writing"))))
            out.append(("L0.tcopy.end", lambda ranks: True, lambda ranks: setattr(rk, "tslot", (s, "ok"))))
        if name.startswith("L1.") and wait3 is not None:
            out.append(wait3)
            wait3 = None
        out.append((name, guard, eff))
        if ".pull(" in name:
            o = int(name[name.index("(") + 1:-1])

            def tpull(ranks, o=o):
                ver, state = ranks[o].tslot
                assert state == "ok" and ver == s, f"rank {r} step {s}: pulled teacher text of rank {o} in {ver, state}"
                rk.tgathered[o] = s
            # the pull job right behind the chunk's text pull: its flag-0 wait has already been observed
            out.append((name.replace("pull", "tpull"), lambda ranks: True, tpull))
    assert wait3 is None, "L1 must exist when W > 1"
    # the loss kernels read the teacher text of the chunks they score: check it alongside the student text
    final = []
    for name, guard, eff in out:
        final.append((name, guard, eff))
        if name.endswith(".mma"):
            k = int(name[1:name.index(".")])
            o = rk.sched[k]
            final.append((f"L{k}.tmma", lambda ranks: True,
                          lambda ranks, o=o, k=k: _check(rk.tgathered.get(o) == s,
                                                         f"rank {r}: L{k} scores stale teacher text of {o}")))
    return final


def _check(cond, msg):
    assert cond, msg


def simulate(world, steps, bidir, seed, lag_rank=None, builder=build_distill_actions):
    rng = random.Random(seed)
    ranks = [Rank(r, world, bidir) for r in range(world)]
    for rk in ranks:
        rk.actions = builder(rk, bidir)
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
            rk.actions = builder(rk, bidir)


def test_the_distill_placement_is_what_the_model_runs():
    rk = Rank(0, 2, False)
    names = [a[0] for a in build_distill_actions(rk, False)]
    assert "L0.wait3" not in names
    assert names.index("L0.tcopy.end") < names.index("L0.copy.begin")
    assert names.index("L0.pull(1)") < names.index("L0.tpull(1)") < names.index("L1.wait3") < names.index("L(W-1).end")


@pytest.mark.parametrize("bidir", [False, True])
@pytest.mark.parametrize("world", [2, 3, 4])
def test_distill_step_protocol_under_random_interleavings(world, bidir):
    for seed in range(40):
        simulate(world, steps=4, bidir=bidir, seed=seed)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_distill_step_protocol_with_a_rank_that_is_always_late(world):
    for lag in range(world):
        for seed in range(8):
            simulate(world, steps=3, bidir=(seed % 2 == 1), seed=100 * lag + seed, lag_rank=lag)


def test_the_model_catches_an_unordered_teacher_pull():
    """Sanity of the model: a teacher pull that does not follow the text pull (no flag-0 wait observed) reads a slot
    that still holds the previous step's teacher text, or one being overwritten."""
    def broken(rk, bidir):
        acts = build_distill_actions(rk, bidir)
        pulls = [a for a in acts if ".tpull(" in a[0]]
        rest = [a for a in acts if ".tpull(" not in a[0]]
        return pulls + rest    # every teacher pull before anything else of the step
    hits = 0
    for seed in range(60):
        try:
            simulate(3, steps=3, bidir=False, seed=seed, lag_rank=seed % 3, builder=broken)
        except AssertionError as ex:
            assert "deadlock" not in str(ex)
            hits += 1
    assert hits > 0
