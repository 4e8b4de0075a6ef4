"""The step sequences' coverage, derived from tests/step_sequences.py and the sources rather than claimed: every option
siglip_ctx_set_option accepts changes both ways between two checked steps, every state item sees a transition in which
a leak would show, each such leak moves a checked output of the oracle by more than 20x the tolerance, every refusal
appears and is followed by a checked step, and no sequence is redundant."""
import dataclasses
import functools
import pathlib
import re

import numpy as np
import pytest

import loopback_exchange as lx
import option_matrix as om
import step_sequences as ss

CAPI = pathlib.Path(__file__).resolve().parents[1] / "distributed_sigmoid_loss_b200" / "csrc" / "siglip_capi.cu"


def set_option_cases():
    """The SIGLIP_OPT_* case labels of siglip_ctx_set_option."""
    src = CAPI.read_text()
    m = re.search(r"^int siglip_ctx_set_option\([^{]*\{(.*?)^\}", src, re.M | re.S)
    assert m, "siglip_ctx_set_option not found"
    return sorted(set(re.findall(r"case SIGLIP_OPT_(\w+):", m.group(1))))


def flips(seq):
    """(option, before, after) of every option change between two consecutive successful steps."""
    ok = [st for st in seq.steps if st.refuse is None]
    out = set()
    for a, b in zip(ok, ok[1:]):
        va, vb = seq.options(a), seq.options(b)
        out |= {(k, va[k], vb[k]) for k in va if va[k] != vb[k]}
    return out


def test_the_model_knows_every_option():
    cases = set(set_option_cases())
    assert cases == set(ss.DEFAULTS) | set(ss.EXEMPT), (
        f"options of siglip_ctx_set_option the model does not know: {sorted(cases - set(ss.DEFAULTS) - set(ss.EXEMPT))}"
        f"; options the model has that the library does not: {sorted(set(ss.DEFAULTS) | set(ss.EXEMPT) - cases)}")


@pytest.mark.parametrize("option", [o for o in set_option_cases() if o not in ss.EXEMPT])
def test_every_option_changes_both_ways_between_checked_steps(option):
    """A pair of values (x, y) with a change x -> y and one y -> x, each between two consecutive successful steps."""
    seen = set()
    for seq in ss.SEQUENCES:
        seen |= {(a, b) for k, a, b in flips(seq) if k == option}
    both = {(a, b) for a, b in seen if (b, a) in seen}
    assert both, f"SIGLIP_OPT_{option} never changes both ways between two checked steps (changes: {sorted(seen)})"


def test_state_table_names_its_code():
    for item in ss.STATE:
        assert re.search(r"\d{3,4}", item.reset), f"{item.name}: the reset rule cites no line"
        assert item.whole or item.part, item.name


@pytest.mark.parametrize("item", ss.ITEMS)
def test_every_state_item_has_a_leak_transition(item):
    n = sum(len(ss.transitions(seq)[item]) for seq in ss.SEQUENCES)
    assert n > 0, f"no sequence has a transition in which a leak of {item} would show"


def test_every_refusal_appears_and_is_followed_by_a_checked_step():
    seen = set()
    for seq in ss.SEQUENCES:
        for i, st in enumerate(seq.steps):
            if st.refuse is None:
                continue
            seen.add(st.refuse)
            assert i + 1 < len(seq.steps) and seq.steps[i + 1].refuse is None, \
                f"{seq.name} step {i}: the refusal is not followed by a checked step"
    assert seen == set(ss.REFUSALS), f"refusals no sequence provokes: {sorted(set(ss.REFUSALS) - seen)}"


def test_refusals_are_refused_by_the_model():
    """The budget refusals are what sigma_panels says: a budget below one panel of the step's cluster, a saving forward
    whose W whole operands exceed the budget; a backward without a saved forward follows a step that saves none."""
    for seq in ss.SEQUENCES:
        for i, st in enumerate(seq.steps):
            Bs, Rs, Ts = seq.cell(st).shapes()
            tp = om._round_up(max(Ts), 256)
            if st.refuse == "budget_below_panel":
                nbuf = 2 if seq.W > 1 else 1
                assert nbuf * 128 * st.cluster * tp * 2 > ss.Seq.budget_of(seq, st) * 2 ** 20, (seq.name, i)
                assert st.sched in ("fused", "scaled")
            if st.refuse == "split_over_budget":
                rp = om._round_up(max(Rs), 256)
                assert st.sched == "split" and seq.W * rp * tp * 2 > seq.budget_of(st) * 2 ** 20, (seq.name, i)
            if st.refuse == "backward_unsaved":
                prev = [s for s in seq.steps[:i] if s.refuse is None][-1]
                assert prev.sched in ("fused", "scaled", "fwd") or seq.W > 1, (seq.name, i)


def test_shapes_and_options_are_valid_for_the_context():
    for seq in ss.SEQUENCES:
        assert 6 <= len(seq.steps) <= 10, seq.name
        for i, st in enumerate(seq.steps):
            o = st.opts
            assert (o.xtexts, o.ximages) == (seq.xtexts, seq.ximages), (seq.name, i)
            assert o.labels in (0, seq.M), (seq.name, i)
            assert not o.teacher or seq.teacher, (seq.name, i)
            if seq.teacher == "distill":   # siglip_ctx_create_distill: no extras, sets, groups under the teacher
                assert not (seq.xtexts or seq.ximages or seq.M)
                assert st.refuse or not (o.teacher and (o.groups or o.losses or o.topk > 1)), (seq.name, i)
            if st.sched == "eval":
                assert seq.W == 1, "a multi-rank forward without save drops the saved state"
            if st.knob("SYNC_SCALAR_GRADS"):
                assert seq.W > 1


def _coverage(seq):
    keys = {("flip",) + f for f in flips(seq)}
    for item, tr in ss.transitions(seq).items():
        kind = (seq.W, seq.xtexts, seq.ximages, seq.M, seq.teacher)   # the context kind
        keys |= {("item", item, kind, seq.steps[b].sched) for a, b in tr}
    keys |= {("refusal", st.refuse) for st in seq.steps if st.refuse}
    return keys


def test_no_sequence_is_redundant():
    cov = [_coverage(s) for s in ss.SEQUENCES]
    for i, seq in enumerate(ss.SEQUENCES):
        others = set().union(*(c for j, c in enumerate(cov) if j != i))
        assert cov[i] - others, f"{seq.name} covers nothing the other sequences do not"


# ---------------------------------------------------------------------------------------------------------------------
# leak sensitivity on the oracle
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _problem(seq_name, i):
    seq = next(s for s in ss.SEQUENCES if s.name == seq_name)
    return om.planted(seq.cell(seq.steps[i]))


@functools.lru_cache(maxsize=None)
def _ref(seq_name, i):
    seq = next(s for s in ss.SEQUENCES if s.name == seq_name)
    st = seq.steps[i]
    res = om.oracle(_problem(seq_name, i), st.opts, st.tp, st.bias, st.lam)[seq.r]
    g = st.grad_out
    return dict(res, dimg=g * res["dimg"], contrib=[g * c for c in res["contrib"]], dt_prime=g * res["dt_prime"],
                dbias=g * res["dbias"])


def _min_block_change(a, b):
    """The smallest relative change of b (the suite's measure) when one 128-row block of it holds a's rows."""
    out = np.inf
    for i0 in range(0, b.shape[0], 128):
        x = b.copy()
        x[i0:i0 + 128] = a[i0:i0 + 128]
        out = min(out, om.rel(x, b))
    return out


def _inputs_read(seq, st):
    """The pulled kinds (loopback_exchange.kinds) a step reads of chunk (r + 1) % W: at W = 1 the own inputs, which are
    context state too (ids_in, lrows, w_in), but not the text or teacher text, which come from the caller's tensors."""
    o, c = st.opts, (seq.r + 1) % seq.W
    Bs, Rs, Ts = seq.cell(st).shapes()
    out = []
    if seq.W > 1:
        out.append("text.f16" if st.f16 else "text.bf16")
    out += [k for k, on in (("ids", o.ids), ("xt_ids", o.xt_ids and Ts[c] > Bs[c]), ("weights", o.weights),
                            ("groups", o.groups)) if on]
    if o.labels:
        out.append(f"sets.M{o.labels}")
    if o.teacher and seq.W > 1:
        out.append("teacher.extras" if seq.teacher == "extras" else "teacher.distill")
    return out


def _exact_leak(visible):
    """An output compared exactly: any visible change fails the step."""
    return np.inf if visible else 0.0


def _leak(seq, item, a, b):
    """The relative change of a checked output under the smallest leak of `item` from step a into step b, per leak."""
    A, B = seq.steps[a], seq.steps[b]
    ra, rb = _ref(seq.name, a), _ref(seq.name, b)
    PA, PB = _problem(seq.name, a), _problem(seq.name, b)
    if item == "partials":
        # one CTA's partial slot: one 128 x 128 tile of the earlier step, taken as the smallest 128-row block's share
        # of the earlier loss over one 128-column tile of the global batch's texts (the block's row sums times
        # 128 / sum T)
        Bs, Rs, Ts, _, _ = PA.view(A.opts)
        block = min(ra["image_loss"][i0:i0 + 128].sum() for i0 in range(0, len(ra["image_loss"]), 128))
        share = block * min(1.0, 128 / sum(Ts)) / Bs[seq.r]
        return {"loss": abs(share) / abs(rb["loss"])}
    if item == "saved_scalars":
        return {"dt_prime": om.rel(ra["dt_prime"] / A.grad_out * B.grad_out, rb["dt_prime"]),
                "dbias": om.rel(ra["dbias"] / A.grad_out * B.grad_out, rb["dbias"])}
    if item in ("sigma", "diag_and_16bit", "accumulators", "split_k"):
        return {"dimg": _min_block_change(ra["dimg"], rb["dimg"]),
                "dtxt": _min_block_change(ra["contrib"][seq.r], rb["contrib"][seq.r])}
    if item == "teacher_focal":   # the previous step's lambda or (gamma, alpha) with this step's data
        o = B.opts
        if o.focal is not None and A.opts.focal is not None and A.opts.focal != o.focal:
            o = dataclasses.replace(o, focal=A.opts.focal)
        res = om.oracle(PB, o, B.tp, B.bias, A.lam if B.opts.teacher else B.lam)[seq.r]
        return {"loss or dimg": max(om.rel(res["loss"], rb["loss"]), om.rel(B.grad_out * res["dimg"], rb["dimg"]))}
    if item == "step_inputs":   # one stale pulled chunk of every kind the later step reads
        out = {}
        for kind in _inputs_read(seq, B):
            res = om.oracle(lx.stale(PB, PA, kind, (seq.r + 1) % seq.W), B.opts, B.tp, B.bias, B.lam)[seq.r]
            vals = [om.rel(res["loss"], rb["loss"])]
            if B.backward:
                vals += [om.rel(B.grad_out * res["dimg"], rb["dimg"])]
            out[kind] = max(vals)
        return out
    if item == "parity_blocks":   # one stale word of each block both steps armed, left by a skipped memset
        out = {}
        oa, ob = A.opts, B.opts
        r = seq.r
        if (oa.keys or oa.topk > 1) and (ob.keys or ob.topk > 1):
            ya, yb = om.retrieval(PA, oa, max(oa.topk, 1))[r], om.retrieval(PB, ob, max(ob.topk, 1))[r]
            rows = slice(yb["off"][r], yb["off"][r + 1])
            Sa, Sb = ya["S"][rows], yb["S"][rows]
            # a stale row key (or list entry) of A wins where A's best logit beats B's (K-th best, for a list) and
            # points elsewhere
            k = max(ob.topk, 1)
            kth = -np.sort(-Sb, axis=1)[:, k - 1] if Sb.shape[1] >= k else np.full(Sb.shape[0], -np.inf)
            wins = (Sa.max(axis=1) > kth) & (Sa.argmax(axis=1) != Sb.argmax(axis=1))
            out["key" if ob.keys else "list entry"] = _exact_leak(wins.any())
        if oa.losses and ob.losses:
            # a stale fixed-point word: one 128-column tile of an image's sum in A, on top of its sum in B
            Ts = PB.view(ob)[2]
            word = ra["image_loss"] * min(1.0, 128 / sum(Ts))
            words = sum((t + 127) // 128 + 1 for t in Ts)
            out["word"] = float(np.max(word / (om.TOL * rb["image_loss"] + words * 2.0 ** -32))) * om.TOL
        return out
    raise AssertionError(item)


def _claims():
    """Every claimed transition whose leak the oracle can show. The counters' leak (a refused call advancing n_fwd /
    n_bwd) is a wrong flag value or request parity, not a value: the step behind each refusal shows it on the device."""
    out = []
    for seq in ss.SEQUENCES:
        for item, tr in ss.transitions(seq).items():
            if item == "counters":
                continue
            for a, b in tr:
                A, B = seq.steps[a], seq.steps[b]
                if item == "step_inputs" and not _inputs_read(seq, B):
                    continue
                if item in ("sigma", "diag_and_16bit", "accumulators", "split_k") and not B.backward:
                    continue
                if item == "parity_blocks" and not (((A.opts.keys or A.opts.topk > 1) and
                                                     (B.opts.keys or B.opts.topk > 1)) or
                                                    (A.opts.losses and B.opts.losses)):
                    continue
                out.append((seq, item, a, b))
    return out


@pytest.mark.parametrize("seq,item,a,b", _claims(), ids=lambda x: getattr(x, "name", str(x)))
def test_a_leak_moves_a_checked_output(seq, item, a, b):
    changes = _leak(seq, item, a, b)
    assert changes, f"{seq.name} {item} {a} -> {b}: no leak measured"
    for kind, change in changes.items():
        assert change > ss.SENSITIVITY * om.TOL, \
            f"{seq.name} {item} {a} -> {b}: a stale {kind} moves the output by {change:.2e}"
