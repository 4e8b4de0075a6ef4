"""The loopback exchange cells (tests/loopback_exchange.py) on the H100: what the pulls move in and what the folds add.

Each cell runs two steps of one rank of a W-rank job. Before each, every peer's chunk (text, ids, groups, label sets,
weights, teacher text) is seeded afresh into the stand-in of the peers' exported allocation, from where only the step's
pulls can bring it to the kernels, and every peer's contribution to this rank's text gradient is seeded afresh (dyadic
values on a coarse grid at the magnitude of the own contribution: their fp32 sum is exact in any order). A pull that
did not run, ran short or read the wrong slot leaves the first step's data in the second; a fold of the wrong peer, a
dropped or shifted one, or one scaled by grad_out again moves dtxt.

Every step runs with grad_out g = 0.75 (siglip_fwd_bwd_scaled, or siglip_backward with grad_out), and the peers'
contributions are already scaled, so dtxt = g own + sum C: the epilogue adds its add_src after the scale. Checked per
step: loss, dimg, dt', dbias and the outgoing slots against the oracle (g times its gradients) within 1e-3, bf16 outputs
within 1e-3 + 2^-8; dtxt - sum C against g own within the same plus the rounding of the output (2^-23, or 2^-8 for a
bf16 output, of |own| + |sum C|). The same step with zero seeds gives every output but dtxt bit for bit (the seeds enter
dtxt only), and a dtxt within the roundings the two results and the fold chain can differ by: the seeded sum goes
through fp32 adds with the own contribution (the first fold's own_part under row panels, G0's epilogue or the final
add), each rounding to the nearest of its result, so the two differ by at most an ulp of each result (bf16 or fp32) and
of the fold chain's partial sums, not bit for bit.

Observed on one H100 80GB HBM3 (700 W power limit): the 36 cells in about 25 s; the largest relative errors: loss
3.8e-7, dimg 3.7e-3 (a bf16 output), dt' 4.9e-7, dbias 5.4e-7, outgoing slots 2.7e-4, dtxt - sum C 1.6e-4 for fp32
outputs and 7.9e-3 for bf16 ones (whose rounding is that of |own| + |sum C|), and the zero-seed comparison at 0.5 of
its bound. Host-only mutations that keep every address in its allocation fail it: G0 folding peer pr + 1's block fails
every fused cell, and the un-overlapped pull skipping the weights copy fails the cell that runs it."""
import numpy as np
import pytest
import torch

import loopback_exchange as lx
import option_matrix as om
from test_gpu_option_matrix import _engine, _inputs, _operand, _references, _scal, _seed_peers

pytestmark = pytest.mark.gpu

BF16_TOL = om.TOL + 2.0 ** -8
OBSERVED = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(OBSERVED):
        print(f"loopback exchange: largest relative error of {k}: {OBSERVED[k]:.3e}")


def _note(kind, err):
    OBSERVED[kind] = max(OBSERVED.get(kind, 0.0), err)


def _check(tag, kind, got, ref, tol):
    got = got.double().cpu().numpy() if torch.is_tensor(got) else np.asarray(got, np.float64)
    err = om.rel(got, ref)
    _note(kind, err)
    assert err <= tol, f"{tag} {kind}: relative error {err:.3e} (tolerance {tol:.2e})"


def _configure(eng, x):
    from distributed_sigmoid_loss_b200 import _capi

    for opt, v in ((_capi.SIGLIP_OPT_OVERLAP_PULL, x.pull), (_capi.SIGLIP_OPT_OVERLAP_REDUCE, x.reduce),
                   (_capi.SIGLIP_OPT_INKERNEL_SYNC, x.sync)):
        eng.set_option(opt, int(v))


def _step(eng, x, cell, P):
    """One step with grad_out: loss, dimg, dtxt, dt', dbias and the outgoing slots (slot<k>)."""
    o, r = cell.opts, cell.r
    Bs, Rs, Ts, imgs, txts = P.view(o)
    teacher = _inputs(eng, cell, P)  # noqa: F841  (kept alive until the step is enqueued)
    img, txt = _operand(imgs[r], cell.f16), _operand(txts[r], cell.f16)
    tp, b, g = _scal(om.TP), _scal(om.BIAS), _scal(lx.GRAD_OUT)
    gdt = torch.bfloat16 if x.bf16 else torch.float32
    out = {}
    if cell.sched == "fused":
        out["loss"], out["dimg"], out["dtxt"], out["dtp"], out["db"] = eng.fwd_bwd(img, txt, tp, b, gdt, g)
    else:
        out["loss"] = eng.forward(img, txt, tp, b, True)
        out["dimg"], out["dtxt"], out["dtp"], out["db"] = eng.backward(img, txt, tp, g, gdt)
    for k in range(cell.W):
        if k != r:
            out[f"slot{k}"] = eng.debug_get_slot(k)
    torch.cuda.synchronize()
    return {k: v.clone() for k, v in out.items()}


def _seed_contributions(eng, x, C):
    for p, blk in C.items():
        eng.debug_set_peer_contribution(p, torch.from_numpy(np.ascontiguousarray(blk, np.float32)).cuda())


@pytest.mark.parametrize("x", lx.CELLS, ids=lambda x: x.name)
def test_exchange_cell(x):
    c = x.base
    tol = BF16_TOL if x.bf16 else om.TOL
    u = 2.0 ** -8 if x.bf16 else 2.0 ** -23   # an output's rounding, relative to its magnitude, with margin
    eng = _engine(c)
    try:
        _configure(eng, x)
        for step in (0, 1):
            cs, P = x.step_seed(step), lx.problem(x, step)
            tag = f"{x.name} step {step}"
            _, _, stand = _references(cs, P)
            ref = lx.references(x, P)
            own = ref["contrib"][c.r]
            C = lx.seeds(x, own, step)
            total = sum(C.values())
            _seed_peers(eng, cs, P, stand)
            _seed_contributions(eng, x, C)
            out = _step(eng, x, cs, P)
            _check(tag, "loss", out["loss"], ref["loss"], om.TOL)
            _check(tag, "dimg", out["dimg"], ref["dimg"], tol)
            _check(tag, "dt_prime", out["dtp"], ref["dt_prime"], om.TOL)
            _check(tag, "dbias", out["db"], ref["dbias"], om.TOL)
            for k in range(c.W):
                if k != c.r:
                    _check(tag, "outgoing slots", out[f"slot{k}"], ref["contrib"][k], om.TOL)
            mag = np.abs(own) + np.abs(total)
            ratio = max(np.linalg.norm(mag) / np.linalg.norm(own), mag.max() / np.abs(own).max())
            got = out["dtxt"].double().cpu().numpy()
            _check(tag, "dtxt - sum C" + (" (bf16)" if x.bf16 else ""), got - total, own, tol + u * ratio)
            # the same step with zero seeds
            _seed_contributions(eng, x, {p: np.zeros_like(blk) for p, blk in C.items()})
            zero = _step(eng, x, cs, P)
            for k, v in zero.items():
                if k != "dtxt":
                    assert torch.equal(v, out[k]), f"{tag}: {k} differs when the peers' contributions are zero"
            z = zero["dtxt"].double().cpu().numpy()
            diff = np.abs(got - total - z)
            bound = u * (np.abs(got) + np.abs(z) + np.abs(total)) + 2.0 ** -22 * np.abs(own).max()
            _note("dtxt - sum C against the zero-seed step, in bounds", float((diff / bound).max()))
            worst = np.unravel_index(int((diff - bound).argmax()), diff.shape)
            assert (diff <= bound).all(), (f"{tag}: dtxt - sum C differs from the zero-seed step at {worst}: "
                                           f"{got[worst]} - {total[worst]} vs {z[worst]}")
    finally:
        eng.close()
