"""The gradient kernel's cells (tests/grad_matrix.py) against the float64 oracle, on the device.

The coverage the CPU suite derives assumes an H100 SXM's co-resident cluster counts. The first test reads the
device's own counts through siglip_debug_max_active_clusters and derives the coverage again from them: if a count
differs and a branch, an instantiation or a split is no longer reached, it fails and names what is missing.

Every cell then runs one rank's step (loopback stand-ins for the peers at W > 1) at trained-regime logits, where the
negatives carry the gradient, and compares with the oracle: dimg, every dtxt contribution (the own chunk's from the
step's dtxt, the others from their slots), the parts of dimg and of the own contribution that pass through the
16-bit sigma operand G (the output minus the oracle's fp32 own-diagonal term), dt' / dbias relative to sum |G| and
t sum |G s|, and the loss. Tensors take the suite's relative Frobenius and max-abs / max measure, and also a per-row
one: each row's error over that row's oracle norm, floored at 1e-3 x the median row norm, so that one wrong row at a
tile edge cannot hide in a whole-tensor norm. A cell with SIGLIP_OPT_SPLIT_K that splits must give bits different from
the same step at SPLIT_K = 0 (proof that it split) and the same bits twice; one that cannot split must give the bits of
SPLIT_K = 0.

Observed on one H100 80GB HBM3 (700 W power limit; co-resident clusters 132, 66 and 30 at cluster sizes 1, 2 and 4),
largest over the cells of each group; `pytest -s` prints them. The file runs in under a minute there.
  group                                     tensors   rows      loss      scalars   tolerance
  M (1 .. 1000 rows, every cluster size)    1.2e-4    3.2e-4    8.2e-6    8.5e-6    TOL 1e-3
  D (8 .. 392 columns, both tile widths)    4.0e-5    4.3e-4    1.7e-6    1.3e-6    TOL
  K (40, 64, 65: below, at, past a k block) 1.1e-4    4.3e-4    7.7e-7    5.3e-7    TOL
  split-K (S = 2, 3, 4; cluster 1 and 2)    3.6e-5    3.5e-4    1.2e-6    9.3e-7    TOL
  branches (W 1..3, extras, panels, f16)    3.2e-3    3.5e-2    7.7e-7    5.6e-7    TOL; BF16_TOL for bf16 outputs
The branch cells' largest errors are bf16 outputs: their rows are the part through G of a bf16 row, measured against
the part's norm, and may carry that row's rounding on top of the tolerance.
"""
import numpy as np
import pytest
import torch

import grad_matrix as gm
from test_grad_matrix_cpu import _derive

pytestmark = pytest.mark.gpu

TOL = 1e-3
BF16_TOL = TOL + 2.0 ** -8     # bf16 outputs: plus half an ulp of the largest binade in the max-abs / max measure
GRAD_OUT = 0.75
_OBSERVED = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(_OBSERVED):
        print(f"grad-matrix max error {k}: {_OBSERVED[k]:.3e}")


def _dev():
    return torch.device("cuda", 0)


def _scal(x):
    return torch.tensor([x], device=_dev(), dtype=torch.float32)


def _group(cell):
    if cell.name.startswith("splitk"):
        return "split-K"
    return cell.name.split("-")[0] if cell.name[0] in "MDK" else "branches"


def _note(key, err):
    _OBSERVED[key] = max(_OBSERVED.get(key, 0.0), err)


def _check(cell, what, got, ref, tol, full=None, bf16=False):
    """ref: the oracle tensor. full: for a part through G, the whole tensor it is a part of (a zero part is then held
    to tol x max |full|). bf16: the output was rounded to bf16, an error of up to 2^-9 of each element of the whole
    tensor, which each row of a part may carry on top of its tolerance."""
    got = got.double().cpu().numpy() if torch.is_tensor(got) else np.asarray(got, np.float64)
    ref = np.asarray(ref, np.float64)
    assert got.shape == ref.shape, (cell.name, what, got.shape, ref.shape)
    d = got - ref
    g = _group(cell)
    if full is not None and not ref.any():   # no pair passes through G (one sample, one chunk)
        err = float(np.abs(d).max() / (np.abs(full).max() + 1e-300))
        _note(f"{g} tensors", err)
        assert err <= tol, f"{cell.name} {what}: {err:.3e} of max |full| where the oracle is 0"
        return
    err = max(float(np.linalg.norm(d) / (np.linalg.norm(ref) + 1e-300)),
              float(np.abs(d).max() / (np.abs(ref).max() + 1e-300)))
    rn = np.linalg.norm(ref, axis=1)
    floor = 1e-3 * float(np.median(rn)) + 1e-300
    rows = np.linalg.norm(d, axis=1) / np.maximum(rn, floor)
    rounding = 2.0 ** -9 * np.linalg.norm(ref if full is None else full, axis=1) if bf16 else 0.0
    excess = np.linalg.norm(d, axis=1) / (tol * np.maximum(rn, floor) + rounding)
    worst = int(excess.argmax())
    _note(f"{g} tensors", err)
    _note(f"{g} rows", float(rows[worst]))
    assert err <= tol, f"{cell.name} {what}: relative error {err:.3e} (tolerance {tol:.1e})"
    assert excess[worst] <= 1.0, (f"{cell.name} {what}: row {worst} relative error {rows[worst]:.3e} "
                                  f"(tolerance {tol:.1e}{' + bf16 rounding' if bf16 else ''})")


def _check_scalar(cell, what, got, ref, scale):
    err = abs(float(got) - ref) / scale
    _note(f"{_group(cell)} scalars", err)
    assert err <= TOL, f"{cell.name} {what}: {float(got)} vs {ref}, error {err:.3e} of the scale {scale:.3e}"


def _operand(x, f16):
    t = torch.from_numpy(x)
    return ((t * gm.X_SCALE).half() if f16 else t.to(torch.bfloat16)).to(_dev())


def _engine(cell, imgs, texts, split_k=None):
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi

    c = cell.ctx
    kw = dict(batch_per_rank=list(c.Bs), texts_per_rank=list(c.Ts))
    if any(r > b for r, b in zip(c.Rs, c.Bs)):
        kw["images_per_rank"] = list(c.Rs)
    if c.W > 1:
        kw.update(rank_world=(c.r, c.W), loopback=True)
    eng = SigmoidLossEngine(c.Bs[c.r], c.D, _dev(), cta_group=c.cg, **kw)
    sk = c.split_k if split_k is None else split_k
    for opt, v in ((_capi.SIGLIP_OPT_MCAST, c.mcast), (_capi.SIGLIP_OPT_STAGES_GRAD, c.stages),
                   (_capi.SIGLIP_OPT_GRAD_TILE_N, 128 if split_k == 0 and c.split_k else c.tile_n),
                   (_capi.SIGLIP_OPT_SPLIT_K, sk), (_capi.SIGLIP_OPT_INPUT_F16, int(c.f16)),
                   (_capi.SIGLIP_OPT_SIGMA_BUDGET_MIB, c.budget_mib),
                   (_capi.SIGLIP_OPT_OVERLAP_REDUCE, int(c.overlap_reduce))):
        eng.set_option(opt, v)
    for k in range(c.W):
        if c.W > 1:
            eng.debug_set_text_chunk(k, _operand(texts[k], c.f16))
    return eng


def _step(cell, eng, imgs, texts, tp, bias):
    """dimg, every contribution (chunk order), dt', dbias, loss."""
    c = cell.ctx
    img, txt = _operand(imgs[c.r], c.f16), _operand(texts[c.r], c.f16)
    gdt = torch.bfloat16 if c.bf16 else torch.float32
    g = _scal(GRAD_OUT) if c.grad_out else None
    if c.sched == "fused":
        loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, _scal(tp), _scal(bias), gdt, g)
    else:
        loss = eng.forward(img, txt, _scal(tp), _scal(bias), True)
        dimg, dtxt, dtp, db = eng.backward(img, txt, _scal(tp), g, gdt)
    contrib = [dtxt.float() if k == c.r else eng.debug_get_slot(k) for k in range(c.W)]
    torch.cuda.synchronize()
    return [dimg.clone()] + [x.clone() for x in contrib] + [dtp.clone(), db.clone(), loss.clone()]


def _device_clusters():
    from distributed_sigmoid_loss_b200 import _capi

    return {cs: _capi.max_active_clusters(cg, mc, gm.TILE, 6) for cs, (cg, mc) in ((1, (1, 1)), (2, (2, 1)),
                                                                                      (4, (2, 2)))}


def test_coverage_holds_with_the_device_cluster_counts():
    from distributed_sigmoid_loss_b200 import _capi

    counts = _device_clusters()
    props = torch.cuda.get_device_properties(0)
    print(f"\n{props.name}, {props.multi_processor_count} SMs: co-resident clusters of the gradient kernel "
          f"(128 columns, 6 stages) {counts}")
    for cg, mc in ((1, 1), (2, 1), (2, 2)):
        n6 = _capi.max_active_clusters(cg, mc, gm.TILE, 6)
        assert _capi.max_active_clusters(cg, mc, gm.TILE, 4) == n6, "4- and 6-stage grids differ: the model has one"
        assert 1 <= n6 <= props.multi_processor_count // (cg * mc)
        print(f"  cta_group {cg} mcast {mc}: 256 columns {_capi.max_active_clusters(cg, mc, gm.WIDE_TILE, 0)}")
    with pytest.raises(_capi.SiglipError):
        _capi.max_active_clusters(3, 1, gm.TILE, 6)
    missing, _ = _derive_on(counts, props.multi_processor_count)
    assert not missing, f"with this device's cluster counts {counts}, not covered: " + "; ".join(missing)


def _derive_on(counts, num_sms):
    if num_sms != gm.NUM_SMS:
        pytest.fail(f"{num_sms} SMs: the matrix's tile-width and workspace rules are derived for {gm.NUM_SMS}")
    return _derive(counts)


@pytest.mark.parametrize("cell", gm.CELLS, ids=[c.name for c in gm.CELLS])
def test_grad_matrix_cell(cell):
    c = cell.ctx
    imgs, texts, tp, bias = gm.cell_inputs(cell)
    ref = gm.oracle(imgs, texts, c.Bs, c.r, tp, bias, GRAD_OUT if c.grad_out else 1.0)
    eng = _engine(cell, imgs, texts)
    out = _step(cell, eng, imgs, texts, tp, bias)
    tol = BF16_TOL if c.bf16 else TOL
    dimg, contrib, dtp, db, loss = out[0], out[1:1 + c.W], out[-3], out[-2], out[-1]
    _check(cell, "dimg", dimg, ref["dimg"], tol)
    _check(cell, "dimg through G", dimg.double().cpu().numpy() - ref["diag_dimg"], ref["rest_dimg"], tol,
           ref["dimg"], c.bf16)
    for k in range(c.W):
        # the own chunk's contribution is the step's dtxt (bf16 under GRAD_BF16); the others are fp32 slots
        t = tol if k == c.r else TOL
        _check(cell, f"contribution to chunk {k}", contrib[k], ref["contrib"][k], t)
        if k == c.r:
            own_diag = ref["contrib"][k] - ref["rest_contrib"]
            _check(cell, "own contribution through G", contrib[k].double().cpu().numpy() - own_diag,
                   ref["rest_contrib"], t, ref["contrib"][k], c.bf16)
    err = abs(float(loss) - ref["loss"]) / abs(ref["loss"])
    _note(f"{_group(cell)} loss", err)
    assert err <= TOL, f"{cell.name} loss: {float(loss)} vs {ref['loss']} (relative error {err:.3e})"
    _check_scalar(cell, "dbias", db, ref["dbias"], ref["sum_abs_g"])
    _check_scalar(cell, "dt_prime", dtp, ref["dt_prime"], ref["sum_abs_gs"])
    if c.split_k:
        counts = _device_clusters()
        splits = any(L.split.S for L in gm.launches(c, counts))
        again = _step(cell, eng, imgs, texts, tp, bias)
        assert all(torch.equal(a, b) for a, b in zip(out, again)), f"{cell.name}: split-K is not repeatable"
        eng.close()
        eng = _engine(cell, imgs, texts, split_k=0)
        base = _step(cell, eng, imgs, texts, tp, bias)
        same = all(torch.equal(a, b) for a, b in zip(out[:1 + c.W], base[:1 + c.W]))
        if splits:
            assert not same, f"{cell.name}: the split step gave the bits of SPLIT_K = 0: it did not split"
        else:
            assert same, f"{cell.name}: no split expected, but the bits differ from SPLIT_K = 0"
    eng.close()
