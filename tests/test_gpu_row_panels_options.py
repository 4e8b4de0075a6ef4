"""Row panels (SIGLIP_OPT_SIGMA_BUDGET_MIB) composed with the other options, on the H100: single rank and loopback
W = 2 / 3 (uneven batches, bidir). Every case runs the same context configuration twice, unbounded and under a budget
that forces 2 to 5 panels (ragged last ones, panels made only of extra-image rows), and checks the panelled step against
the float64 oracle of the option group to the suite's 1e-3, and against the unbounded step: dimg bit-identical at W = 1,
everything else within fp32 summation order. Groups: positional labels, sample ids, hard negatives, extra texts with
ids, extra images with and without ids, extra images with hard negatives (the iota-id own chunk), weights,
distillation, bidir, uneven batches, split-K, both gradient tile widths, cta_group / multicast shapes, bf16 gradients,
fp32 inputs through the module, sync_scalar_grads, and the host-buffer entries."""
import math

import numpy as np
import pytest
import torch

import test_gpu_distill as dist
from test_gpu_extra_images import _check_rank, _data, _engine, _ids, _oracle, _prepare, _step

pytestmark = pytest.mark.gpu

MIB = 1 << 20


def _dev():
    return torch.device("cuda", 0)


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-300))


def _budget(eng):
    """The smallest whole-MiB budget that splits this rank's rows into at least two panels."""
    for mib in range(1, 64):
        eng.set_sigma_budget(mib * MIB)
        rows, n, _ = eng.sigma_panels()
        if rows and n >= 2:
            return n
    raise AssertionError("no budget gives panels")


def _weights(seed, Rs, Ts):
    g = torch.Generator().manual_seed(seed)
    wi = [torch.rand(r, generator=g) for r in Rs]
    wt = [torch.rand(t, generator=g) for t in Ts]
    wi[0][::5] = 0.0
    return wi, wt


CASES = {
    # name: (Bs, E (extra images per rank), K (extra texts per rank), ids, xtxt_ids, ximg_ids, weights, bidir)
    "w1_positional": ([1000], 0, 0, False, False, False, False, False),
    "w1_ids": ([1000], 0, 0, True, False, False, False, False),
    "w1_hard_negatives": ([900], 0, 300, False, False, False, False, False),
    "w1_extra_texts_ids": ([900], 0, 300, True, True, False, False, False),
    "w1_extra_images": ([600], 500, 0, False, False, False, False, False),
    "w1_extra_images_ids": ([600], 500, 0, True, False, True, False, False),
    "w1_extra_images_hard_negatives": ([600], 500, 200, False, False, False, False, False),
    "w1_weights": ([1000], 0, 0, False, False, False, True, False),
    "w2_uneven": ([1000, 700], 0, 0, False, False, False, False, False),
    "w2_extra_texts_ids_weights": ([800, 600], 0, 200, True, True, False, True, False),
    "w3_uneven_bidir_ids_weights": ([900, 700, 1000], 0, 0, True, False, False, True, True),
    "w3_extra_images_hard_negatives_ids": ([600, 500, 700], 400, 150, True, False, True, False, False),
}


@pytest.mark.parametrize("name", list(CASES))
def test_option_groups_against_oracle_and_unbounded(name):
    Bs, E, K, ids_on, xtxt, ximg, w_on, bidir = CASES[name]
    from distributed_sigmoid_loss_b200 import _capi
    W, D = len(Bs), 136
    Rs, Ts = [b + E for b in Bs], [b + K for b in Bs]
    imgs, txts = _data(Bs, Rs, Ts, D, seed=len(name))
    ids = xt = xi = None
    if ids_on:
        ids, xt, xi = _ids(Bs, Rs, Ts, seed=3)
    wi = wt = None
    if w_on:
        wi, wt = _weights(5, Rs, Ts)
    ref = _oracle(imgs, txts, Bs, ids if ids_on else None, xt if xtxt else None, xi if ximg else None, wi, wt)
    for r in range(W):
        outs = []
        for bounded in (False, True):
            eng = _engine(r, Bs, Rs, Ts, D, ids=ids_on, ximg_ids=ximg, xtxt_ids=xtxt, weights=w_on)
            if bidir:
                eng.set_option(_capi.SIGLIP_OPT_BIDIR, 1)
            if bounded:
                assert _budget(eng) >= 2
            _prepare(eng, r, txts, ids, xt, xi, wi, wt)
            outs.append(_step(eng, "fused", imgs[r].to(_dev()), txts[r].to(_dev())))
            torch.cuda.synchronize()
            eng.close()
        unb, pan = outs
        _check_rank(f"{name} rank {r} panelled", eng, r, pan, ref)
        if W == 1:
            assert torch.equal(pan[1], unb[1]), "dimg must be bit-identical at W = 1"
        for a, b in zip(pan, unb):
            assert _rel(a, b) <= 1e-5


@pytest.mark.parametrize("W,Bs,ids,weights", [(1, [1000], True, True), (3, [900, 700, 1000], True, True)])
def test_distillation_against_oracle_and_unbounded(W, Bs, ids, weights):
    D, DT = 136, 72
    P = dist._problem(Bs, D, DT, seed=41 + W, ids=ids, weights=weights)
    ref = dist._oracle(P, 0.7)
    for r in range(W):
        outs = []
        for bounded in (False, True):
            eng = dist._engine(Bs[r], D, DT, W=W, r=r, Bs=Bs if W > 1 else None, ids=ids, weights=weights)
            if bounded:
                assert _budget(eng) >= 2
            outs.append(dist._step(eng, P, r, 0.7, "fused"))
            eng.close()
        unb, pan = outs
        dist._check_step(f"distill W={W} rank {r}", pan, ref[r], r, W)
        if W == 1:
            assert torch.equal(pan[1], unb[1])
        for a, b in zip(pan, unb):
            assert _rel(a, b) <= 1e-5


@pytest.mark.parametrize("opt", ["split_k", "tile128", "tile256", "cg1", "mcast2", "bf16_grads"])
@pytest.mark.parametrize("Bs", [[1000], [1000, 700]])
def test_kernel_options_against_unbounded(opt, Bs):
    from distributed_sigmoid_loss_b200 import _capi
    W, D = len(Bs), 264
    imgs, txts = _data(Bs, Bs, Bs, D, seed=17)
    ref = _oracle(imgs, txts, Bs)
    gdt = torch.bfloat16 if opt == "bf16_grads" else torch.float32
    for r in range(W):
        outs = []
        for bounded in (False, True):
            eng = _engine(r, Bs, Bs, Bs, D, cg=1 if opt == "cg1" else 2, mcast=2 if opt == "mcast2" else 1)
            if opt == "split_k":
                eng.set_option(_capi.SIGLIP_OPT_SPLIT_K, -1)
            if opt.startswith("tile"):
                eng.set_option(_capi.SIGLIP_OPT_GRAD_TILE_N, int(opt[4:]))
            if bounded:
                assert _budget(eng) >= 2
            _prepare(eng, r, txts, None, None, None, None, None)
            outs.append(_step(eng, "fused", imgs[r].to(_dev()), txts[r].to(_dev()), gdt))
            torch.cuda.synchronize()
            eng.close()
        unb, pan = outs
        # bf16 gradients: 2^-9 rounding of the results (the module tolerance of the suite)
        _check_rank(f"{opt} rank {r} panelled", eng, r, pan, ref, 4e-3 if gdt == torch.bfloat16 else 1e-3)
        if W == 1 and opt != "split_k":
            assert torch.equal(pan[1], unb[1]), "dimg must be bit-identical at W = 1 without split-K"
        for a, b in zip(pan, unb):
            assert _rel(a, b) <= (4e-3 if gdt == torch.bfloat16 else 1e-5)


def test_sync_scalar_grads_loopback():
    from distributed_sigmoid_loss_b200 import _capi
    Bs, D = [1000, 700], 136
    imgs, txts = _data(Bs, Bs, Bs, D, seed=23)
    outs = []
    for bounded in (False, True):
        eng = _engine(0, Bs, Bs, Bs, D)
        eng.set_option(_capi.SIGLIP_OPT_SYNC_SCALAR_GRADS, 1)
        eng.debug_set_mailbox(1, 0.25, -0.5)
        if bounded:
            assert _budget(eng) >= 2
        _prepare(eng, 0, txts, None, None, None, None, None)
        outs.append(_step(eng, "fused", imgs[0].to(_dev()), txts[0].to(_dev())))
        torch.cuda.synchronize()
        eng.close()
    for a, b in zip(*outs):
        assert _rel(a, b) <= 1e-5


def test_fp32_inputs_through_the_module():
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss
    B, D = 1000, 136
    g = torch.Generator().manual_seed(29)
    x = torch.randn(B, D, generator=g).to(_dev())
    y = (x + 0.8 * torch.randn(B, D, generator=g).to(_dev()))
    res = []
    for kind in ("ddp", "siglip"):
        for budget in (None, MIB):
            if kind == "ddp":
                mod = DDPSigmoidLoss(B, normalize_inputs=True, sigma_budget_bytes=budget).to(_dev())
                xi, yi = x.clone().requires_grad_(), y.clone().requires_grad_()
                loss = mod(xi, yi)
            else:
                mod = SigLipLoss(sigma_budget_bytes=budget).to(_dev())
                xi = torch.nn.functional.normalize(x).requires_grad_()
                yi = torch.nn.functional.normalize(y).requires_grad_()
                loss = mod(xi, yi, torch.tensor(math.log(10.0), device=_dev()), torch.tensor(-10.0, device=_dev()))
            loss.backward()
            if budget:
                eng = next(iter(mod._cache._engines.values()))
                rows, n, _ = eng.sigma_panels()
                assert n >= 2, (rows, n)
            res.append((loss.detach(), xi.grad, yi.grad))
    for k in (0, 2):
        for a, b in zip(res[k + 1], res[k]):
            assert _rel(a.float(), b.float()) <= 1e-5
        assert torch.equal(res[k + 1][1], res[k][1])


def test_host_entries_run_under_the_budget():
    from distributed_sigmoid_loss_b200.loss import SigmoidLossEngine
    B, D = 1000, 136
    imgs, txts = _data([B], [B], [B], D, seed=31)
    outs = []
    for bounded in (False, True):
        eng = SigmoidLossEngine(B, D, _dev())
        if bounded:
            assert _budget(eng) >= 2
        dimg, dtxt = torch.empty(B, D), torch.empty(B, D)
        scal = eng.fwd_bwd_host(imgs[0].contiguous(), txts[0].contiguous(), math.log(10.0), -10.0, dimg, dtxt)
        outs.append((torch.tensor(scal), dimg, dtxt))
        eng.close()
    unb, pan = outs
    assert torch.equal(pan[1], unb[1]), "dimg must be bit-identical at W = 1"
    for a, b in zip(pan, unb):
        assert _rel(a, b) <= 1e-5
