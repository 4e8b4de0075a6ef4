"""Row panels (SIGLIP_OPT_SIGMA_BUDGET_MIB) on the H100: the panelled fused step against the unbounded one on the same
context configuration. dimg, retrieval metrics and per-sample losses are bit-identical (the sigma values, the dimg
k-order and the fixed-point geometry do not depend on the panel); loss, dtxt, dt' and dbias agree up to fp32 summation
order. Also: forward-only within the budget, the split forward's refusal, CUDA-graph replay and the module."""
import math

import pytest
import torch

from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, _capi
from distributed_sigmoid_loss_b200.loss import SigmoidLossEngine

pytestmark = pytest.mark.gpu

MIB = 1 << 20
TP, BIAS = math.log(10.0), -10.0


def _dev():
    return torch.device("cuda", 0)


def _scal(x):
    return torch.tensor([x], device=_dev(), dtype=torch.float32)


def _data(B, D, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    img = torch.nn.functional.normalize(torch.randn(B, D, generator=g), dim=1)
    txt = torch.nn.functional.normalize(img + 0.7 * torch.randn(B, D, generator=g), dim=1)
    return img.to(_dev(), torch.bfloat16).contiguous(), txt.to(_dev(), torch.bfloat16).contiguous()


def _step(eng, img, txt, armed):
    bufs = None
    if armed:
        bufs = (torch.empty(2, device=_dev()), torch.empty(eng.metric_images, device=_dev(), dtype=torch.int64),
                torch.empty(eng.metric_texts, device=_dev(), dtype=torch.int64),
                torch.empty(eng.images, device=_dev()), torch.empty(eng.texts, device=_dev()))
        eng.request_metrics(*bufs[:3])
        eng.request_sample_losses(*bufs[3:])
    outs = [x.clone() for x in eng.fwd_bwd(img, txt, _scal(TP), _scal(BIAS))]
    torch.cuda.synchronize()
    return outs, bufs


def _close(a, b, tol=2e-5):
    err = (a.double() - b.double()).abs().max().item()
    scale = b.double().abs().max().item() + 1e-30
    assert err <= tol * scale, (err, scale)


@pytest.mark.parametrize("B,D,cg,budget_mib,panels", [
    (3000, 136, 2, 3, 6),    # 512-row panels, ragged last one of 440 rows
    (3000, 136, 2, 5, 4),
    (3000, 136, 1, 2, 12),   # 128-row unit: 256-row panels
    (1000, 64, 2, 1, 2),     # Tp = 1024: 1 MiB holds 512 rows -> 2 panels
])
def test_panelled_matches_unbounded_single_rank(B, D, cg, budget_mib, panels):
    img, txt = _data(B, D, seed=B + D)
    ref = SigmoidLossEngine(B, D, _dev(), cta_group=cg)
    eng = SigmoidLossEngine(B, D, _dev(), cta_group=cg)
    eng.set_sigma_budget(budget_mib * MIB)
    P = eng._L.siglip_sigma_panel_rows(B, (B + 255) // 256 * 256, (B + 255) // 256 * 256, 1, 128 * cg, budget_mib, None)
    assert 0 < P < B
    for armed in (False, True):
        (l0, di0, dt0, dtp0, db0), b0 = _step(ref, img, txt, armed)
        (l1, di1, dt1, dtp1, db1), b1 = _step(eng, img, txt, armed)
        assert torch.equal(di0, di1), "dimg must be bit-identical"
        _close(l1, l0)
        _close(dt1, dt0)
        _close(dtp1, dtp0, 1e-4)
        _close(db1, db0, 1e-4)
        if armed:
            for x, y in zip(b0, b1):
                assert torch.equal(x, y), "metrics and per-sample losses must be bit-identical"
    assert eng.workspace_bytes < ref.workspace_bytes


def test_forward_only_and_split_refusal():
    B, D = 3000, 136
    img, txt = _data(B, D, seed=7)
    ref = SigmoidLossEngine(B, D, _dev())
    want = ref.fwd(img, txt, _scal(TP), _scal(BIAS)).clone()
    eng = SigmoidLossEngine(B, D, _dev())
    full = 3072 * 3072 * 2
    eng.set_sigma_budget(3 * MIB)
    before = eng.workspace_bytes
    got = eng.fwd(img, txt, _scal(TP), _scal(BIAS))
    torch.cuda.synchronize()
    _close(got, want)
    assert eng.workspace_bytes - before <= 3 * MIB + 3072 * D * 2 < full
    with pytest.raises(_capi.SiglipError) as e:
        eng.forward(img, txt, _scal(TP), _scal(BIAS), True)
    assert e.value.code == _capi.SIGLIP_ERR_STATE and "siglip_fwd_bwd" in str(e.value)
    eng.set_sigma_budget(1 * MIB)   # below one 256-row panel of 3072 columns
    with pytest.raises(_capi.SiglipError) as e:
        eng.fwd_bwd(img, txt, _scal(TP), _scal(BIAS))
    assert e.value.code == _capi.SIGLIP_ERR_INVALID and "MiB" in str(e.value)


def test_graph_replay_matches_eager():
    B, D = 3000, 136
    img, txt = _data(B, D, seed=11)
    eng = SigmoidLossEngine(B, D, _dev())
    eng.set_sigma_budget(3 * MIB)
    tp, b = _scal(TP), _scal(BIAS)
    eager = [x.clone() for x in eng.fwd_bwd(img, txt, tp, b)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eng.fwd_bwd(img, txt, tp, b)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = eng.fwd_bwd(img, txt, tp, b)
    g.replay()
    torch.cuda.synchronize()
    for x, y in zip(outs, eager):
        assert torch.equal(x, y)


def test_module_budget_matches_engine():
    B, D = 3000, 136
    img, txt = _data(B, D, seed=13)
    mod = DDPSigmoidLoss(B, sigma_budget_bytes=3 * MIB).to(_dev())
    i, t = img.clone().requires_grad_(), txt.clone().requires_grad_()
    loss = mod(i, t)
    loss.backward()
    eng = mod.engine_for(B, D, _dev())
    assert eng.sigma_budget_mib == 3
    l, di, dt, _, _ = eng.fwd_bwd(img, txt, mod.t_prime.detach().float().reshape(1).contiguous(),
                                  mod.bias.detach().float().reshape(1).contiguous(), torch.bfloat16)
    torch.cuda.synchronize()
    _close(loss.detach().float().reshape(1), l)
    assert torch.equal(i.grad, di)
    _close(t.grad.float(), dt.float(), 1e-2)
    with pytest.raises(ValueError):
        DDPSigmoidLoss(B, sigma_budget_bytes=3 * MIB, fused_step=False).to(_dev())(img, txt)


def test_large_batch_single_rank():
    B, D, budget = 131072, 768, 4 << 30
    img, txt = _data(B, D, seed=17)
    eng = SigmoidLossEngine(B, D, _dev())
    eng.set_sigma_budget(budget)
    loss, dimg, dtxt, _, _ = eng.fwd_bwd(img, txt, _scal(TP), _scal(BIAS))
    torch.cuda.synchronize()
    assert eng.workspace_bytes < 32 << 30
    # fp32 torch reference in row blocks
    t, bb = math.exp(TP), BIAS
    x, y = img.float(), txt.float()
    tot = torch.zeros((), device=_dev(), dtype=torch.float64)
    gi = torch.empty_like(x)
    gt = torch.zeros_like(y)
    for r0 in range(0, B, 8192):
        z = t * (x[r0:r0 + 8192] @ y.T) + bb
        lab = -torch.ones_like(z)
        idx = torch.arange(z.shape[0], device=_dev())
        lab[idx, r0 + idx] = 1.0
        tot += torch.nn.functional.softplus(-lab * z).double().sum()
        g = -lab * torch.sigmoid(-lab * z) * t / B
        gi[r0:r0 + 8192] = g @ y
        gt += g.T @ x[r0:r0 + 8192]
    _close(loss.double(), (tot / B).reshape(1), 1e-3)
    _close(dimg, gi, 1e-3)
    _close(dtxt, gt, 1e-3)
