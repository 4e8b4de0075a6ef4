"""Per-sample losses (siglip_request_sample_losses, return_sample_losses=True) on the H100.

Accuracy: image_loss / text_loss against the float64 oracle of tests/sample_losses_oracle.py, per sample within 1e-3
relative (largest error observed on an H100: 4.3e-6 against the oracle of the kernel's own bf16 operands, and 5.9e-4
through the module with bf16 normalize_inputs, where the oracle normalises in float64 and the kernel takes the normalised
embeddings rounded to bf16), at W = 1 on partial-tile shapes and at
B = 16384, D = 1024; with positional labels, ids, hard negatives, extra texts with ids, extra images with and without
ids, weights (weight-0 samples exactly 0), the trained-regime generator (t = 100 and 300), fp32 and normalize_inputs
inputs through the module, and the fused, split and forward-only schedules. Bitwise: arming changes no loss, gradient
or metric bit, and the per-sample outputs are the same bits across repeated steps, schedules, cluster shapes
(cta_group 1 / 2, mcast) and stage counts, with metrics armed or not. Loopback W = 3 (uneven) and W = 4 (bidir) with
seeded peer partials, a CUDA-graph capture (the first request allocating the workspace), the launch counts and the
error statuses."""
import ctypes
import math

import numpy as np
import pytest
import torch

from extra_images_oracle import label_blocks
from sample_losses_oracle import sample_losses
from test_gpu_extra_images import _data, _engine, _ids, _prepare
from trained_regime import REGIMES, make_batch

pytestmark = pytest.mark.gpu

TOL = 1e-3
TP, BIAS = math.log(10.0), -10.0
WORST = {}


def _dev():
    return torch.device("cuda", 0)


def _scal(x):
    return torch.tensor([x], device=_dev(), dtype=torch.float32)


def _bufs(eng):
    return (torch.full((eng.images,), -1.0, device=_dev()), torch.full((eng.texts,), -1.0, device=_dev()))


def _mbufs(eng):
    return (torch.full((2,), -1.0, device=_dev()), torch.full((eng.metric_images,), -7, device=_dev(), dtype=torch.int64),
            torch.full((eng.metric_texts,), -7, device=_dev(), dtype=torch.int64))


def _step(eng, sched, img, txt, tp, b, losses=None, metrics=None, gdt=torch.float32):
    if metrics is not None:
        eng.request_metrics(*metrics)
    if losses is not None:
        eng.request_sample_losses(*losses)
    if sched == "fused":
        outs = list(eng.fwd_bwd(img, txt, tp, b, gdt))
    elif sched == "split":
        loss = eng.forward(img, txt, tp, b, True)
        outs = [loss] + list(eng.backward(img, txt, tp, None, gdt))
    else:
        outs = [eng.fwd(img, txt, tp, b)]
    if eng.world > 1:
        outs += [eng.debug_get_slot(k) for k in range(eng.world) if k != eng.rank]
    return [x.clone() for x in outs]


def _check(tag, got, want, zero=None):
    """Per-sample relative error; samples flagged in `zero` must be exactly 0."""
    g = got.double().cpu().numpy()
    w = np.asarray(want, np.float64)
    assert np.isfinite(g).all(), f"{tag}: non-finite values"
    if zero is not None and zero.any():
        assert (g[zero] == 0).all(), f"{tag}: a weight-0 sample is not exactly 0"
    keep = w > 0
    err = float(np.max(np.abs(g[keep] - w[keep]) / w[keep])) if keep.any() else 0.0
    WORST[tag] = err
    print(f"{tag}: max per-sample rel error {err:.3e}")
    assert err <= TOL, f"{tag}: max per-sample rel error {err:.3e}"


def _identity(tag, img_loss, loss, B):
    s = float(img_loss.double().sum()) / B
    loss = float(loss.detach())
    assert abs(s - loss) <= 1e-5 * abs(loss), f"{tag}: image_loss.sum()/B {s} vs loss {loss}"


def _weights(seed, R, T):
    g = torch.Generator().manual_seed(seed)
    wi = torch.where(torch.rand(R, generator=g) < 0.2, 0.0, torch.rand(R, generator=g))
    wt = torch.where(torch.rand(T, generator=g) < 0.2, 0.0, torch.rand(T, generator=g))
    return wi, wt


# ---------------------------------------------------------------------------------------------------------------------
# 1. one rank against the oracle; arming changes no bit of the step
# ---------------------------------------------------------------------------------------------------------------------
CASES = [
    # B, R, T, D, labels, weights, schedule
    (300, 300, 300, 136, "pos", False, "fused"),
    (300, 300, 300, 136, "pos", False, "split"),
    (300, 300, 300, 136, "pos", False, "fwd"),
    (1000, 1000, 1000, 264, "pos", False, "fused"),
    (1000, 1000, 1000, 264, "ids", True, "split"),
    (300, 300, 340, 136, "hn", True, "fused"),         # hard negatives
    (300, 300, 360, 136, "xt", False, "fwd"),          # extra texts with ids
    (300, 364, 300, 136, "pos", True, "split"),        # extra (hard-negative) images
    (300, 364, 330, 136, "xi", True, "fused"),         # extra images and extra texts, both with ids
]


@pytest.mark.parametrize("B,R,T,D,mode,weights,sched", CASES)
def test_single_rank_matches_oracle_and_changes_no_bit(B, R, T, D, mode, weights, sched):
    Bs, Rs, Ts = (B,), (R,), (T,)
    imgs, txts = _data(Bs, Rs, Ts, D, seed=B + R + T)
    ids = xt = xi = None
    flags = {}
    if mode in ("ids", "xt", "xi"):
        ids, xt, xi = _ids(Bs, Rs, Ts, seed=3)
        flags = dict(ids=True, xtxt_ids=mode in ("xt", "xi") and T > B, ximg_ids=mode == "xi")
    wi = wt = None
    if weights:
        wi, wt = _weights(R + T, R, T)
    plain = _engine(0, Bs, Rs, Ts, D, weights=weights, **flags)
    armed = _engine(0, Bs, Rs, Ts, D, weights=weights, **flags)
    img, txt = imgs[0].to(_dev()), txts[0].to(_dev())
    tp, b = _scal(TP), _scal(BIAS)
    wiL, wtL = ([wi], [wt]) if weights else (None, None)
    _prepare(plain, 0, txts, ids, xt, xi, wiL, wtL)
    a = _step(plain, sched, img, txt, tp, b)
    _prepare(armed, 0, txts, ids, xt, xi, wiL, wtL)
    bufs = _bufs(armed)
    c = _step(armed, sched, img, txt, tp, b, losses=bufs)
    torch.cuda.synchronize()
    for x, y in zip(a, c):
        assert torch.equal(x, y), f"{mode} {sched}: the armed step differs from the plain one"
    xt_l = [xt[0]] if flags.get("xtxt_ids") else None
    xi_l = [xi[0]] if flags.get("ximg_ids") else None
    labels = label_blocks(Bs, Rs, Ts, ids, xt_l, xi_l)
    ref = sample_losses([imgs[0].float().numpy()], [txts[0].float().numpy()], Bs, TP, BIAS, labels,
                        None if wi is None else [wi.numpy()], None if wt is None else [wt.numpy()])[0]
    tag = f"W=1 {B}x{T} R={R} D={D} {mode} w={weights} {sched}"
    _check(tag + " image_loss", bufs[0], ref["image_loss"], None if wi is None else wi.numpy() == 0)
    _check(tag + " text_loss", bufs[1], ref["text_loss"], None if wt is None else wt.numpy() == 0)
    _identity(tag, bufs[0], c[0], B)
    plain.close()
    armed.close()


@pytest.mark.parametrize("regime", ["trained", "t300"])
def test_trained_regime(regime):
    R_ = REGIMES[regime]
    B, D = 1000, 264
    (img,), (txt,), _, _ = make_batch(R_, (B,), (0,), D, 7, "pos")
    eng = _engine(0, (B,), (B,), (B,), D)
    tp, b = _scal(R_.t_prime), _scal(R_.bias)
    bufs = _bufs(eng)
    out = _step(eng, "fused", img.to(_dev()), txt.to(_dev()), tp, b, losses=bufs)
    torch.cuda.synchronize()
    ref = sample_losses([img.float().numpy()], [txt.float().numpy()], (B,), R_.t_prime, R_.bias)[0]
    _check(f"{regime} image_loss", bufs[0], ref["image_loss"])
    _check(f"{regime} text_loss", bufs[1], ref["text_loss"])
    _identity(regime, bufs[0], out[0], B)
    eng.close()


def test_large_batch_against_a_float64_reference():
    """B = 16384, D = 1024, bf16: the reference sums of the float64 logits are formed on the GPU in float64."""
    B, D = 16384, 1024
    g = torch.Generator().manual_seed(16384)
    img = torch.nn.functional.normalize(torch.randn(B, D, generator=g)).to(torch.bfloat16).to(_dev())
    txt = torch.nn.functional.normalize(torch.randn(B, D, generator=g)).to(torch.bfloat16).to(_dev())
    eng = _engine(0, (B,), (B,), (B,), D)
    bufs = _bufs(eng)
    out = _step(eng, "fused", img, txt, _scal(TP), _scal(BIAS), losses=bufs)
    z = math.exp(TP) * (img.double() @ txt.double().T) + BIAS
    z.diagonal().neg_()
    L = torch.nn.functional.softplus(z)
    ri, rt = L.sum(1).cpu().numpy(), L.sum(0).cpu().numpy()
    del z, L
    _check("B=16384 image_loss", bufs[0], ri)
    _check("B=16384 text_loss", bufs[1], rt)
    _identity("B=16384", bufs[0], out[0], B)
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. the same bits across schedules, cluster shapes, stage counts and repeated steps, with metrics armed or not
# ---------------------------------------------------------------------------------------------------------------------
def test_bitwise_reproducible_across_configurations():
    from distributed_sigmoid_loss_b200 import _capi

    Bs, Rs, Ts, D = (1000,), (1040,), (1064,), 264
    imgs, txts = _data(Bs, Rs, Ts, D, seed=9)
    ids, xt, xi = _ids(Bs, Rs, Ts, seed=9)
    wi, wt = _weights(9, Rs[0], Ts[0])
    img, txt = imgs[0].to(_dev()), txts[0].to(_dev())
    tp, b = _scal(TP), _scal(BIAS)
    first = None
    for cg, mcast, stages in [(2, 1, 0), (1, 1, 0), (2, 2, 0), (1, 2, 4), (2, 1, 4)]:
        kw = dict(cg=cg, mcast=mcast, ids=True, xtxt_ids=True, ximg_ids=True, weights=True)
        plain, armed = _engine(0, Bs, Rs, Ts, D, **kw), _engine(0, Bs, Rs, Ts, D, **kw)
        for e in (plain, armed):
            if stages:
                e.set_option(_capi.SIGLIP_OPT_STAGES_LOSS, stages)
        for sched in ("fused", "split", "fwd"):
            for with_metrics in (False, True):
                _prepare(plain, 0, txts, ids, xt, xi, [wi], [wt])
                m0 = _mbufs(plain) if with_metrics else None
                a = _step(plain, sched, img, txt, tp, b, metrics=m0)
                for rep in range(2):
                    _prepare(armed, 0, txts, ids, xt, xi, [wi], [wt])
                    bufs = _bufs(armed)
                    m1 = _mbufs(armed) if with_metrics else None
                    c = _step(armed, sched, img, txt, tp, b, losses=bufs, metrics=m1)
                    torch.cuda.synchronize()
                    tag = f"cg={cg} mcast={mcast} stages={stages} {sched} metrics={with_metrics} rep={rep}"
                    for x, y in zip(a, c):
                        assert torch.equal(x, y), f"{tag}: the armed step differs from the plain one"
                    if with_metrics:
                        for x, y in zip(m0, m1):
                            assert torch.equal(x, y), f"{tag}: metrics differ from a metrics-only step"
                    if first is None:
                        first = [x.clone() for x in bufs]
                    assert torch.equal(bufs[0], first[0]) and torch.equal(bufs[1], first[1]), \
                        f"{tag}: per-sample losses differ from the first configuration"
        plain.close()
        armed.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. loopback W-rank schedules with seeded peer partials
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Bs,r,bidir", [((300, 200, 264), 1, False), ((256, 256, 256, 256), 2, True)])
@pytest.mark.parametrize("sched", ["fused", "fwd"])
def test_loopback_with_seeded_peer_partials(Bs, r, bidir, sched):
    from distributed_sigmoid_loss_b200 import _capi

    D = 136
    W = len(Bs)
    imgs, txts = _data(Bs, Bs, Bs, D, seed=W * 11)
    eng = _engine(r, Bs, Bs, Bs, D)
    if bidir:
        eng.set_option(_capi.SIGLIP_OPT_BIDIR, 1)
    _prepare(eng, r, txts, None, None, None, None, None)
    f = [x.float().numpy() for x in imgs], [x.float().numpy() for x in txts]
    ref = sample_losses(f[0], f[1], Bs, TP, BIAS)
    # peer p's partial of my chunk: its images' column sums over my texts, one fixed-point word per text
    t = math.exp(TP)
    labels = label_blocks(Bs, Bs, Bs)
    for p in range(W):
        if p == r:
            continue
        z = t * (f[0][p].astype(np.float64) @ f[1][r].astype(np.float64).T) + BIAS
        part = np.log1p(np.exp(-np.abs(-labels[p][r] * z))) + np.maximum(-labels[p][r] * z, 0)
        words = np.rint(part.sum(axis=0) * 2.0 ** 32).astype(np.int64)
        eng.debug_set_peer_sample_loss_partials(p, torch.from_numpy(words).to(_dev()))
    bufs = _bufs(eng)
    out = _step(eng, sched, imgs[r].to(_dev()), txts[r].to(_dev()), _scal(TP), _scal(BIAS), losses=bufs)
    torch.cuda.synchronize()
    tag = f"loopback W={W} r={r} bidir={bidir} {sched}"
    _check(tag + " image_loss", bufs[0], ref[r]["image_loss"])
    _check(tag + " text_loss", bufs[1], ref[r]["text_loss"])
    _identity(tag, bufs[0], out[0], Bs[r])
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. capture, workspace, launches, the modules, errors
# ---------------------------------------------------------------------------------------------------------------------
def test_first_request_inside_a_capture_allocates_the_workspace():
    B, D = 256, 128
    eng = _engine(0, (B,), (B,), (B,), D)
    imgs, txts = _data((B,), (B,), (B,), D, seed=44)
    img, txt = imgs[0].to(_dev()).clone(), txts[0].to(_dev()).clone()
    tp, b = _scal(TP), _scal(BIAS)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eng.fwd_bwd(img, txt, tp, b, torch.float32)   # warm-up without the request
        torch.cuda.synchronize()
        ws = eng.workspace_bytes
        bufs = _bufs(eng)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            eng.request_sample_losses(*bufs)
            eng.fwd_bwd(img, txt, tp, b, torch.float32)
    assert eng.workspace_bytes == ws + 32 * (B + B)
    for seed in (45, 46):
        i1, t1 = _data((B,), (B,), (B,), D, seed=seed)
        img.copy_(i1[0].to(_dev()))
        txt.copy_(t1[0].to(_dev()))
        graph.replay()
        torch.cuda.synchronize()
        ref = sample_losses([i1[0].float().numpy()], [t1[0].float().numpy()], (B,), TP, BIAS)[0]
        _check(f"graph replay {seed} image_loss", bufs[0], ref["image_loss"])
        _check(f"graph replay {seed} text_loss", bufs[1], ref["text_loss"])
    eng.close()


def test_launch_counts():
    B, D = 256, 128
    eng = _engine(0, (B,), (B,), (B,), D)
    imgs, txts = _data((B,), (B,), (B,), D, seed=47)
    img, txt = imgs[0].to(_dev()), txts[0].to(_dev())
    tp, b = _scal(TP), _scal(BIAS)

    def count(**kw):
        n = eng.launch_count
        _step(eng, "fused", img, txt, tp, b, **kw)
        return eng.launch_count - n

    plain = count()
    assert count(losses=_bufs(eng)) == plain + 2          # the memset and the finalisation
    assert count() == plain
    metrics = count(metrics=_mbufs(eng))
    assert count(losses=_bufs(eng), metrics=_mbufs(eng)) == metrics + 2
    eng.close()


@pytest.mark.parametrize("fp32,normalize", [(True, False), (True, True), (False, True)])
def test_modules_return_sample_losses(fp32, normalize):
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    B, D = 300, 136
    g = torch.Generator().manual_seed(61)
    x_i = torch.randn(B, D, generator=g)
    x_t = torch.randn(B, D, generator=g)
    if not normalize:
        x_i, x_t = torch.nn.functional.normalize(x_i), torch.nn.functional.normalize(x_t)
    dt = torch.float32 if fp32 else torch.bfloat16
    a = x_i.to(dt).to(_dev()).requires_grad_(True)
    t = x_t.to(dt).to(_dev()).requires_grad_(True)
    mod = DDPSigmoidLoss(B, normalize_inputs=normalize).to(_dev())
    loss, metrics, sl = mod(a, t, return_metrics=True, return_sample_losses=True)
    loss.backward()
    assert set(sl) == {"image_loss", "text_loss"} and not sl["image_loss"].requires_grad
    assert "i2t_top1" in metrics
    n_i = torch.nn.functional.normalize(a.detach().double()) if normalize else a.detach().double()
    n_t = torch.nn.functional.normalize(t.detach().double()) if normalize else t.detach().double()
    ref = sample_losses([n_i.cpu().numpy()], [n_t.cpu().numpy()], (B,), math.log(10.0), -10.0)[0]
    tag = f"module fp32={fp32} normalize={normalize}"
    _check(tag + " image_loss", sl["image_loss"], ref["image_loss"])
    _check(tag + " text_loss", sl["text_loss"], ref["text_loss"])
    _identity(tag, sl["image_loss"], loss, B)
    with torch.no_grad():
        loss2, sl2 = mod(a, t, return_sample_losses=True)
    assert torch.equal(sl2["image_loss"], sl["image_loss"]) and torch.equal(sl2["text_loss"], sl["text_loss"])
    if not normalize:   # SigLipLoss takes normalised features
        sig = SigLipLoss()
        out, sl3 = sig(a.detach(), t.detach(), torch.tensor(math.log(10.0), device=_dev()),
                       torch.tensor(-10.0, device=_dev()), output_dict=True, return_sample_losses=True)
        assert set(out) == {"contrastive_loss"}
        torch.testing.assert_close(sl3["image_loss"], sl["image_loss"], rtol=1e-5, atol=0)
        torch.testing.assert_close(sl3["text_loss"], sl["text_loss"], rtol=1e-5, atol=0)


def test_error_statuses():
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi

    B, D = 64, 64
    L = _capi.lib()
    eng = _engine(0, (B,), (B,), (B,), D)
    bufs = _bufs(eng)
    assert L.siglip_request_sample_losses(eng._h, None, bufs[1].data_ptr()) == _capi.SIGLIP_ERR_INVALID
    assert L.siglip_request_sample_losses(eng._h, bufs[0].data_ptr(), None) == _capi.SIGLIP_ERR_INVALID
    assert L.siglip_request_sample_losses(None, bufs[0].data_ptr(), bufs[1].data_ptr()) == _capi.SIGLIP_ERR_INVALID
    assert L.siglip_request_sample_losses(eng._h, bufs[0].data_ptr(), bufs[1].data_ptr()) == _capi.SIGLIP_OK
    h = torch.zeros(B, D, dtype=torch.bfloat16)
    ticket = ctypes.c_ulonglong(0)
    rc = L.siglip_host_submit(eng._h, h.data_ptr(), h.data_ptr(), 0.0, 0.0, ctypes.byref(ticket),
                              torch.cuda.current_stream().cuda_stream)
    assert rc == _capi.SIGLIP_ERR_STATE and b"per-sample losses" in L.siglip_last_error()
    eng.close()
    dis = SigmoidLossEngine(B, D, _dev(), teacher_dim=D)
    dis.set_option(_capi.SIGLIP_OPT_DISTILL, 1)
    bufs = _bufs(dis)
    assert L.siglip_request_sample_losses(dis._h, bufs[0].data_ptr(), bufs[1].data_ptr()) == _capi.SIGLIP_ERR_STATE
    dis.close()
