"""Distillation from a frozen teacher (SIGLIP_OPT_DISTILL, DDPSigmoidLoss / SigLipLoss(distill=lambda)) on the H100:
the engine against the float64 oracle at W = 1 and loopback W = 3 / W = 4 bidir (uneven batches, partial tiles, teacher
width != student width, sample ids, weights, both schedules), the metrics against the undistilled step, the modules with
bf16 / fp32 / normalize_inputs at trained-model logits, and the properties: a teacher equal to the student at lambda = 1
leaves no gradient, lambda -> 0 approaches the plain step, a teacher that requires grad is refused."""
import math

import pytest
import torch

from distill_oracle import closed_form_distill
from sample_weights_oracle import closed_form_weighted, label_blocks

pytestmark = pytest.mark.gpu

TOL = 1e-3
TP, BIAS = math.log(10.0), -10.0
TTP, TBIAS = math.log(20.0), -8.0


def _dev():
    return torch.device("cuda", 0)


def _scal(x):
    return torch.tensor([x], device=_dev(), dtype=torch.float32)


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return max(float((a - b).norm() / (b.norm() + 1e-300)), float((a - b).abs().max() / (b.abs().max() + 1e-300)))


def _check(name, got, ref, tol=TOL):
    err = _rel(got, ref)
    assert err <= tol, f"{name}: relative error {err:.3e}"


def _unit(g, n, D, scale=1.0):
    return (torch.nn.functional.normalize(torch.randn(n, D, generator=g)) * scale).to(torch.bfloat16)


def _engine(B, D, DT, W=1, r=0, Bs=None, cg=2, mcast=1, ids=False, weights=False, bidir=False):
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi

    eng = SigmoidLossEngine(B, D, _dev(), cta_group=cg, rank_world=(r, W), loopback=W > 1, batch_per_rank=Bs,
                            teacher_dim=DT)
    if mcast != 1:
        eng.set_option(_capi.SIGLIP_OPT_MCAST, mcast)
    if bidir:
        eng.set_option(_capi.SIGLIP_OPT_BIDIR, 1)
    if ids:
        eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 1)
    if weights:
        eng.set_option(_capi.SIGLIP_OPT_SAMPLE_WEIGHTS, 1)
    eng.set_option(_capi.SIGLIP_OPT_DISTILL, 1)
    return eng


def _problem(Bs, D, DT, seed, ids=False, weights=False, tscale=1.0):
    g = torch.Generator().manual_seed(seed)
    P = dict(imgs=[_unit(g, b, D) for b in Bs], txts=[_unit(g, b, D) for b in Bs],
             timgs=[_unit(g, b, DT, tscale) for b in Bs], ttxts=[_unit(g, b, DT, tscale) for b in Bs], ids=None,
             iws=None, tws=None)
    if ids:
        P["ids"] = list(torch.split(torch.randint(0, max(Bs), (sum(Bs),), generator=g), list(Bs)))
    if weights:
        P["iws"] = [torch.rand(b, generator=g) for b in Bs]
        P["tws"] = [torch.rand(b, generator=g) for b in Bs]
        P["iws"][0][::7] = 0.0
    return P


def _oracle(P, lam, r=None):
    f = (lambda xs: None if xs is None else [x.double().numpy() for x in xs])  # noqa: E731
    Bs = [x.shape[0] for x in P["imgs"]]
    labels = label_blocks(Bs, Bs, f(P["ids"]) if P["ids"] is not None else None)
    return closed_form_distill(f(P["imgs"]), f(P["txts"]), TP, BIAS, f(P["timgs"]), f(P["ttxts"]), TTP, TBIAS, lam,
                               f(P["iws"]), f(P["tws"]), labels)


def _step(eng, P, r, lam, sched, tp=TP, bias=BIAS, ttp=TTP, tbias=TBIAS, metrics=None):
    d = _dev()
    W = eng.world
    for k in range(W):
        if W > 1:
            eng.debug_set_text_chunk(k, P["txts"][k].to(d))
            eng.debug_set_teacher_text_chunk(k, P["ttxts"][k].to(d))
            if k != r and P["ids"] is not None:
                eng.debug_set_chunk_ids(k, P["ids"][k].to(d))
            if k != r and P["tws"] is not None:
                eng.debug_set_chunk_weights(k, P["tws"][k].to(d))
    if P["ids"] is not None:
        eng.set_sample_ids(P["ids"][r].to(d))
    if P["tws"] is not None:
        eng.set_sample_weights(P["iws"][r].to(d), P["tws"][r].to(d))
    timg, ttxt = P["timgs"][r].to(d), P["ttxts"][r].to(d)
    tsc = (_scal(ttp), _scal(tbias))
    eng.set_teacher(timg, ttxt, *tsc, lam)
    if metrics is not None:
        eng.request_metrics(*metrics)
    img, txt = P["imgs"][r].to(d), P["txts"][r].to(d)
    if sched == "fused":
        loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, _scal(tp), _scal(bias))
    else:
        loss = eng.forward(img, txt, _scal(tp), _scal(bias), True)
        dimg, dtxt, dtp, db = eng.backward(img, txt, _scal(tp), None)
    out = [loss, dimg, dtxt, dtp, db]
    if W > 1:
        out += [eng.debug_get_slot(k) for k in range(W) if k != r]
    torch.cuda.synchronize()
    return [x.clone() for x in out]


def _check_step(tag, out, ref, r, W):
    _check(f"{tag} loss", out[0], ref["loss"])
    _check(f"{tag} dimg", out[1], ref["dimg"])
    _check(f"{tag} dt_prime", out[3], ref["dt_prime"])
    _check(f"{tag} dbias", out[4], ref["dbias"])
    slots = iter(out[5:])
    for k in range(W):
        got = out[2].float() if k == r else next(slots)
        _check(f"{tag} contribution to chunk {k}", got, ref["contrib"][k])


@pytest.mark.parametrize("sched", ["fused", "split"])
@pytest.mark.parametrize("cg,mcast", [(1, 1), (2, 1), (2, 2)])
@pytest.mark.parametrize("B,D,DT", [(300, 136, 64), (512, 64, 136), (1000, 264, 72)])
def test_single_rank_matches_the_oracle(B, D, DT, cg, mcast, sched):
    P = _problem([B], D, DT, seed=B + D + DT, tscale=1.0)
    eng = _engine(B, D, DT, cg=cg, mcast=mcast)
    for lam in (1.0, 0.5):
        out = _step(eng, P, 0, lam, sched)
        _check_step(f"W=1 lam={lam}", out, _oracle(P, lam)[0], 0, 1)


@pytest.mark.parametrize("sched", ["fused", "split"])
@pytest.mark.parametrize("ids,weights", [(False, False), (True, False), (False, True), (True, True)])
@pytest.mark.parametrize("Bs,bidir", [([200, 130, 257], False), ([64, 96, 40, 128], True)])
def test_loopback_matches_the_oracle(Bs, bidir, ids, weights, sched):
    W = len(Bs)
    P = _problem(Bs, 136, 72, seed=W * 31 + ids + 2 * weights, ids=ids, weights=weights)
    for r in range(W):
        eng = _engine(Bs[r], 136, 72, W=W, r=r, Bs=Bs, ids=ids, weights=weights, bidir=bidir)
        out = _step(eng, P, r, 0.7, sched)
        _check_step(f"W={W} rank {r}", out, _oracle(P, 0.7)[r], r, W)
        eng.close()


def test_weight_zero_samples_drop_out_exactly():
    B, D, DT = 384, 128, 96
    P = _problem([B], D, DT, seed=5, weights=True)
    keep = P["iws"][0] > 0
    eng = _engine(B, D, DT, weights=True)
    out = _step(eng, P, 0, 0.8, "fused")
    assert torch.all(out[1][~keep.to(_dev())] == 0)
    assert torch.all(out[2][(P["tws"][0] == 0).to(_dev())] == 0)


def test_teacher_equal_to_student_leaves_no_gradient():
    B, D = 512, 128
    g = torch.Generator().manual_seed(3)
    img, txt = _unit(g, B, D), _unit(g, B, D)
    P = dict(imgs=[img], txts=[txt], timgs=[img], ttxts=[txt], ids=None, iws=None, tws=None)
    eng = _engine(B, D, D)
    out = _step(eng, P, 0, 1.0, "fused", ttp=TP, tbias=BIAS)
    hard = closed_form_weighted([img.double().numpy()], [txt.double().numpy()], TP, BIAS)[0]
    for i, k in ((1, "dimg"), (3, "dt_prime"), (4, "dbias")):
        assert float(out[i].double().norm()) <= 1e-5 * float(torch.as_tensor(hard[k]).norm()), k
    assert float(out[2].double().norm()) <= 1e-5 * float(torch.as_tensor(hard["contrib"][0]).norm())


def test_small_lambda_approaches_the_plain_step():
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine

    B, D, DT = 512, 128, 64
    P = _problem([B], D, DT, seed=9)
    plain = SigmoidLossEngine(B, D, _dev())
    d = _dev()
    ref = plain.fwd_bwd(P["imgs"][0].to(d), P["txts"][0].to(d), _scal(TP), _scal(BIAS))
    eng = _engine(B, D, DT)
    prev = None
    for lam in (1e-1, 1e-2, 1e-3):
        out = _step(eng, P, 0, lam, "fused")
        err = _rel(out[1], ref[1])
        assert prev is None or err < prev
        prev = err
    assert prev < 5e-3


def test_metrics_equal_the_undistilled_step():
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine

    B, D, DT = 700, 128, 64
    P = _problem([B], D, DT, seed=11)
    d = _dev()
    bufs = lambda: (torch.empty(2, device=d), torch.empty(B, device=d, dtype=torch.int64),  # noqa: E731
                    torch.empty(B, device=d, dtype=torch.int64))
    plain = SigmoidLossEngine(B, D, d)
    m0 = bufs()
    plain.request_metrics(*m0)
    plain.fwd_bwd(P["imgs"][0].to(d), P["txts"][0].to(d), _scal(TP), _scal(BIAS))
    m1 = bufs()
    _step(_engine(B, D, DT), P, 0, 0.5, "fused", metrics=m1)
    for a, b in zip(m0, m1):
        assert torch.equal(a, b)


@pytest.mark.parametrize("dtype,normalize", [(torch.bfloat16, False), (torch.float32, False), (torch.float32, True)])
@pytest.mark.parametrize("fused", [True, False])
def test_modules_match_the_oracle(dtype, normalize, fused):
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    B, D, DT = 640, 136, 60   # a teacher width that is no multiple of 8
    g = torch.Generator().manual_seed(2)
    img = torch.randn(B, D, generator=g).to(dtype)
    txt = torch.randn(B, D, generator=g).to(dtype)
    timg = torch.randn(B, DT, generator=g).to(dtype)
    ttxt = torch.randn(B, DT, generator=g).to(dtype)
    if not normalize:
        img, txt, timg, ttxt = (torch.nn.functional.normalize(x.float()).to(dtype) for x in (img, txt, timg, ttxt))
    d = _dev()
    nz = (lambda x: torch.nn.functional.normalize(x.double())) if normalize else (lambda x: x.double())  # noqa: E731
    ref = closed_form_distill([nz(img).numpy()], [nz(txt).numpy()], TP, BIAS, [nz(timg).numpy()], [nz(ttxt).numpy()],
                              TTP, TBIAS, 0.6)[0]
    mod = DDPSigmoidLoss(B, normalize_inputs=normalize, fused_step=fused, distill=0.6).to(d)
    a, b = img.to(d).requires_grad_(True), txt.to(d).requires_grad_(True)
    loss = mod(a, b, teacher_image=timg.to(d), teacher_text=ttxt.to(d),
               teacher_t_prime=torch.tensor(TTP, device=d, dtype=torch.float64),
               teacher_bias=torch.tensor(TBIAS, device=d))
    loss.backward()
    tol = TOL + (2 ** -8 if dtype == torch.bfloat16 else 0.0)   # bf16 gradients carry their own rounding
    if normalize:
        # gradients with respect to the raw inputs: chain through F.normalize in float64
        x, y = img.double().requires_grad_(True), txt.double().requires_grad_(True)
        xn, yn = torch.nn.functional.normalize(x), torch.nn.functional.normalize(y)
        (xn * torch.as_tensor(ref["dimg"])).sum().backward()
        (yn * torch.as_tensor(ref["contrib"][0])).sum().backward()
        gi, gt = x.grad, y.grad
    else:
        gi, gt = ref["dimg"], ref["contrib"][0]
    _check("module loss", loss.detach(), ref["loss"])
    _check("module dimg", a.grad, gi, tol)
    _check("module dtxt", b.grad, gt, tol)
    _check("module dt'", mod.t_prime.grad, ref["dt_prime"])
    _check("module dbias", mod.bias.grad, ref["dbias"])
    sl = SigLipLoss(world_size=1, fused_step=fused, distill=0.6)
    a2, b2 = (nz(img).to(dtype) if normalize else img).to(d), (nz(txt).to(dtype) if normalize else txt).to(d)
    loss2 = sl(a2, b2, _scal(TP), _scal(BIAS), teacher_image=(nz(timg).to(dtype) if normalize else timg).to(d),
               teacher_text=(nz(ttxt).to(dtype) if normalize else ttxt).to(d), teacher_logit_scale=_scal(TTP)[0],
               teacher_logit_bias=_scal(TBIAS)[0])
    _check("SigLipLoss loss", loss2.detach(), ref["loss"], tol)


def test_trained_regime_logits_match_the_oracle():
    from trained_regime import REGIMES, make_batch

    B, D, DT = 1024, 256, 128
    st, te = REGIMES["trained"], REGIMES["separated"]
    imgs, txts, _, _ = make_batch(st, [B], [0], D, seed=4)
    timgs, ttxts, _, _ = make_batch(te, [B], [0], DT, seed=5)
    P = dict(imgs=imgs, txts=txts, timgs=timgs, ttxts=ttxts, ids=None, iws=None, tws=None)
    tp, ttp = math.log(st.t), math.log(te.t)
    eng = _engine(B, D, DT)
    f = (lambda xs: [x.double().numpy() for x in xs])  # noqa: E731
    for lam in (1.0, 0.3):
        out = _step(eng, P, 0, lam, "fused", tp=tp, bias=st.bias, ttp=ttp, tbias=te.bias)
        ref = closed_form_distill(f(imgs), f(txts), tp, st.bias, f(timgs), f(ttxts), ttp, te.bias, lam)[0]
        _check_step(f"trained lam={lam}", out, ref, 0, 1)


def test_teacher_that_requires_grad_is_refused():
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss

    B, D = 64, 32
    d = _dev()
    mod = DDPSigmoidLoss(B, distill=1.0).to(d)
    x = torch.nn.functional.normalize(torch.randn(B, D, device=d))
    with pytest.raises(RuntimeError, match="requires grad"):
        mod(x, x, teacher_image=x.clone().requires_grad_(True), teacher_text=x, teacher_t_prime=_scal(TTP)[0],
            teacher_bias=_scal(TBIAS)[0])


def test_step_without_set_teacher_is_a_state_error():
    from distributed_sigmoid_loss_b200 import _capi

    B, D = 256, 64
    eng = _engine(B, D, 64)
    img = torch.zeros(B, D, device=_dev(), dtype=torch.bfloat16)
    before = eng.launch_count
    with pytest.raises(_capi.SiglipError) as e:
        eng.fwd_bwd(img, img, _scal(TP), _scal(BIAS))
    assert e.value.code == _capi.SIGLIP_ERR_STATE and eng.launch_count == before
