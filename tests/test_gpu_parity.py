"""Parity of the sm_90a path against the reference (golden fixtures from the unmodified reference, and the pinned
oracle at sizes the fixtures do not reach). Everything here goes through the C ABI (ctypes) or the module mirror.

Tolerances (BASELINE.json north_star: "within 1e-3 relative of the reference"):
  * loss, dt', dbias : |x - ref| <= 1e-3 |ref|        (observed ~1e-6)
  * dimg, dtxt       : relative Frobenius error <= 1e-3 and max-abs error <= 1e-3 max|ref|   (SURVEY.md §8c)
The kernels emit fp32 gradients; the module casts them to the input dtype exactly like autograd does.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from conftest import golden_cases, load_golden

pytestmark = pytest.mark.gpu

TOL = 1e-3


def _dev():
    return torch.device("cuda", 0)


def _rel_f(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-300))


def _max_rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-300))


def _check(name, got, ref, tol=TOL, max_tol=None):
    if np.ndim(ref) == 0 and not torch.is_tensor(ref):
        err = abs(float(got) - float(ref)) / (abs(float(ref)) + 1e-30)
        assert err <= tol, f"{name}: {float(got)} vs {float(ref)} (rel {err:.3e})"
    else:
        ef, em = _rel_f(got, ref), _max_rel(got, ref)
        mt = tol if max_tol is None else max_tol
        assert ef <= tol and em <= mt, f"{name}: rel-Frobenius {ef:.3e}, max-abs/max {em:.3e}"


def _engine(B, D, cg=2, **kw):
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine

    return SigmoidLossEngine(B, D, _dev(), cta_group=cg, **kw)


def _scal(x):
    return torch.tensor([x], device=_dev(), dtype=torch.float32)


def _contribution(eng, k, dtxt):
    """This rank's contribution to the text gradient of chunk k in a loopback context: slot k for another rank's
    chunk; for the own chunk the step's dtxt output (own contribution + the all-zero "peer" contributions)."""
    return dtxt.float() if k == eng.rank else eng.debug_get_slot(k)


# ---------------------------------------------------------------------------------------------------------
# operand layouts of the wgmma mainloop
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("a_f16", [0, 1])
@pytest.mark.parametrize("amn,bmn", [(0, 0), (0, 1), (1, 1), (1, 0)])
def test_mainloop_operand_layouts(cg, amn, bmn, a_f16, monkeypatch):
    """K-major / MN-major operands, cta_group 1 and 2, bf16 x bf16 (loss kernel) and fp16 x fp16 (gradient kernel:
    scaled sigma operand x scaled embeddings)."""
    from distributed_sigmoid_loss_b200 import _capi

    L = _capi.lib()
    dev = _dev()
    torch.manual_seed(0)
    adt = torch.float16 if a_f16 else torch.bfloat16
    if a_f16:
        monkeypatch.setenv("SIGLIP_DEBUG_AB_F16", "1")
    else:
        monkeypatch.delenv("SIGLIP_DEBUG_AB_F16", raising=False)
    for (M, N, K) in [(256, 256, 64), (512, 768, 1024), (300, 264, 200), (128, 256, 64), (2000, 520, 328),
                      (512, 384, 256), (640, 1152, 192), (256, 128, 128), (256, 72, 64)]:
        A = torch.randn(M, K, device=dev).to(adt)
        B = torch.randn(N, K, device=dev).to(adt)
        ref = A.float() @ B.float().T

        def store(X, mn):
            if not mn:
                ld = (X.shape[1] + 7) // 8 * 8
                buf = torch.zeros(X.shape[0], ld, device=dev, dtype=X.dtype)
                buf[:, : X.shape[1]] = X
            else:
                ld = (X.shape[0] + 7) // 8 * 8
                buf = torch.zeros(X.shape[1], ld, device=dev, dtype=X.dtype)
                buf[:, : X.shape[0]] = X.T
            return buf, ld

        Ab, lda = store(A, amn)
        Bb, ldb = store(B, bmn)
        C = torch.full((M, N), float("nan"), device=dev, dtype=torch.float32)
        rc = L.siglip_debug_gemm(0, cg, M, N, K, Ab.data_ptr(), lda, amn, Bb.data_ptr(), ldb, bmn, C.data_ptr(), N,
                                 torch.cuda.current_stream().cuda_stream)
        assert rc == 0, _capi.last_error()
        torch.cuda.synchronize()
        assert not torch.isnan(C).any()
        # fp32 accumulation of exact bf16 products: only summation-order noise
        assert float((C - ref).abs().max()) <= 1e-5 * float(ref.abs().max()) * math.sqrt(K) + 1e-4


# ---------------------------------------------------------------------------------------------------------
# golden fixtures: the reference's own outputs
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cg", [1, 2])
def test_mainloop_multicast_clusters(cg, monkeypatch):
    """SIGLIP_OPT_MCAST = 2: clusters of two CTAs (cg 1) or two MMA pairs (cg 2, a 2x2 cluster) share the B tile through
    TMA multicast; odd tile-row counts leave a fully masked phantom tile."""
    from distributed_sigmoid_loss_b200 import _capi

    L = _capi.lib()
    dev = _dev()
    torch.manual_seed(1)
    monkeypatch.setenv("SIGLIP_DEBUG_MCAST", "2")
    monkeypatch.delenv("SIGLIP_DEBUG_AB_F16", raising=False)
    for (M, N, K, bmn) in [(512, 512, 256, 0), (768, 520, 320, 1), (300, 264, 200, 0), (1300, 1024, 512, 1)]:
        A = torch.randn(M, K, device=dev).to(torch.bfloat16)
        B = torch.randn(N, K, device=dev).to(torch.bfloat16)
        ref = A.float() @ B.float().T
        Bb = B.T.contiguous() if bmn else B
        C = torch.full((M, N), float("nan"), device=dev, dtype=torch.float32)
        rc = L.siglip_debug_gemm(0, cg, M, N, K, A.data_ptr(), K, 0, Bb.data_ptr(), Bb.shape[1], bmn, C.data_ptr(), N,
                                 torch.cuda.current_stream().cuda_stream)
        assert rc == 0, _capi.last_error()
        torch.cuda.synchronize()
        assert float((C - ref).abs().max()) <= 1e-5 * float(ref.abs().max()) * math.sqrt(K) + 1e-4


def _golden_rank_inputs(c, r):
    B = c["batch"]
    img = torch.from_numpy(c["img_all"][r * B:(r + 1) * B]).to(torch.bfloat16).to(_dev()).contiguous()
    txt = torch.from_numpy(c["txt_all"][r * B:(r + 1) * B]).to(torch.bfloat16).to(_dev()).contiguous()
    return img, txt


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("name", [n for n in golden_cases() if n.startswith("w1_")])
def test_single_rank_matches_reference_fixture(name, cg):
    c = load_golden(name)
    img, txt = _golden_rank_inputs(c, 0)
    # fixtures hold bf16-representable inputs: the conversion above is exact
    assert torch.equal(img.float().cpu(), torch.from_numpy(c["img_all"]))
    eng = _engine(c["batch"], c["dim"], cg)
    loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, _scal(c["t_prime"]), _scal(c["bias"]))
    loss_f = eng.fwd(img, txt, _scal(c["t_prime"]), _scal(c["bias"]))
    torch.cuda.synchronize()
    for variant in ("ddp", "rw_bidir"):
        ref = c["variants"][variant][0]
        _check("loss", loss, ref["loss"])
        _check("loss (forward only)", loss_f, ref["loss"])
        _check("dimg", dimg, ref["dimg"])
        _check("dtxt", dtxt, ref["dtxt"])
        _check("dt_prime", dtp, ref["dt_prime"])
        _check("dbias", db, ref["dbias"])
    eng.close()


@pytest.mark.parametrize("name", [n for n in golden_cases() if not n.startswith("w1_")])
def test_multi_chunk_schedule_matches_reference_fixture(name):
    """One GPU plays every rank of the W-rank job in turn (loopback context): per-rank loss / dimg / dt' / dbias must
    equal the reference's rank outputs, and the per-owner dtxt contributions summed over ranks must equal the text
    gradient the reference gets from all_gather's backward (distributed_sigmoid_loss.py:35)."""
    c = load_golden(name)
    W, B, D = c["world"], c["batch"], c["dim"]
    dtxt_sum = [torch.zeros(B, D, device=_dev()) for _ in range(W)]
    for r in range(W):
        eng = _engine(B, D, 2, rank_world=(r, W), loopback=True)
        for k in range(W):
            eng.debug_set_text_chunk(k, _golden_rank_inputs(c, k)[1])
        img, txt = _golden_rank_inputs(c, r)
        loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, _scal(c["t_prime"]), _scal(c["bias"]))
        n0 = eng.launch_count
        loss2, dimg2, dtxt2, _, _ = eng.fwd_bwd(img, txt, _scal(c["t_prime"]), _scal(c["bias"]))   # step-to-step flags
        assert eng.launch_count - n0 == 2 * W      # a W-chunk step is W loss + W gradient launches, nothing else
        loss_f = eng.fwd(img, txt, _scal(c["t_prime"]), _scal(c["bias"]))
        torch.cuda.synchronize()
        assert torch.equal(loss, loss2) and torch.equal(dimg, dimg2) and torch.equal(dtxt, dtxt2)
        ref = c["variants"]["ddp"][r]
        _check(f"loss r{r}", loss, ref["loss"])
        _check(f"loss fwd r{r}", loss_f, ref["loss"])
        _check(f"dimg r{r}", dimg, ref["dimg"])
        _check(f"dt_prime r{r}", dtp, ref["dt_prime"])
        _check(f"dbias r{r}", db, ref["dbias"])
        for k in range(W):
            dtxt_sum[k] += _contribution(eng, k, dtxt)
        torch.cuda.synchronize()
        eng.close()
    for k in range(W):
        _check(f"dtxt owner {k}", dtxt_sum[k], c["variants"]["ddp"][k]["dtxt"])
        _check(f"dtxt owner {k} (ring variant)", dtxt_sum[k], c["variants"]["rw_uni"][k]["dtxt"])


@pytest.mark.parametrize("name", ["w3_b5_d16", "w4_b8_d64", "w2_b24_d40_warm"])
@pytest.mark.parametrize("inkernel", [1, 0])
def test_split_api_and_helper_launch_variant_match_reference_fixture(name, inkernel):
    """The same loopback replay through (a) the split siglip_forward / siglip_backward API (one sigma operand per chunk
    kept between the calls, grad_out folded into the epilogues) and (b) the fused step with SIGLIP_OPT_INKERNEL_SYNC
    = 0 (flags handled by separate one-block kernels): identical results to the fused in-kernel default."""
    from distributed_sigmoid_loss_b200 import _capi
    c = load_golden(name)
    W, B, D = c["world"], c["batch"], c["dim"]
    dtxt_split = [torch.zeros(B, D, device=_dev()) for _ in range(W)]
    for r in range(W):
        eng = _engine(B, D, 2, rank_world=(r, W), loopback=True)
        eng.set_option(_capi.SIGLIP_OPT_INKERNEL_SYNC, inkernel)
        for k in range(W):
            eng.debug_set_text_chunk(k, _golden_rank_inputs(c, k)[1])
        img, txt = _golden_rank_inputs(c, r)
        tp, b = _scal(c["t_prime"]), _scal(c["bias"])
        loss_a, dimg_a, dtxt_a, dtp_a, db_a = eng.fwd_bwd(img, txt, tp, b)
        slots_a = [_contribution(eng, k, dtxt_a).clone() for k in range(W)]
        loss_b = eng.forward(img, txt, tp, b, True)
        dimg_b, dtxt_b, dtp_b, db_b = eng.backward(img, txt, tp, None)
        torch.cuda.synchronize()
        ref = c["variants"]["ddp"][r]
        _check(f"loss r{r}", loss_b, ref["loss"])
        _check(f"dimg r{r}", dimg_b, ref["dimg"])
        _check(f"dt_prime r{r}", dtp_b, ref["dt_prime"])
        _check(f"dbias r{r}", db_b, ref["dbias"])
        # same kernels on the same operands: the two schedules agree to the last bit
        assert torch.equal(loss_a, loss_b) and torch.equal(dimg_a, dimg_b)
        assert torch.equal(dtp_a, dtp_b) and torch.equal(db_a, db_b)
        for k in range(W):
            got = dtxt_b.float() if k == r else eng.debug_get_slot(k)
            assert torch.equal(got, slots_a[k])
            dtxt_split[k] += got
        torch.cuda.synchronize()
        eng.close()
    for k in range(W):
        _check(f"dtxt owner {k}", dtxt_split[k], c["variants"]["ddp"][k]["dtxt"])


# ---------------------------------------------------------------------------------------------------------
# sizes beyond the fixtures: fp32 autograd of the same math on the GPU (oracle.torch_reference_fp32, pinned on CPU)
# ---------------------------------------------------------------------------------------------------------
def _synth(B, D, seed=1234):
    g = torch.Generator().manual_seed(seed)
    img = torch.nn.functional.normalize(torch.randn(B, D, generator=g)).to(torch.bfloat16).to(_dev())
    txt = torch.nn.functional.normalize(torch.randn(B, D, generator=g)).to(torch.bfloat16).to(_dev())
    return img, txt


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("B,D,tp,bias", [
    (4096, 768, math.log(10.0), -10.0),    # BASELINE.json configs[1]
    (1000, 136, math.log(10.0), -10.0),    # ragged against every tile size
    (520, 264, math.log(20.0), -6.0),
    (2048, 1152, math.log(10.0), -10.0),   # D of configs[4]
])
def test_against_fp32_autograd(B, D, tp, bias, cg):
    from oracle.siglip_oracle import torch_reference_fp32

    img, txt = _synth(B, D)
    ref = torch_reference_fp32(img, [txt], tp, bias, 0)
    eng = _engine(B, D, cg)
    loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, _scal(tp), _scal(bias))
    torch.cuda.synchronize()
    _check("loss", loss, ref["loss"])
    _check("dimg", dimg, ref["dimg"])
    _check("dtxt", dtxt, ref["dtxt_chunks"][0])
    _check("dt_prime", dtp, ref["dt_prime"])
    _check("dbias", db, ref["dbias"])
    eng.close()


def test_warm_logits_general_path():
    """Logits around zero (t = 30, b = -3): every slab takes the general softplus/sigmoid path and the negatives carry
    real weight in the gradients (this is the case a bf16 sigma operand failed at 1.1e-3; the fp16 operand passes)."""
    from oracle.siglip_oracle import torch_reference_fp32

    B, D, tp, bias = 512, 256, math.log(30.0), -3.0
    img, txt = _synth(B, D)
    ref = torch_reference_fp32(img, [txt], tp, bias, 0)
    eng = _engine(B, D, 2)
    loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, _scal(tp), _scal(bias))
    torch.cuda.synchronize()
    _check("loss", loss, ref["loss"])
    _check("dt_prime", dtp, ref["dt_prime"])
    _check("dbias", db, ref["dbias"])
    _check("dimg", dimg, ref["dimg"])
    _check("dtxt", dtxt, ref["dtxt_chunks"][0])
    eng.close()


def test_two_chunks_large_loopback():
    from oracle.siglip_oracle import torch_reference_fp32

    B, D, W = 768, 512, 2
    img, txt0 = _synth(B, D, 1)
    _, txt1 = _synth(B, D, 2)
    chunks = [txt0, txt1]
    for r in range(W):
        ref = torch_reference_fp32(img, chunks, math.log(10.0), -10.0, r)
        eng = _engine(B, D, 2, rank_world=(r, W), loopback=True)
        for k in range(W):
            eng.debug_set_text_chunk(k, chunks[k])
        loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, chunks[r], _scal(math.log(10.0)), _scal(-10.0))
        torch.cuda.synchronize()
        _check("loss", loss, ref["loss"])
        _check("dimg", dimg, ref["dimg"])
        _check("dt_prime", dtp, ref["dt_prime"])
        _check("dbias", db, ref["dbias"])
        for k in range(W):
            _check(f"dtxt contribution to owner {k}", _contribution(eng, k, dtxt), ref["dtxt_chunks"][k])
        eng.close()


# ---------------------------------------------------------------------------------------------------------
# full headline size: direct comparison + size-independent properties
# ---------------------------------------------------------------------------------------------------------
def test_headline_shape_properties():
    from oracle.siglip_oracle import torch_reference_fp32

    B, D = 16384, 1024
    tp, bias = math.log(10.0), -10.0
    img, txt = _synth(B, D)
    eng = _engine(B, D, 2)
    loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, _scal(tp), _scal(bias))
    loss2, dimg2, dtxt2, dtp2, db2 = eng.fwd_bwd(img, txt, _scal(tp), _scal(bias))
    torch.cuda.synchronize()
    # determinism: fixed tile schedule and fixed-order reductions => bitwise repeatable
    assert torch.equal(loss, loss2) and torch.equal(dimg, dimg2) and torch.equal(dtxt, dtxt2)
    assert torch.equal(dtp, dtp2) and torch.equal(db, db2)
    # Euler-type identities of the math (SURVEY.md §0): <dimg, img> = <dtxt, txt> = dt'   (single rank)
    s_img = float((dimg.double() * img.double()).sum())
    s_txt = float((dtxt.double() * txt.double()).sum())
    assert abs(s_img - float(dtp)) <= 1e-3 * abs(float(dtp))
    assert abs(s_txt - float(dtp)) <= 1e-3 * abs(float(dtp))
    # permutation equivariance: permuting the pairs permutes the gradients and leaves the scalars unchanged
    perm = torch.randperm(B, device=_dev())
    lp, dip, dtp_p, dtpp, dbp = eng.fwd_bwd(img[perm].contiguous(), txt[perm].contiguous(), _scal(tp), _scal(bias))
    torch.cuda.synchronize()
    _check("loss under permutation", lp, float(loss), tol=1e-5)
    _check("dimg under permutation", dip, dimg[perm], tol=1e-4)
    _check("dtxt under permutation", dtp_p, dtxt[perm], tol=1e-4)
    # direct comparison with fp32 autograd at the full size (a few GiB of B x B intermediates on the GPU)
    ref = torch_reference_fp32(img, [txt], tp, bias, 0)
    _check("loss", loss, ref["loss"])
    _check("dimg", dimg, ref["dimg"])
    _check("dtxt", dtxt, ref["dtxt_chunks"][0])
    _check("dt_prime", dtp, ref["dt_prime"])
    _check("dbias", db, ref["dbias"])
    eng.close()


# ---------------------------------------------------------------------------------------------------------
# module mirror (the reference-facing surface)
# ---------------------------------------------------------------------------------------------------------
def test_module_forward_backward_like_reference():
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    c = load_golden("w1_b300_d136")
    ref = c["variants"]["ddp"][0]
    img, txt = _golden_rank_inputs(c, 0)
    a, b = img.clone().requires_grad_(True), txt.clone().requires_grad_(True)
    mod = DDPSigmoidLoss(c["batch"]).to(_dev())
    loss = mod(a, b)
    assert loss.dim() == 0 and loss.dtype == torch.float32
    (2.0 * loss).backward()                       # upstream gradient 2: backward only rescales the fused gradients
    assert a.grad.dtype == torch.bfloat16 and mod.t_prime.grad.dtype == torch.float64
    _check("loss", loss.detach(), ref["loss"])
    _check("dimg (bf16 output)", a.grad.float() / 2, ref["dimg"], tol=4e-3)   # bf16 rounding of the result
    _check("dtxt (bf16 output)", b.grad.float() / 2, ref["dtxt"], tol=4e-3)
    _check("dt_prime", mod.t_prime.grad / 2, ref["dt_prime"])
    _check("dbias", mod.bias.grad / 2, ref["dbias"])
    # fp32 inputs are accepted (rounded to bf16 internally; exact here because the fixture is bf16-representable)
    a32, b32 = img.float().requires_grad_(True), txt.float().requires_grad_(True)
    loss32 = mod(a32, b32)
    loss32.backward()
    assert a32.grad.dtype == torch.float32
    _check("dimg (fp32 output)", a32.grad, ref["dimg"])
    with torch.no_grad():
        _check("loss (no_grad)", mod(img, txt), ref["loss"])
    with pytest.raises(RuntimeError):
        mod(img[:100], txt[:100])                 # B != gpu_batch_size, like the reference's broadcast error
    # open_clip-signature adapter
    ref_rw = c["variants"]["rw_bidir"][0]
    scale = torch.nn.Parameter(torch.tensor(c["t_prime"], device=_dev(), dtype=torch.float32))
    lbias = torch.nn.Parameter(torch.tensor(c["bias"], device=_dev(), dtype=torch.float32))
    out = SigLipLoss(rank=0, world_size=1)(img.clone().requires_grad_(True), txt, scale, lbias, output_dict=True)
    out["contrastive_loss"].backward()
    _check("SigLipLoss loss", out["contrastive_loss"].detach(), ref_rw["loss"])
    _check("SigLipLoss dscale", scale.grad, ref_rw["dt_prime"])
    _check("SigLipLoss dbias", lbias.grad, ref_rw["dbias"])


def test_host_buffer_entry_matches_device_entry():
    B, D = 1024, 256
    img, txt = _synth(B, D)
    eng = _engine(B, D, 2)
    tp, bias = math.log(10.0), -10.0
    loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, _scal(tp), _scal(bias))
    torch.cuda.synchronize()
    ih, th = img.cpu().pin_memory(), txt.cpu().pin_memory()
    dih = torch.empty(B, D, dtype=torch.float32).pin_memory()
    dth = torch.empty(B, D, dtype=torch.float32).pin_memory()
    lh, dtph, dbh = eng.fwd_bwd_host(ih, th, tp, bias, dih, dth)
    assert lh == float(loss) and dtph == float(dtp) and dbh == float(db)
    assert torch.equal(dih, dimg.cpu()) and torch.equal(dth, dtxt.cpu())
    eng.close()


def test_pipelined_host_entry_keeps_steps_apart():
    """siglip_host_submit / siglip_host_wait with two steps in flight: the copies of step n+1 overlap the kernels of
    step n, every step must still see ITS inputs (two staging sets) and return ITS results (bitwise = device entry)."""
    B, D = 2048, 256
    eng = _engine(B, D, 2)
    steps = []
    for i in range(6):
        img, txt = _synth(B, D, seed=300 + i)
        tp, bias = math.log(10.0) + 0.05 * i, -10.0 + 0.5 * i
        loss, _, _, dtp, db = eng.fwd_bwd(img, txt, _scal(tp), _scal(bias))
        torch.cuda.synchronize()
        steps.append((img.cpu().pin_memory(), txt.cpu().pin_memory(), tp, bias, float(loss), float(dtp), float(db)))
    got = []
    prev = None
    for (ih, th, tp, bias, *_r) in steps:
        t = eng.host_submit(ih, th, tp, bias)
        if prev is not None:
            got.append(eng.host_wait(prev))
        prev = t
    got.append(eng.host_wait(prev))
    for i, (st, g) in enumerate(zip(steps, got)):
        assert g == (st[4], st[5], st[6]), f"step {i}: {g} vs {st[4:]}"
    with pytest.raises(RuntimeError):
        eng.host_wait(0)            # only the last two tickets are retrievable
    # the synchronous entry still works after pipelined use
    lh, dtph, dbh = eng.fwd_bwd_host(steps[2][0], steps[2][1], steps[2][2], steps[2][3])
    assert (lh, dtph, dbh) == (steps[2][4], steps[2][5], steps[2][6])
    eng.close()


def test_bf16_gradient_outputs_and_fused_scale():
    """SIGLIP_OPT_GRAD_BF16: the epilogue writes bf16 gradients = round-to-nearest of the fp32 ones; siglip_scale is
    the module's whole backward (multi-chunk dimg accumulation stays fp32 until the last chunk)."""
    B, D = 1024, 256
    img, txt = _synth(B, D)
    eng = _engine(B, D, 2)
    tp, bias = _scal(math.log(10.0)), _scal(-10.0)
    _, dimg32, dtxt32, _, _ = eng.fwd_bwd(img, txt, tp, bias)
    _, dimg16, dtxt16, _, _ = eng.fwd_bwd(img, txt, tp, bias, torch.bfloat16)
    torch.cuda.synchronize()
    assert dimg16.dtype == torch.bfloat16
    assert torch.equal(dimg16, dimg32.to(torch.bfloat16)) and torch.equal(dtxt16, dtxt32.to(torch.bfloat16))
    g = _scal(0.5)
    assert torch.equal(eng.scale(dimg32, g), dimg32 * 0.5)
    assert torch.equal(eng.scale(dimg16, g), (dimg16.float() * 0.5).to(torch.bfloat16))
    eng.close()
    # two chunks on one GPU (loopback): bf16 dimg of the last chunk == rounded fp32 result
    W = 2
    _, txt1 = _synth(B, D, 7)
    outs = []
    for dt in (torch.float32, torch.bfloat16):
        e2 = _engine(B, D, 2, rank_world=(0, W), loopback=True)
        e2.debug_set_text_chunk(0, txt)
        e2.debug_set_text_chunk(1, txt1)
        outs.append(e2.fwd_bwd(img, txt, tp, bias, dt)[1])
        torch.cuda.synchronize()
        e2.close()
    assert torch.equal(outs[1], outs[0].to(torch.bfloat16))


def test_split_forward_backward_and_generation_guard():
    """siglip_forward / siglip_backward: grad_out folded into the epilogues; a backward after an intervening forward of
    the same module recomputes the saved state instead of using stale sigma operands."""
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss

    B, D = 768, 256
    img, txt = _synth(B, D)
    img2, txt2 = _synth(B, D, 5)
    eng = _engine(B, D, 2)
    tp, bias = _scal(math.log(10.0)), _scal(-10.0)
    _, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, tp, bias)
    eng.forward(img, txt, tp, bias, True)
    g = _scal(-1.75)
    d2, t2, p2, b2 = eng.backward(img, txt, tp, g)
    torch.cuda.synchronize()
    _check("dimg * g", d2, dimg * -1.75, tol=1e-6)
    _check("dtxt * g", t2, dtxt * -1.75, tol=1e-6)
    _check("dt' * g", p2, float(dtp) * -1.75, tol=1e-6)
    _check("dbias * g", b2, float(db) * -1.75, tol=1e-6)
    eng.close()
    # an evaluation forward (no_grad) between forward and backward must not disturb the saved state
    e0 = _engine(B, D, 2)
    e0.forward(img, txt, tp, bias, True)
    e0.forward(img2, txt2, tp, bias, False)
    d3, t3, p3, b3 = e0.backward(img, txt, tp, None)
    torch.cuda.synchronize()
    _check("dimg after an interleaved eval forward", d3, dimg, tol=1e-6)
    _check("dt' after an interleaved eval forward", p3, float(dtp), tol=1e-6)
    _check("dbias after an interleaved eval forward", b3, float(db), tol=1e-6)
    e0.close()
    # two graphs on one module, backward in reverse order
    mod = DDPSigmoidLoss(B).to(_dev())
    a1, a2 = img.clone().requires_grad_(True), img2.clone().requires_grad_(True)
    l1 = mod(a1, txt)
    l2 = mod(a2, txt2)
    l1.backward()
    l2.backward()
    e1 = _engine(B, D, 2)
    _, r1, _, _, _ = e1.fwd_bwd(img, txt, _scal(float(mod.t_prime)), _scal(float(mod.bias)))
    _, r2, _, _, _ = e1.fwd_bwd(img2, txt2, _scal(float(mod.t_prime)), _scal(float(mod.bias)))
    torch.cuda.synchronize()
    _check("graph 1 dimg", a1.grad.float(), r1, tol=4e-3)
    _check("graph 2 dimg", a2.grad.float(), r2, tol=4e-3)
    e1.close()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_fused_l2_normalisation(dtype):
    """normalize_inputs=True: raw encoder outputs in, F.normalize + loss + both backwards fused. Oracle: torch autograd
    of F.normalize -> fp32 loss (bf16 leaves: with the straight-through bf16 rounding of the bf16 operand format)."""
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss

    B, D = 1024, 384
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(B, D, generator=g) * 3.0 + 0.2).to(dtype).to(_dev())
    y = (torch.randn(B, D, generator=g) * 0.5).to(dtype).to(_dev())
    mod = DDPSigmoidLoss(B, normalize_inputs=True).to(_dev())
    a, b = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
    loss = mod(a, b)
    loss.backward()

    def ref_side(v):
        v32 = v.detach().float().requires_grad_(True)
        n = torch.nn.functional.normalize(v32)
        if dtype == torch.bfloat16:
            n = n + (n.to(torch.bfloat16).float() - n).detach()  # rounding to bf16, gradient passes straight through
        # fp32 leaves: plain fp32 autograd, no rounding — the module feeds fp16(16 xhat) operands (11 bits)
        return v32, n

    a32, an = ref_side(x)
    b32, bn = ref_side(y)
    t = torch.tensor(float(mod.t_prime), device=_dev(), requires_grad=True)
    bb = torch.tensor(float(mod.bias), device=_dev(), requires_grad=True)
    z = an @ bn.T * t.exp() + bb
    ref = (-torch.nn.functional.logsigmoid((2 * torch.eye(B, device=_dev()) - 1) * z)).sum() / B
    ref.backward()
    torch.cuda.synchronize()
    tol = 1e-3 if dtype == torch.float32 else 4e-3      # bf16 leaves: the returned gradient is rounded to bf16
    _check("loss", loss.detach(), float(ref))
    # the projection (I - xhat xhat^T) cancels the radial part of the loss gradient: single elements of rows with a
    # small norm amplify the 1e-4 error of dxhat; the matrix-level error stays ~3e-5 (observed)
    _check("d raw img", a.grad.float(), a32.grad, tol=tol, max_tol=5e-3)
    _check("d raw txt", b.grad.float(), b32.grad, tol=tol, max_tol=5e-3)
    _check("dt_prime", mod.t_prime.grad, float(t.grad))
    _check("dbias", mod.bias.grad, float(bb.grad))


def test_kernel_launch_accounting():
    B, D = 512, 128
    img, txt = _synth(B, D)
    eng = _engine(B, D, 2)
    from distributed_sigmoid_loss_b200 import _capi

    eng.set_option(_capi.SIGLIP_OPT_KERNEL_TIMING, 1)
    n0 = eng.launch_count
    eng.fwd_bwd(img, txt, _scal(1.0), _scal(-5.0))
    assert eng.launch_count - n0 == 2          # loss kernel (its last CTA finalises) | gradient kernel (+ scalar grads)
    lm, ln, gm, gn = eng.kernel_times()
    assert ln == 1 and gn == 1 and lm > 0 and gm > 0
    eng.close()
    # a 3-chunk step (loopback): 3 loss + 3 gradient launches; with the helper-launch variant 11 more
    # (wait, copy is a memcpy, signal | signal | wait | 2 signals | signal: wait x2 + signal x5 kernels)
    e3 = _engine(B, D, 2, rank_world=(0, 3), loopback=True)
    for k in range(3):
        e3.debug_set_text_chunk(k, txt)
    e3.fwd_bwd(img, txt, _scal(1.0), _scal(-5.0))
    n0 = e3.launch_count
    e3.fwd_bwd(img, txt, _scal(1.0), _scal(-5.0))
    assert e3.launch_count - n0 == 6
    e3.set_option(_capi.SIGLIP_OPT_INKERNEL_SYNC, 0)
    n0 = e3.launch_count
    e3.fwd_bwd(img, txt, _scal(1.0), _scal(-5.0))
    assert e3.launch_count - n0 == 6 + 7
    torch.cuda.synchronize()
    e3.close()


def test_scalar_gradient_mean_option_loopback():
    """SIGLIP_OPT_SYNC_SCALAR_GRADS on a loopback context: the one-warp exchange runs its full signal / wait / gather
    protocol; the "peers'" mailboxes are seeded with DISTINCT values the kernel did not produce (debug hook), so the
    mean it returns is checked against (own + seeded values) / W in rank order — a skipped peer, a wrong peer or a wrong
    divisor fails (test_distributed_sigmoid_loss.py:79-83 semantics: all_reduce SUM, then / size)."""
    from distributed_sigmoid_loss_b200 import _capi
    B, D, W = 256, 128, 4
    me = 1
    img, txt = _synth(B, D, seed=5)
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    eng = _engine(B, D, 2, rank_world=(me, W), loopback=True)
    for k in range(W):
        eng.debug_set_text_chunk(k, _synth(B, D, seed=20 + k)[1])
    _, _, _, dtp0, db0 = eng.fwd_bwd(img, txt, tp, b)
    torch.cuda.synchronize()
    seeded = {0: (0.37, -1.25), 2: (-4.5, 0.03125), 3: (11.0, 2.75)}
    for p, (a_, b_) in seeded.items():
        eng.debug_set_mailbox(p, a_, b_)
    eng.set_option(_capi.SIGLIP_OPT_SYNC_SCALAR_GRADS, 1)

    def expect(own, idx):
        acc = np.float32(0.0)
        for p in range(W):       # the kernel adds the W mailboxes in rank order in fp32
            acc = np.float32(acc + (np.float32(own) if p == me else np.float32(seeded[p][idx])))
        return float(np.float32(acc * np.float32(1.0 / W)))
    for rep in range(3):
        for fused in (True, False):
            if fused:
                _, _, _, dtp1, db1 = eng.fwd_bwd(img, txt, tp, b)
            else:
                eng.forward(img, txt, tp, b, True)
                _, _, dtp1, db1 = eng.backward(img, txt, tp, None)
            torch.cuda.synchronize()
            assert float(dtp1) == expect(float(dtp0), 0), (float(dtp1), expect(float(dtp0), 0))
            assert float(db1) == expect(float(db0), 1), (float(db1), expect(float(db0), 1))
    # a different seed for ONE peer must move the result (that peer is really read)
    eng.debug_set_mailbox(3, 12.0, 2.75)
    _, _, _, dtp2, _ = eng.fwd_bwd(img, txt, tp, b)
    torch.cuda.synchronize()
    assert abs(float(dtp2) - float(dtp1) - 0.25) < 1e-5
    eng.close()


@pytest.mark.parametrize("name", ["w4_b8_d64", "w5_b4_d32", "w4_b40_d1152", "w8_b12_d1152_warm"])
def test_bidirectional_order_matches_reference_fixture(name):
    """SIGLIP_OPT_BIDIR (chunks visited right, left, right+1, ... like rwightman_sigmoid_loss.py:75-107): same pairs,
    so the loopback replay of every rank must reproduce the reference's bidirectional-variant outputs."""
    from distributed_sigmoid_loss_b200 import _capi
    if name not in golden_cases():
        pytest.skip("fixture not present")
    c = load_golden(name)
    W, B, D = c["world"], c["batch"], c["dim"]
    variant = "rw_bidir" if "rw_bidir" in c["variants"] else "ddp"
    dtxt_sum = [torch.zeros(B, D, device=_dev()) for _ in range(W)]
    for r in range(W):
        eng = _engine(B, D, 2, rank_world=(r, W), loopback=True)
        eng.set_option(_capi.SIGLIP_OPT_BIDIR, 1)
        for k in range(W):
            eng.debug_set_text_chunk(k, _golden_rank_inputs(c, k)[1])
        img, txt = _golden_rank_inputs(c, r)
        loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, _scal(c["t_prime"]), _scal(c["bias"]))
        torch.cuda.synchronize()
        ref = c["variants"][variant][r]
        _check(f"loss r{r}", loss, ref["loss"])
        _check(f"dimg r{r}", dimg, ref["dimg"])
        _check(f"dt_prime r{r}", dtp, ref["dt_prime"])
        _check(f"dbias r{r}", db, ref["dbias"])
        for k in range(W):
            dtxt_sum[k] += _contribution(eng, k, dtxt)
        torch.cuda.synchronize()
        eng.close()
    for k in range(W):
        _check(f"dtxt owner {k}", dtxt_sum[k], c["variants"][variant][k]["dtxt"])


# ---------------------------------------------------------------------------------------------------------
# fp32 callers (the reference's own test feeds fp32, test_distributed_sigmoid_loss.py:57-68): fixtures generated from
# RAW fp32 inputs; the module converts them to fp16(16 x) operands (11 significant bits) instead of bf16
# ---------------------------------------------------------------------------------------------------------
def _raw_rank_inputs(c, r):
    B = c["batch"]
    img = torch.from_numpy(c["img_all"][r * B:(r + 1) * B]).to(_dev()).contiguous()
    txt = torch.from_numpy(c["txt_all"][r * B:(r + 1) * B]).to(_dev()).contiguous()
    return img, txt


@pytest.mark.parametrize("cg", [1, 2])
def test_fp32_inputs_single_rank_match_raw_fp32_fixture(cg):
    c = load_golden("w1_b300_d136_f32")
    img, txt = _raw_rank_inputs(c, 0)
    assert not torch.equal(img.to(torch.bfloat16).float(), img)      # genuinely not bf16-representable
    eng = _engine(c["batch"], c["dim"], cg)
    ih, th = eng.convert_f32(img, True), eng.convert_f32(txt, True)
    assert ih.dtype == torch.float16 and float((ih.float() / 16 - img).abs().max()) <= 2.0 ** -11
    loss, dimg, dtxt, dtp, db = eng.fwd_bwd(ih, th, _scal(c["t_prime"]), _scal(c["bias"]))
    loss_f = eng.fwd(ih, th, _scal(c["t_prime"]), _scal(c["bias"]))
    torch.cuda.synchronize()
    ref = c["variants"]["ddp"][0]
    _check("loss", loss, ref["loss"])
    _check("loss (forward only)", loss_f, ref["loss"])
    _check("dimg", dimg, ref["dimg"])
    _check("dtxt", dtxt, ref["dtxt"])
    _check("dt_prime", dtp, ref["dt_prime"])
    _check("dbias", db, ref["dbias"])
    # the same engine still serves bf16 operands afterwards (the option follows the dtype)
    cb = load_golden("w1_b300_d136")
    ib, tb = _golden_rank_inputs(cb, 0)
    loss_b, dimg_b, _, _, _ = eng.fwd_bwd(ib, tb, _scal(cb["t_prime"]), _scal(cb["bias"]))
    torch.cuda.synchronize()
    _check("bf16 loss after fp16 use", loss_b, cb["variants"]["ddp"][0]["loss"])
    _check("bf16 dimg after fp16 use", dimg_b, cb["variants"]["ddp"][0]["dimg"])
    eng.close()


def test_fp32_inputs_through_the_module_beat_bf16_rounding():
    """DDPSigmoidLoss on fp32 tensors: fp32 gradients within 1e-3 of the reference run on the SAME raw fp32 inputs
    (rounding them to bf16 first costs 1.7e-3 — measured here too, as the reason for the format)."""
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss
    c = load_golden("w1_b300_d136_f32")
    img, txt = _raw_rank_inputs(c, 0)
    ref = c["variants"]["ddp"][0]
    mod = DDPSigmoidLoss(c["batch"]).to(_dev())
    a, b = img.clone().requires_grad_(True), txt.clone().requires_grad_(True)
    loss = mod(a, b)
    loss.backward()
    torch.cuda.synchronize()
    assert a.grad.dtype == torch.float32 and loss.dtype == torch.float32
    _check("loss", loss.detach(), ref["loss"])
    _check("dimg", a.grad, ref["dimg"])
    _check("dtxt", b.grad, ref["dtxt"])
    _check("dt_prime", mod.t_prime.grad, ref["dt_prime"])
    _check("dbias", mod.bias.grad, ref["dbias"])
    err_f16 = float((a.grad.cpu() - torch.from_numpy(ref["dimg"])).norm() / torch.from_numpy(ref["dimg"]).norm())
    # bf16-rounded inputs through the bf16 path, against the same raw-input reference
    eng = mod.engine_for(c["batch"], c["dim"], _dev())
    _, dimg_b, _, _, _ = eng.fwd_bwd(img.to(torch.bfloat16), txt.to(torch.bfloat16), _scal(c["t_prime"]),
                                     _scal(c["bias"]))
    err_bf16 = float((dimg_b.cpu() - torch.from_numpy(ref["dimg"])).norm() / torch.from_numpy(ref["dimg"]).norm())
    assert err_f16 < 5e-4 < err_bf16, (err_f16, err_bf16)
    # fused normalisation of raw fp32 encoder outputs takes the same 11-bit route
    raw_i, raw_t = (img * 3.0).clone().requires_grad_(True), (txt * 0.5).clone().requires_grad_(True)
    modn = DDPSigmoidLoss(c["batch"], normalize_inputs=True).to(_dev())
    ln = modn(raw_i, raw_t)
    ln.backward()
    torch.cuda.synchronize()
    _check("normalised loss", ln.detach(), ref["loss"])
    _check("normalised dimg (chain rule: / 3)", raw_i.grad * 3.0, ref["dimg"] - (ref["dimg"] * c["img_all"]).sum(1, keepdims=True) * c["img_all"], tol=2e-3, max_tol=5e-3)


@pytest.mark.parametrize("name", ["w2_b32_d512_f32", "w3_b40_d64_f32_warm"])
def test_fp32_inputs_multi_chunk_schedule_matches_raw_fp32_fixture(name):
    """BASELINE.json configs[0] (world 2, B=32/rank, D=512, fp32) with the reference's raw fp32 inputs: every rank
    replayed on one GPU (loopback), fp16(16 x) operands, text chunks exchanged in that format."""
    c = load_golden(name)
    W, B, D = c["world"], c["batch"], c["dim"]
    dtxt_sum = [torch.zeros(B, D, device=_dev()) for _ in range(W)]
    for r in range(W):
        eng = _engine(B, D, 2, rank_world=(r, W), loopback=True)
        for k in range(W):
            eng.debug_set_text_chunk(k, eng.convert_f32(_raw_rank_inputs(c, k)[1], True))
        img, txt = _raw_rank_inputs(c, r)
        ih, th = eng.convert_f32(img, True), eng.convert_f32(txt, True)
        loss, dimg, dtxt, dtp, db = eng.fwd_bwd(ih, th, _scal(c["t_prime"]), _scal(c["bias"]))
        torch.cuda.synchronize()
        ref = c["variants"]["ddp"][r]
        _check(f"loss r{r}", loss, ref["loss"])
        _check(f"dimg r{r}", dimg, ref["dimg"])
        _check(f"dt_prime r{r}", dtp, ref["dt_prime"])
        _check(f"dbias r{r}", db, ref["dbias"])
        for k in range(W):
            dtxt_sum[k] += _contribution(eng, k, dtxt)
        torch.cuda.synchronize()
        eng.close()
    for k in range(W):
        _check(f"dtxt owner {k}", dtxt_sum[k], c["variants"]["ddp"][k]["dtxt"])


@pytest.mark.parametrize("shape", [(1000, 136), (1024, 384), (2048, 1152), (4096, 768)])
@pytest.mark.parametrize("cg", [1, 2])
def test_gradient_column_tile_width_does_not_change_the_result(shape, cg):
    """SIGLIP_OPT_GRAD_TILE_N: 128-wide column tiles (chosen automatically when they fill the waves better, e.g.
    B=4096 D=768) accumulate every output element over k in the same order as 256-wide ones: bitwise equal gradients."""
    from distributed_sigmoid_loss_b200 import _capi
    B, D = shape
    img, txt = _synth(B, D, seed=11)
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    eng = _engine(B, D, cg)
    eng.set_option(_capi.SIGLIP_OPT_SPLIT_K, 0)     # split-K regroups the K sum per tile shape (tested separately)
    out = {}
    for tn in (256, 128, 0):
        eng.set_option(_capi.SIGLIP_OPT_GRAD_TILE_N, tn)
        _, dimg, dtxt, _, _ = eng.fwd_bwd(img, txt, tp, b)
        torch.cuda.synchronize()
        out[tn] = (dimg.clone(), dtxt.clone())
    assert torch.equal(out[128][0], out[256][0]) and torch.equal(out[128][1], out[256][1])
    assert torch.equal(out[0][0], out[256][0]) and torch.equal(out[0][1], out[256][1])
    eng.close()


# ---------------------------------------------------------------------------------------------------------
# the remaining BASELINE.json configs: configs[2] (B=8192/rank, D=768) and configs[4] (B=32768/rank, D=1152)
# ---------------------------------------------------------------------------------------------------------
def test_config2_shape_single_chunk_and_two_chunk_loopback():
    """BASELINE.json configs[2] per-rank shape (B=8192, D=768): one chunk against fp32 autograd, then rank 1 of a
    2-rank job (loopback): loss / dimg / scalars and both dtxt contributions against fp32 autograd of the 2-chunk loss."""
    from oracle.siglip_oracle import torch_reference_fp32

    B, D = 8192, 768
    tp, bias = math.log(10.0), -10.0
    img, txt = _synth(B, D)
    ref = torch_reference_fp32(img, [txt], tp, bias, 0)
    eng = _engine(B, D, 2)
    loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, _scal(tp), _scal(bias))
    torch.cuda.synchronize()
    _check("loss", loss, ref["loss"])
    _check("dimg", dimg, ref["dimg"])
    _check("dtxt", dtxt, ref["dtxt_chunks"][0])
    _check("dt_prime", dtp, ref["dt_prime"])
    _check("dbias", db, ref["dbias"])
    eng.close()
    del ref
    _, txt0 = _synth(B, D, 77)
    chunks = [txt0, txt]                       # rank 1 owns chunk 1
    ref = torch_reference_fp32(img, chunks, tp, bias, 1)
    eng = _engine(B, D, 2, rank_world=(1, 2), loopback=True)
    eng.debug_set_text_chunk(0, txt0)
    eng.debug_set_text_chunk(1, txt)
    loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, _scal(tp), _scal(bias))
    torch.cuda.synchronize()
    assert eng.workspace_bytes < 3 * 2 * B * B + (1 << 30)     # two sigma operands + O(B D) buffers
    _check("loss (2 chunks)", loss, ref["loss"])
    _check("dimg (2 chunks)", dimg, ref["dimg"])
    _check("dt_prime (2 chunks)", dtp, ref["dt_prime"])
    _check("dbias (2 chunks)", db, ref["dbias"])
    for k in range(2):
        _check(f"dtxt contribution to owner {k}", _contribution(eng, k, dtxt), ref["dtxt_chunks"][k])
    eng.close()


def test_config4_shape_single_chunk():
    """BASELINE.json configs[4] per-rank shape (B=32768, D=1152): one full chunk against fp32 autograd on the GPU
    (a 32768 x 32768 fp32 logits matrix is 4 GiB; autograd keeps a handful of them: fits the 80 GB), plus the
    size-independent identities."""
    from oracle.siglip_oracle import torch_reference_fp32

    B, D = 32768, 1152
    tp, bias = math.log(10.0), -10.0
    img, txt = _synth(B, D)
    eng = _engine(B, D, 2)
    loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, _scal(tp), _scal(bias))
    loss2, dimg2, dtxt2, dtp2, db2 = eng.fwd_bwd(img, txt, _scal(tp), _scal(bias))
    torch.cuda.synchronize()
    assert torch.equal(loss, loss2) and torch.equal(dimg, dimg2) and torch.equal(dtxt, dtxt2)
    s_img = float((dimg.double() * img.double()).sum())
    s_txt = float((dtxt.double() * txt.double()).sum())
    assert abs(s_img - float(dtp)) <= 1e-3 * abs(float(dtp)) and abs(s_txt - float(dtp)) <= 1e-3 * abs(float(dtp))
    eng.close()
    ref = torch_reference_fp32(img, [txt], tp, bias, 0)
    _check("loss", loss, ref["loss"])
    _check("dimg", dimg, ref["dimg"])
    _check("dtxt", dtxt, ref["dtxt_chunks"][0])
    _check("dt_prime", dtp, ref["dt_prime"])
    _check("dbias", db, ref["dbias"])


@pytest.mark.parametrize("name", ["w4_b40_d1152", "w8_b12_d1152_warm"])
def test_d1152_sweep_against_both_reference_variants(name):
    """configs[4] "parity sweep vs rwightman_sigmoid_loss.py": D = 1152 fixtures produced by the unmodified reference's
    DDPSigmoidLoss AND SigLipLoss (uni- and bidirectional ring, rwightman_sigmoid_loss.py:68-124); every rank of the
    W = 4 / 8 job replayed on one GPU in the unidirectional order (the bidirectional order is the test above)."""
    c = load_golden(name)
    W, B, D = c["world"], c["batch"], c["dim"]
    dtxt_sum = [torch.zeros(B, D, device=_dev()) for _ in range(W)]
    for r in range(W):
        eng = _engine(B, D, 2, rank_world=(r, W), loopback=True)
        for k in range(W):
            eng.debug_set_text_chunk(k, _golden_rank_inputs(c, k)[1])
        img, txt = _golden_rank_inputs(c, r)
        loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, _scal(c["t_prime"]), _scal(c["bias"]))
        torch.cuda.synchronize()
        for variant in ("ddp", "rw_uni", "rw_bidir"):
            ref = c["variants"][variant][r]
            _check(f"{variant} loss r{r}", loss, ref["loss"])
            _check(f"{variant} dimg r{r}", dimg, ref["dimg"])
            _check(f"{variant} dt_prime r{r}", dtp, ref["dt_prime"])
            _check(f"{variant} dbias r{r}", db, ref["dbias"])
        for k in range(W):
            dtxt_sum[k] += _contribution(eng, k, dtxt)
        torch.cuda.synchronize()
        eng.close()
    for k in range(W):
        for variant in ("ddp", "rw_uni", "rw_bidir"):
            _check(f"{variant} dtxt owner {k}", dtxt_sum[k], c["variants"][variant][k]["dtxt"])


# ---------------------------------------------------------------------------------------------------------
# SURVEY.md §8(f)4: uneven per-rank batch
# ---------------------------------------------------------------------------------------------------------
def test_uneven_per_rank_batches_loopback():
    """Ranks with B = (40, 24, 33) (siglip_ctx_create_uneven): every rank replayed on one GPU; per-rank loss / dimg /
    scalars and the per-owner dtxt sums against the float64 closed form."""
    Bs, D = (40, 24, 33), 72
    W = len(Bs)
    tp, bias = math.log(10.0), -8.0
    g = torch.Generator().manual_seed(31)
    imgs = [torch.nn.functional.normalize(torch.randn(b, D, generator=g)).to(torch.bfloat16) for b in Bs]
    txts = [torch.nn.functional.normalize(torch.randn(b, D, generator=g)).to(torch.bfloat16) for b in Bs]
    from oracle.siglip_oracle import closed_form_uneven
    ref = closed_form_uneven([x.float().numpy() for x in imgs], [x.float().numpy() for x in txts], tp, bias)
    for sched in ("fused", "split"):
        dtxt_sum = [torch.zeros(b, D, device=_dev()) for b in Bs]
        for r in range(W):
            eng = _engine(Bs[r], D, 2, rank_world=(r, W), loopback=True, batch_per_rank=Bs)
            for k in range(W):
                eng.debug_set_text_chunk(k, txts[k].to(_dev()))
            img, txt = imgs[r].to(_dev()), txts[r].to(_dev())
            if sched == "fused":
                loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, _scal(tp), _scal(bias))
            else:
                loss = eng.forward(img, txt, _scal(tp), _scal(bias), True)
                dimg, dtxt, dtp, db = eng.backward(img, txt, _scal(tp), None)
            torch.cuda.synchronize()
            _check(f"{sched} loss r{r}", loss, ref[r]["loss"])
            _check(f"{sched} dimg r{r}", dimg, ref[r]["dimg"])
            _check(f"{sched} dt_prime r{r}", dtp, ref[r]["dt_prime"])
            _check(f"{sched} dbias r{r}", db, ref[r]["dbias"])
            for k in range(W):
                got = _contribution(eng, k, dtxt)
                assert tuple(got.shape) == (Bs[k], D)
                _check(f"{sched} contribution r{r} -> owner {k}", got, ref[r]["contrib"][k])
                dtxt_sum[k] += got
            eng.close()
        for k in range(W):
            _check(f"{sched} dtxt owner {k}", dtxt_sum[k], sum(ref[r]["contrib"][k] for r in range(W)))
    with pytest.raises(RuntimeError):
        _engine(40, D, 2, rank_world=(1, W), loopback=True, batch_per_rank=Bs)    # rank 1's batch is 24, not 40


# ---------------------------------------------------------------------------------------------------------
# module surface: fused schedule, odd embedding widths, views, siglip_scale on any size
# ---------------------------------------------------------------------------------------------------------
def test_module_fused_schedule_equals_split_schedule():
    """DDPSigmoidLoss(fused_step=True) (what a multi-rank group uses by default) against fused_step=False: the fused
    step leaves gradients for an upstream gradient of 1 and backward() multiplies by grad_output — same numbers up to
    the order of the two roundings (fp32 result x g, then bf16)."""
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss
    B, D = 640, 192
    img, txt = _synth(B, D, seed=9)
    outs = []
    for fused in (False, True):
        mod = DDPSigmoidLoss(B, fused_step=fused).to(_dev())
        a, b = img.clone().requires_grad_(True), txt.clone().requires_grad_(True)
        loss = mod(a, b)
        (0.5 * loss).backward()
        torch.cuda.synchronize()
        outs.append((loss.detach(), a.grad, b.grad, mod.t_prime.grad, mod.bias.grad))
    assert torch.equal(outs[0][0], outs[1][0])
    _check("dimg", outs[1][1].float(), outs[0][1].float(), tol=4e-3)
    _check("dtxt", outs[1][2].float(), outs[0][2].float(), tol=4e-3)
    _check("dt_prime", outs[1][3], float(outs[0][3]), tol=1e-6)
    _check("dbias", outs[1][4], float(outs[0][4]), tol=1e-6)
    # fp32 leaves take the fp32-gradient route in both schedules: equal to 1e-6
    g32 = []
    for fused in (False, True):
        mod = DDPSigmoidLoss(B, fused_step=fused).to(_dev())
        a = img.float().requires_grad_(True)
        mod(a, txt.float()).backward()
        torch.cuda.synchronize()
        g32.append(a.grad)
    _check("fp32 dimg", g32[1], g32[0], tol=1e-6)


def test_module_accepts_any_embedding_width_and_views():
    """The reference's own test uses output_dim = 2 (test_distributed_sigmoid_loss.py:144): widths that are not a
    multiple of 8 are zero-padded (zero columns change no dot product) and the gradient comes back sliced;
    non-contiguous and 16-byte-misaligned views are copied instead of rejected."""
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss
    from oracle.siglip_oracle import torch_reference_fp32
    B = 96
    for D in (2, 20, 515):
        g = torch.Generator().manual_seed(D)
        img = torch.nn.functional.normalize(torch.randn(B, D, generator=g)).to(_dev())
        txt = torch.nn.functional.normalize(torch.randn(B, D, generator=g)).to(_dev())
        ref = torch_reference_fp32(img, [txt], math.log(10.0), -10.0, 0)
        mod = DDPSigmoidLoss(B).to(_dev())
        a, b = img.clone().requires_grad_(True), txt.clone().requires_grad_(True)
        loss = mod(a, b)
        loss.backward()
        torch.cuda.synchronize()
        assert a.grad.shape == (B, D) and b.grad.shape == (B, D)
        # fp32 leaves -> fp16(16 x) operands (11 significant bits); at D = 2 nothing averages the rounding of a single
        # operand element, so the element-wise bound is looser than the matrix-level one
        _check(f"D={D} loss", loss.detach(), ref["loss"])
        _check(f"D={D} dimg", a.grad, ref["dimg"], max_tol=4e-3)
        _check(f"D={D} dtxt", b.grad, ref["dtxt_chunks"][0], max_tol=4e-3)
    # a misaligned, strided view of a larger bf16 buffer
    D = 64
    big = torch.nn.functional.normalize(torch.randn(B, 2 * D + 3, device=_dev())).to(torch.bfloat16)
    view = big[:, 3:3 + D]
    assert view.data_ptr() % 16 != 0 and not view.is_contiguous()
    txt = _synth(B, D, 3)[1]
    mod = DDPSigmoidLoss(B).to(_dev())
    l_view = mod(view, txt)
    l_copy = mod(view.clone(), txt)
    torch.cuda.synchronize()
    assert torch.equal(l_view, l_copy)


def test_scale_any_size_and_alignment():
    eng = _engine(256, 64, 2)
    g = _scal(-0.75)
    for n in (1, 7, 8, 1000, 4099):
        for dt in (torch.float32, torch.bfloat16):
            x = torch.randn(n + 3, device=_dev()).to(dt)
            for off in (0, 1, 3):
                v = x[off:off + n]
                want = (v.float() * -0.75).to(dt)
                assert torch.equal(eng.scale(v, g), want), (n, dt, off)
    with pytest.raises(RuntimeError):
        eng.scale(torch.zeros(4, device=_dev(), dtype=torch.float16), g)
    eng.close()


def test_host_entry_returns_bf16_gradients():
    """siglip_host_submit_grads: the bf16 gradients of every pipelined step arrive in the caller's host buffers and equal
    the device entry's bf16 gradients bit for bit."""
    B, D = 1024, 256
    eng = _engine(B, D, 2)
    want, tickets = [], []
    hosts = []
    for i in range(4):
        img, txt = _synth(B, D, seed=500 + i)
        tp, bias = math.log(10.0) + 0.1 * i, -10.0 + i
        loss, dimg, dtxt, _, _ = eng.fwd_bwd(img, txt, _scal(tp), _scal(bias), torch.bfloat16)
        torch.cuda.synchronize()
        want.append((float(loss), dimg.cpu(), dtxt.cpu()))
        hosts.append((img.cpu().pin_memory(), txt.cpu().pin_memory(), tp, bias,
                      torch.empty(B, D, dtype=torch.bfloat16).pin_memory(),
                      torch.empty(B, D, dtype=torch.bfloat16).pin_memory()))
    prev = None
    got = []
    for (ih, th, tp, bias, gi, gt) in hosts:
        t = eng.host_submit(ih, th, tp, bias, gi, gt)
        if prev is not None:
            got.append(eng.host_wait(prev))
        prev = t
    got.append(eng.host_wait(prev))
    for i in range(4):
        assert got[i][0] == want[i][0]
        assert torch.equal(hosts[i][4], want[i][1]) and torch.equal(hosts[i][5], want[i][2])
    with pytest.raises(RuntimeError):
        eng.host_submit(hosts[0][0], hosts[0][1], 1.0, 1.0, hosts[0][4], None)
    eng.close()


def test_peer_timeout_option_and_trace_hook():
    from distributed_sigmoid_loss_b200 import _capi
    B, D = 256, 64
    img, txt = _synth(B, D)
    eng = _engine(B, D, 2, rank_world=(0, 2), loopback=True)
    eng.set_option(_capi.SIGLIP_OPT_PEER_TIMEOUT_MS, 5000)
    with pytest.raises(RuntimeError):
        eng.set_option(_capi.SIGLIP_OPT_PEER_TIMEOUT_MS, 0)
    eng.debug_set_text_chunk(0, txt)
    eng.debug_set_text_chunk(1, txt)
    eng.set_option(_capi.SIGLIP_OPT_AUX_TRACE, 1)
    eng.fwd_bwd(img, txt, _scal(1.0), _scal(-5.0))
    tr = eng.aux_trace()
    assert len(tr) == 4                       # L0 L1 G1 G0
    for (t0, tflag, tdone, tend, *_rest) in tr:
        assert t0 > 0 and tdone >= t0 and (tend == 0 or tend >= t0)
    eng.close()


# ---------------------------------------------------------------------------------------------------------
# split-K of the gradient kernel's ragged last wave; fp8 (wgmma e4m3) measurement path
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(4096, 768), (1000, 136), (2048, 1152), (520, 264), (8192, 768)])
@pytest.mark.parametrize("cg", [1, 2])
def test_split_k_is_deterministic_and_matches_unsplit(shape, cg):
    """SIGLIP_OPT_SPLIT_K: the tiles of a ragged last wave are cut into K-slices whose fp32 partial accumulators meet in
    a workspace and are added in slice order — bitwise repeatable, and equal to the unsplit result up to fp32
    summation order."""
    from distributed_sigmoid_loss_b200 import _capi
    B, D = shape
    img, txt = _synth(B, D, seed=13)
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    eng = _engine(B, D, cg)
    out = {}
    for sk in (0, -1, 2, 3):
        eng.set_option(_capi.SIGLIP_OPT_SPLIT_K, sk)
        runs = []
        for _ in range(2):
            _, dimg, dtxt, _, _ = eng.fwd_bwd(img, txt, tp, b)
            torch.cuda.synchronize()
            runs.append((dimg.clone(), dtxt.clone()))
        assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
        out[sk] = runs[0]
    for sk in (-1, 2, 3):
        _check(f"dimg split {sk}", out[sk][0], out[0][0], tol=2e-6)
        _check(f"dtxt split {sk}", out[sk][1], out[0][1], tol=2e-6)
    with pytest.raises(RuntimeError):
        eng.set_option(_capi.SIGLIP_OPT_SPLIT_K, 1)
    eng.close()


@pytest.mark.parametrize("cg", [1, 2])
def test_fp8_measurement_path_computes_the_e4m3_product(cg, monkeypatch):
    """siglip_debug_gemm under SIGLIP_DEBUG_AB_FP8: e4m3 x e4m3 -> fp32 on the same mainloop (wgmma e4m3, each
    instruction's result summed in fp32). Products of e4m3 values are exact in fp32, so the result equals the fp32
    product of the dequantised operands."""
    from distributed_sigmoid_loss_b200 import _capi
    L = _capi.lib()
    monkeypatch.setenv("SIGLIP_DEBUG_AB_FP8", "1")
    monkeypatch.delenv("SIGLIP_DEBUG_AB_F16", raising=False)
    monkeypatch.delenv("SIGLIP_DEBUG_MCAST", raising=False)
    torch.manual_seed(2)
    for (M, N, K) in [(256, 256, 128), (512, 768, 1024), (300, 264, 400)]:
        A = torch.randn(M, K, device=_dev()).to(torch.float8_e4m3fn)
        Bm = torch.randn(N, K, device=_dev()).to(torch.float8_e4m3fn)
        ld = (K + 15) // 16 * 16
        Ab = torch.zeros(M, ld, device=_dev(), dtype=torch.uint8)
        Bb = torch.zeros(N, ld, device=_dev(), dtype=torch.uint8)
        Ab[:, :K] = A.view(torch.uint8)
        Bb[:, :K] = Bm.view(torch.uint8)
        C = torch.full((M, N), float("nan"), device=_dev())
        rc = L.siglip_debug_gemm(0, cg, M, N, K, Ab.data_ptr(), ld, 0, Bb.data_ptr(), ld, 0, C.data_ptr(), N,
                                 torch.cuda.current_stream().cuda_stream)
        assert rc == 0, _capi.last_error()
        torch.cuda.synchronize()
        ref = A.float() @ Bm.float().T
        assert float((C - ref).abs().max()) <= 1e-5 * float(ref.abs().max()) * math.sqrt(K) + 1e-4


def test_programmatic_dependent_launch_changes_nothing_but_timing():
    """SIGLIP_OPT_PDL: the kernels' set-up may overlap the previous kernel's tail; every global access stays ordered
    behind it (griddepcontrol.wait), so results are bitwise those of plain launches — also back to back on one stream
    with a multi-chunk loopback schedule, where consecutive launches hand sigma operands and flags to each other."""
    from distributed_sigmoid_loss_b200 import _capi
    B, D, W = 1024, 256, 3
    img, txt = _synth(B, D, seed=21)
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    outs = {}
    for pdl in (0, 1):
        eng = _engine(B, D, 2, rank_world=(1, W), loopback=True)
        eng.set_option(_capi.SIGLIP_OPT_PDL, pdl)
        for k in range(W):
            eng.debug_set_text_chunk(k, _synth(B, D, seed=40 + k)[1])
        res = None
        for _ in range(6):          # back-to-back steps: no host synchronisation between the launches
            res = eng.fwd_bwd(img, txt, tp, b)
        torch.cuda.synchronize()
        outs[pdl] = [x.clone() for x in res] + [eng.debug_get_slot(0).clone(), eng.debug_get_slot(2).clone()]
        eng.close()
    for x, y in zip(outs[0], outs[1]):
        assert torch.equal(x, y)


def test_t_prime_is_taken_in_the_references_own_dtype():
    """The reference's t_prime is a float64 parameter (torch.tensor(np.log(10)), distributed_sigmoid_loss.py:11): the C ABI
    reads it (and writes dt_prime) as fp64 under SIGLIP_OPT_TPRIME_F64, which the engine sets from the tensor's dtype —
    no conversion kernels around the step. Same numbers as the fp32 hand-over (exp is evaluated in fp32 either way)."""
    B, D = 768, 128
    img, txt = _synth(B, D, seed=17)
    eng = _engine(B, D, 2)
    tp32, b = _scal(math.log(10.0)), _scal(-10.0)
    tp64 = torch.tensor([math.log(10.0)], device=_dev(), dtype=torch.float64)
    r32 = eng.fwd_bwd(img, txt, tp32, b)
    r64 = eng.fwd_bwd(img, txt, tp64, b)
    l64 = eng.forward(img, txt, tp64, b, True)
    d64 = eng.backward(img, txt, tp64, _scal(2.0))
    r32b = eng.fwd_bwd(img, txt, tp32, b)             # and back
    torch.cuda.synchronize()
    assert r64[3].dtype == torch.float64 and d64[2].dtype == torch.float64 and r32[3].dtype == torch.float32
    assert torch.equal(r32[0], r64[0]) and torch.equal(r32[1], r64[1]) and torch.equal(r32[2], r64[2])
    assert float(r64[3]) == float(r32[3]) and torch.equal(r32[4], r64[4]) and torch.equal(l64, r32[0])
    assert abs(float(d64[2]) - 2.0 * float(r32[3])) <= 1e-6 * abs(float(r32[3]))
    assert torch.equal(r32b[1], r32[1]) and torch.equal(r32b[3], r32[3])
    eng.close()


def test_fused_step_is_cuda_graph_capturable():
    """The fused single-rank step is two stream-ordered launches with no host synchronisation, no allocation after the
    first call and kernel parameters passed by value (tensor maps are __grid_constant__): it can be captured into a CUDA
    graph and replayed; replays reproduce the eager results bit for bit and follow the inputs' CONTENT (same buffers)."""
    B, D = 1024, 256
    eng = _engine(B, D, 2)
    img, txt = _synth(B, D, seed=31)
    img2, txt2 = _synth(B, D, seed=32)
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    eager1 = [x.clone() for x in eng.fwd_bwd(img, txt, tp, b, torch.bfloat16)]
    eager2 = [x.clone() for x in eng.fwd_bwd(img2, txt2, tp, b, torch.bfloat16)]
    si, st_ = img.clone(), txt.clone()                  # static input buffers of the graph
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        eng.fwd_bwd(si, st_, tp, b, torch.bfloat16)      # warm-up on the capture stream
        with torch.cuda.graph(g, stream=side):
            outs = eng.fwd_bwd(si, st_, tp, b, torch.bfloat16)
    torch.cuda.current_stream().wait_stream(side)
    g.replay()
    torch.cuda.synchronize()
    for a, e in zip(outs, eager1):
        assert torch.equal(a, e)
    si.copy_(img2)
    st_.copy_(txt2)
    g.replay()
    g.replay()
    torch.cuda.synchronize()
    for a, e in zip(outs, eager2):
        assert torch.equal(a, e)
    del g
    eng.close()


def test_fused_schedule_composes_with_normalisation_and_the_siglip_adapter():
    """The fused schedule (default on multi-rank groups) through the two other module surfaces: fused L2 normalisation
    (fp32 gradients of the normalised embeddings, then the projection) and the open_clip-signature adapter — same
    numbers as the split schedule."""
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss
    B, D = 512, 192
    g = torch.Generator().manual_seed(8)
    x = (torch.randn(B, D, generator=g) * 2.0 + 0.1).to(_dev())
    y = (torch.randn(B, D, generator=g) * 0.7).to(_dev())
    res = []
    for fused in (False, True):
        mod = DDPSigmoidLoss(B, normalize_inputs=True, fused_step=fused).to(_dev())
        a, b = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
        loss = mod(a, b)
        (3.0 * loss).backward()
        torch.cuda.synchronize()
        res.append((loss.detach(), a.grad, b.grad, mod.t_prime.grad.clone(), mod.bias.grad.clone()))
    assert torch.equal(res[0][0], res[1][0])
    _check("d raw img", res[1][1], res[0][1], tol=1e-5)
    _check("d raw txt", res[1][2], res[0][2], tol=1e-5)
    _check("dt_prime", res[1][3], float(res[0][3]), tol=1e-6)
    _check("dbias", res[1][4], float(res[0][4]), tol=1e-6)
    img, txt = _synth(B, D, seed=12)
    out = []
    for fused in (False, True):
        scale = torch.nn.Parameter(torch.tensor(math.log(10.0), device=_dev()))
        lbias = torch.nn.Parameter(torch.tensor(-10.0, device=_dev()))
        a = img.clone().requires_grad_(True)
        l = SigLipLoss(rank=0, world_size=1, fused_step=fused)(a, txt, scale, lbias)
        l.backward()
        torch.cuda.synchronize()
        out.append((l.detach(), a.grad, scale.grad.clone(), lbias.grad.clone()))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])
    _check("dscale", out[1][2], float(out[0][2]), tol=1e-6)
    _check("dbias", out[1][3], float(out[0][3]), tol=1e-6)


def test_multi_rank_step_refuses_graph_capture():
    B, D = 256, 64
    img, txt = _synth(B, D)
    eng = _engine(B, D, 2, rank_world=(0, 2), loopback=True)
    eng.debug_set_text_chunk(0, txt)
    eng.debug_set_text_chunk(1, txt)
    tp, b = _scal(1.0), _scal(-5.0)
    eng.fwd_bwd(img, txt, tp, b)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    raised = False
    with torch.cuda.stream(side):
        try:
            with torch.cuda.graph(g, stream=side):
                try:
                    eng.fwd_bwd(img, txt, tp, b)
                except RuntimeError as ex:
                    raised = "cannot be captured" in str(ex)
        except Exception:       # an empty / aborted capture may itself complain: irrelevant here
            pass
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    assert raised
    eng.fwd_bwd(img, txt, tp, b)                          # the context is still usable
    torch.cuda.synchronize()
    eng.close()
