"""NaN and +-inf in embeddings and scalars on the H100, against float64 autograd of ``exclude_groups_oracle.torch_loss``
on the operand values the kernels consume (``operand_values``: bf16 as it is, fp32 / fp16 through fp16(16 x) / 16 for
finite entries, non-finite entries kept). The contract, element by element: every output (loss, dimg, dtxt or a peer's
contribution slot, dt', dbias) is non-finite exactly where the reference is (NaN and inf are not told apart: the
compensated sums turn +inf into NaN through inf - inf); where the reference is finite the kernel is within 1e-3 of it;
per-sample losses are exactly +inf for a +inf or >= 2^16 partial, NaN for a NaN partial and the oracle's value elsewhere
(``sample_loss_classes``). Covered: one bad entry or a whole NaN row in a paired image, the own paired text, a hard
negative, an extra image and a peer's chunk (loopback W = 3); bf16 and SIGLIP_OPT_INPUT_F16 engines; fused, split and
forward-only steps and row panels; NaN / infinite t' and NaN bias; an fp32 teacher under distillation; the modules with
bf16, fp32 and fp16 inputs and normalize_inputs; per-sample-loss overflow and poison words seeded for loopback peers;
the fp32 conversion bit for bit at edge values; metrics and top-K on a NaN step; GradScaler skipping the step of fp16
towers that overflow under autocast; zero rows (finite and degenerate)."""
import math

import numpy as np
import pytest
import torch

from exclude_groups_oracle import operand_values, sample_loss_classes, torch_loss, torch_terms
from retrieval_topk_oracle import topk_retrieval

pytestmark = pytest.mark.gpu

TOL = 1e-3
TP, BIAS = math.log(10.0), -10.0
B1, K1, E1, D1 = 300, 23, 17, 136     # one rank: paired batch, hard negatives, extra images
B3, W3, R3 = 136, 3, 1                # loopback: batch, world, own rank
NAN, INF = float("nan"), float("inf")
VALUES = ["nan", "inf", "-inf", "nan_row"]


def _dev():
    return torch.device("cuda", 0)


def _scal(x):
    return torch.tensor([x], device=_dev(), dtype=torch.float32)


def _rel(a, b):
    a, b = a.double().cpu().reshape(-1), b.double().cpu().reshape(-1)
    return max(float((a - b).norm() / (b.norm() + 1e-300)), float((a - b).abs().max() / (b.abs().max() + 1e-300)))


def _contract(name, got, ref, tol=TOL):
    """Non-finite exactly where the reference is; within tol of it over the finite elements."""
    got = torch.as_tensor(got).double().cpu().reshape(-1)
    ref = torch.as_tensor(ref).double().cpu().reshape(-1)
    assert got.shape == ref.shape, f"{name}: shape {tuple(got.shape)} != {tuple(ref.shape)}"
    gb, rb = ~torch.isfinite(got), ~torch.isfinite(ref)
    extra, missing = int((gb & ~rb).sum()), int((rb & ~gb).sum())
    assert extra == 0 and missing == 0, (f"{name}: {extra} elements non-finite where the reference is finite, "
                                         f"{missing} finite where it is not (of {ref.numel()}, {int(rb.sum())} "
                                         f"non-finite in the reference)")
    if bool((~rb).any()):
        err = _rel(got[~rb], ref[~rb])
        assert err <= tol, f"{name}: relative error {err:.3e} over the finite elements"


def _classes(name, got, want, tol=TOL):
    """Per-sample losses: NaN, +inf and finite exactly as the oracle's classes, finite values within tol."""
    got = got.double().cpu()
    want = torch.as_tensor(want).double()
    assert torch.equal(torch.isnan(got), torch.isnan(want)), f"{name}: NaN at {torch.isnan(got).nonzero().flatten()[:8]}" \
        f" where the oracle has {torch.isnan(want).nonzero().flatten()[:8]}"
    assert torch.equal(got == INF, want == INF), f"{name}: +inf at {(got == INF).nonzero().flatten()[:8]} where the " \
        f"oracle has {(want == INF).nonzero().flatten()[:8]}"
    assert not bool((got == -INF).any()), f"{name}: -inf"
    fin = torch.isfinite(want)
    if bool(fin.any()):
        err = _rel(got[fin], want[fin])
        assert err <= tol, f"{name}: relative error {err:.3e} over the finite samples"


def _reference(img, txts, y, tp, bias, batch, normalize=False, teacher=None):
    """float64 autograd of torch_loss over the chunks side by side: loss, dimg, contrib[c], dtp, db and the pair terms."""
    xi = img.detach().double().cpu().requires_grad_(True)
    xt = torch.cat([t.detach().double().cpu() for t in txts]).requires_grad_(True)
    tpt = torch.tensor(float(tp), dtype=torch.float64, requires_grad=True)
    bt = torch.tensor(float(bias), dtype=torch.float64, requires_grad=True)
    loss = torch_loss(xi, xt, tpt, bt, y, normalize=normalize, batch=batch, teacher=teacher)
    loss.backward()
    terms = torch_terms(xi.detach(), xt.detach(), tpt.detach(), bt.detach(), y, normalize=normalize, teacher=teacher)
    return dict(loss=loss.detach(), dimg=xi.grad, contrib=list(torch.split(xt.grad, [t.shape[0] for t in txts])),
                dtp=tpt.grad, db=bt.grad, terms=terms.detach())


def _labels(R, B, Ts, own):
    """[R, sum T_c]: image i < B is positive with text i of the own chunk, every other pair negative."""
    y = -torch.ones(R, sum(Ts), dtype=torch.float64)
    off = sum(Ts[:own])
    y[torch.arange(B), off + torch.arange(B)] = 1.0
    return y


def _unit(g, n, D):
    return torch.nn.functional.normalize(torch.randn(n, D, generator=g))


def _spoil(x, row, value, col=9):
    """x with one entry (or the whole row, nan_row) of row `row` set to the value."""
    x = x.clone()
    if value == "nan_row":
        x[row] = NAN
    else:
        x[row, col] = {"nan": NAN, "inf": INF, "-inf": -INF}[value]
    return x


_ENGINES = {}


def _engine(kind):
    """Cached engines: "w1" one rank with hard negatives and extra images, "w3" rank 1 of a loopback W = 3 job, "panels"
    a one-rank engine whose sigma budget forces row panels."""
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine

    if kind not in _ENGINES:
        if kind == "w1":
            eng = SigmoidLossEngine(B1, D1, _dev(), texts_per_rank=[B1 + K1], images_per_rank=[B1 + E1])
        elif kind == "w3":
            eng = SigmoidLossEngine(B3, D1, _dev(), rank_world=(R3, W3), loopback=True)
        else:
            eng = SigmoidLossEngine(1000, D1, _dev())
            eng.set_sigma_budget(1 << 20)
            assert eng.sigma_panels()[1] > 1
        _ENGINES[kind] = eng
    return _ENGINES[kind]


def _operand(eng, x, f16):
    """The device operand of x (fp32 master values): bf16, or the fp32 conversion to fp16(16 x) (INPUT_F16)."""
    if f16:
        return eng.convert_f32(x.float().contiguous().to(_dev()), True)
    return x.to(torch.bfloat16).contiguous().to(_dev())


def _consumed(x, f16):
    return operand_values(x.float() if f16 else x.to(torch.bfloat16))


def _run(eng, img_op, txt_ops, tp, bias, sched, losses=False):
    """One step of the engine on device operands; returns its outputs by name (a peer chunk's contribution as slot<k>)."""
    r = eng.rank
    if eng.world > 1:
        for k in range(eng.world):
            eng.debug_set_text_chunk(k, txt_ops[k])
    out = {}
    if losses:
        out["image_loss"] = torch.full((eng.images,), -1.0, device=_dev())
        out["text_loss"] = torch.full((eng.texts,), -1.0, device=_dev())
        eng.request_sample_losses(out["image_loss"], out["text_loss"])
    tpt, bt = _scal(tp), _scal(bias)
    if sched == "fused":
        out["loss"], out["dimg"], out["dtxt"], out["dtp"], out["db"] = eng.fwd_bwd(img_op, txt_ops[r], tpt, bt)
    elif sched == "split":
        out["loss"] = eng.forward(img_op, txt_ops[r], tpt, bt, True)
        out["dimg"], out["dtxt"], out["dtp"], out["db"] = eng.backward(img_op, txt_ops[r], tpt, None)
    else:
        out["loss"] = eng.fwd(img_op, txt_ops[r], tpt, bt)
    if sched != "fwd":
        for k in range(eng.world):
            if k != r:
                out[f"slot{k}"] = eng.debug_get_slot(k)
    torch.cuda.synchronize()
    return {k: v.clone() for k, v in out.items()}


def _check_step(tag, eng, out, ref):
    _contract(f"{tag} loss", out["loss"], ref["loss"])
    if "dimg" not in out:
        return
    _contract(f"{tag} dimg", out["dimg"], ref["dimg"])
    _contract(f"{tag} dt'", out["dtp"], ref["dtp"])
    _contract(f"{tag} dbias", out["db"], ref["db"])
    for k in range(eng.world):
        got = out["dtxt"] if k == eng.rank else out[f"slot{k}"]
        _contract(f"{tag} contribution to chunk {k}", got, ref["contrib"][k])
    if "image_loss" in out:
        cls = sample_loss_classes(ref["terms"], [t.shape[0] for t in ref["contrib"]])
        _classes(f"{tag} image_loss", out["image_loss"], cls["image_loss"])
        if eng.world == 1:
            _classes(f"{tag} text_loss", out["text_loss"], cls["text_loss_part"])


def _problem(kind, seed):
    """fp32 master embeddings of the engine's rank: images [R, D] and the chunks' texts."""
    g = torch.Generator().manual_seed(seed)
    if kind == "w1":
        return _unit(g, B1 + E1, D1), [_unit(g, B1 + K1, D1)]
    return _unit(g, B3, D1), [_unit(g, B3, D1) for _ in range(W3)]


PLACES = {"image": ("w1", None, 7), "text": ("w1", 0, 11), "negative": ("w1", 0, B1 + 2),
          "extra_image": ("w1", None, B1 + 5), "peer": ("w3", (R3 + 1) % W3, 5)}


# ---------------------------------------------------------------------------------------------------------------------
# 1. the engine: where the value sits, bf16 and INPUT_F16, every schedule
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("f16", [False, True], ids=["bf16", "input_f16"])
@pytest.mark.parametrize("place", list(PLACES))
@pytest.mark.parametrize("value", VALUES)
def test_engine_non_finite_embedding(value, place, f16):
    kind, chunk, row = PLACES[place]
    eng = _engine(kind)
    img, txts = _problem(kind, seed=VALUES.index(value) + 7 * list(PLACES).index(place))
    if chunk is None:
        img = _spoil(img, row, value)
    else:
        txts[chunk] = _spoil(txts[chunk], row, value)
    img_op, txt_ops = _operand(eng, img, f16), [_operand(eng, t, f16) for t in txts]
    y = _labels(img.shape[0], eng.batch, [t.shape[0] for t in txts], eng.rank)
    ref = _reference(_consumed(img, f16), [_consumed(t, f16) for t in txts], y, TP, BIAS, eng.batch)
    assert not bool(torch.isfinite(ref["loss"]))   # the case has something to get wrong
    for sched in ("fused", "split", "fwd"):
        out = _run(eng, img_op, txt_ops, TP, BIAS, sched, losses=(sched == "fused"))
        _check_step(f"{value} in {place} {'f16' if f16 else 'bf16'} {sched}", eng, out, ref)


@pytest.mark.parametrize("f16", [False, True], ids=["bf16", "input_f16"])
@pytest.mark.parametrize("tp,bias", [(NAN, BIAS), (1000.0, BIAS), (TP, NAN)], ids=["tprime_nan", "t_inf", "bias_nan"])
def test_engine_non_finite_scalars(tp, bias, f16):
    """t' = NaN or bias = NaN: every output NaN. t' = 1000: t = exp(t') = +inf in fp32 and float64, every logit +-inf,
    the loss +inf, dimg / dtxt / dt' non-finite, dbias = sum G finite."""
    eng = _engine("w1")
    img, txts = _problem("w1", seed=100)
    y = _labels(img.shape[0], eng.batch, [txts[0].shape[0]], 0)
    ref = _reference(_consumed(img, f16), [_consumed(txts[0], f16)], y, tp, bias, eng.batch)
    img_op, txt_ops = _operand(eng, img, f16), [_operand(eng, txts[0], f16)]
    for sched in ("fused", "split", "fwd"):
        out = _run(eng, img_op, txt_ops, tp, bias, sched, losses=(sched == "fused"))
        _check_step(f"t'={tp} b={bias} {sched}", eng, out, ref)


def test_row_panels_with_a_nan_text():
    eng = _engine("panels")
    g = torch.Generator().manual_seed(5)
    img, txt = _unit(g, 1000, D1), _spoil(_unit(g, 1000, D1), 611, "nan")
    y = _labels(1000, 1000, [1000], 0)
    ref = _reference(_consumed(img, False), [_consumed(txt, False)], y, TP, BIAS, 1000)
    out = _run(eng, _operand(eng, img, False), [_operand(eng, txt, False)], TP, BIAS, "fused", losses=True)
    _check_step("row panels", eng, out, ref)


# ---------------------------------------------------------------------------------------------------------------------
# 2. per-sample losses: the overflow class inside the supported range
# ---------------------------------------------------------------------------------------------------------------------
def test_sample_loss_overflow_is_exactly_inf():
    """Unnormalised bf16 image rows a * e (|x| <= 4094) against texts with <e, txt_j> ~ 0.6: every 128-column row partial
    of those images is ~10^5 > 2^16, so their image losses are exactly +inf, while every loss term, the loss, the
    gradients and the text losses stay finite and match the oracle."""
    eng = _engine("w1")
    g = torch.Generator().manual_seed(11)
    e = _unit(g, 1, D1)
    txt = torch.nn.functional.normalize(0.6 * e + 0.8 * _unit(g, B1 + K1, D1))
    img = _unit(g, B1 + E1, D1)
    hot = [3, 40, 77, B1 + 4]   # in different 16-row groups: no column partial reaches 2^16
    img[hot] = 400.0 * e
    assert float(img.abs().max()) <= 4094
    y = _labels(img.shape[0], B1, [txt.shape[0]], 0)
    ref = _reference(_consumed(img, False), [_consumed(txt, False)], y, TP, BIAS, B1)
    cls = sample_loss_classes(ref["terms"], [txt.shape[0]])
    assert np.isinf(cls["image_loss"]).tolist() == [i in hot for i in range(img.shape[0])]
    assert np.isfinite(cls["text_loss_part"]).all() and bool(torch.isfinite(ref["terms"]).all())
    out = _run(eng, _operand(eng, img, False), [_operand(eng, txt, False)], TP, BIAS, "fused", losses=True)
    _check_step("overflow", eng, out, ref)
    assert bool(torch.isfinite(out["loss"]).all())


def test_loopback_peer_poison_words():
    """Loopback W = 3: the own chunk's text losses add the peers' seeded partials and OR their poison words. Poison bit 1
    makes that text exactly +inf, bit 2 NaN (NaN wins, from either peer); every other text is the own partial plus the
    seeded values."""
    eng = _engine("w3")
    r, peers = eng.rank, [k for k in range(W3) if k != eng.rank]
    img, txts = _problem("w3", seed=61)
    ref = _reference(_consumed(img, False), [_consumed(t, False) for t in txts], _labels(B3, B3, [B3] * W3, r), TP,
                     BIAS, B3)
    rng = np.random.default_rng(3)
    seeded = np.zeros(B3)
    poison = [np.zeros(B3, np.int64) for _ in peers]
    poison[0][[4, 50, 120]] = [1, 1, 3]
    poison[1][[50, 90]] = 2
    for k, pw in zip(peers, poison):
        words = np.rint(rng.random(B3) * 50 * 2.0 ** 32).astype(np.int64)
        seeded += words / 2.0 ** 32
        eng.debug_set_peer_sample_loss_partials(k, torch.from_numpy(words).to(_dev()))
        eng.debug_set_peer_sample_loss_poison(k, torch.from_numpy(pw).to(_dev()))
    try:
        out = _run(eng, _operand(eng, img, False), [_operand(eng, t, False) for t in txts], TP, BIAS, "fused",
                   losses=True)
    finally:   # the engine is shared: no stand-in poison or partials for the tests after this one
        for k in peers:
            zero = torch.zeros(B3, dtype=torch.int64, device=_dev())
            eng.debug_set_peer_sample_loss_partials(k, zero)
            eng.debug_set_peer_sample_loss_poison(k, zero)
    _check_step("peer poison", eng, out, ref)
    want = ref["terms"][:, r * B3:(r + 1) * B3].sum(dim=0).numpy() + seeded
    want[4] = INF
    want[[50, 90, 120]] = NAN
    _classes("peer poison text_loss", out["text_loss"], want)


def test_convert_f32_keeps_non_finite_and_saturates_finite_values():
    """The fp32 -> fp16(16 x) conversion bit for bit: finite values as fp16(clamp(16 x, +-65504)), product overflow and
    signed zeros included; NaN stays NaN and +-inf stays +-inf."""
    eng = _engine("w1")
    vals = torch.tensor([0.0, -0.0, 1e-9, -3e-6, 1.0 / 3.0, -2.5, 4093.9, 4094.0, 4094.3, 4094.6, -4095.0, 4096.0, 5e3,
                         1e30, -3e38, 3.4e38, 1e-40, NAN, INF, -INF])
    x = vals.repeat(B1 * D1 // len(vals) + 1)[:B1 * D1].reshape(B1, D1).contiguous()
    got = eng.convert_f32(x.to(_dev()), True).cpu()
    y = x * 16.0
    want = torch.where(torch.isfinite(x), y.clamp(-65504.0, 65504.0), y).half()
    assert torch.equal(torch.isnan(got), torch.isnan(want))
    fin = ~torch.isnan(want)
    assert torch.equal(got[fin].view(torch.int16), want[fin].view(torch.int16))


# ---------------------------------------------------------------------------------------------------------------------
# 3. teacher embeddings (distillation, fp32 teacher through the fp16 conversion)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("where,value", [("teacher_image", "nan"), ("teacher_text", "nan"), ("teacher_text", "inf"),
                                         ("teacher_image", "nan_row")])
@pytest.mark.parametrize("fused", [True, False])
def test_fp32_teacher_non_finite(where, value, fused):
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss

    B, D, DT, lam = B1, D1, 72, 0.5
    ttp, tb = math.log(20.0), -8.0
    g = torch.Generator().manual_seed(21)
    img, txt = _unit(g, B, D).to(torch.bfloat16), _unit(g, B, D).to(torch.bfloat16)
    timg, ttxt = _unit(g, B, DT), _unit(g, B, DT)
    if where == "teacher_image":
        timg = _spoil(timg, 17, value)
    else:
        ttxt = _spoil(ttxt, 23, value)
    mod = DDPSigmoidLoss(B, distill=lam, fused_step=fused).to(_dev())
    a, b = img.to(_dev()).requires_grad_(True), txt.to(_dev()).requires_grad_(True)
    loss = mod(a, b, teacher_image=timg.to(_dev()), teacher_text=ttxt.to(_dev()),
               teacher_t_prime=torch.tensor(ttp, device=_dev()), teacher_bias=torch.tensor(tb, device=_dev()))
    loss.backward()
    y = _labels(B, B, [B], 0)
    teacher = (operand_values(timg), operand_values(ttxt), ttp, tb, lam)
    ref = _reference(img, [txt], y, TP, -10.0, B, teacher=teacher)
    # a NaN teacher entry makes targets NaN; an infinite one only saturates the teacher's sigma to 0 or 1
    assert bool(torch.isfinite(ref["loss"])) == (value == "inf")
    tag = f"{value} in {where} fused={fused}"
    _contract(f"{tag} loss", loss.detach(), ref["loss"])
    _contract(f"{tag} dimg", a.grad, ref["dimg"], 4e-3)   # bf16 gradients: 2^-9 rounding
    _contract(f"{tag} dtxt", b.grad, ref["contrib"][0], 4e-3)
    _contract(f"{tag} dt'", mod.t_prime.grad, ref["dtp"])
    _contract(f"{tag} dbias", mod.bias.grad, ref["db"])


# ---------------------------------------------------------------------------------------------------------------------
# 4. the modules
# ---------------------------------------------------------------------------------------------------------------------
MODULE_CASES = [(torch.bfloat16, False), (torch.float32, False), (torch.float16, False), (torch.float32, True),
                (torch.bfloat16, True)]


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("value,where", [("nan", "image"), ("inf", "text"), ("-inf", "image"), ("nan_row", "text")])
@pytest.mark.parametrize("dtype,normalize", MODULE_CASES, ids=lambda v: str(v).replace("torch.", ""))
def test_module_against_autograd(dtype, normalize, value, where, fused):
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss

    B, D, K = B1, D1, 20
    g = torch.Generator().manual_seed(31)
    scale = 3.0 if normalize else 1.0
    img, txt, neg = _unit(g, B, D) * scale, _unit(g, B, D) * scale, _unit(g, K, D) * scale
    if where == "image":
        img = _spoil(img, 8, value)
    else:
        txt = _spoil(txt, 13, value)
    img, txt, neg = img.to(dtype), txt.to(dtype), neg.to(dtype)
    mod = DDPSigmoidLoss(B, normalize_inputs=normalize, hard_negatives=K, fused_step=fused).to(_dev())
    a = img.to(_dev()).requires_grad_(True)
    b, c = txt.to(_dev()).requires_grad_(True), neg.to(_dev()).requires_grad_(True)
    loss = mod(a, b, negative_text=c)
    loss.backward()
    # normalize_inputs: the kernels normalise the raw values; otherwise they consume the operand values
    cv = (lambda x: x.double()) if normalize else operand_values  # noqa: E731
    ref = _reference(cv(img), [torch.cat([cv(txt), cv(neg)])], _labels(B, B, [B + K], 0), math.log(10), -10.0, B,
                     normalize=normalize)
    # bf16 gradients come back rounded to 2^-9; fp16 ones to 2^-11, inside the suite's 1e-3
    tol = 4e-3 if dtype == torch.bfloat16 else TOL
    tag = f"{dtype} normalize={normalize} {value} in {where} fused={fused}"
    _contract(f"{tag} loss", loss.detach(), ref["loss"])
    _contract(f"{tag} dimg", a.grad, ref["dimg"], tol)
    _contract(f"{tag} dtxt", torch.cat([b.grad, c.grad]), ref["contrib"][0], tol)
    _contract(f"{tag} dt'", mod.t_prime.grad, ref["dtp"])
    _contract(f"{tag} dbias", mod.bias.grad, ref["db"])


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_siglip_loss_nan_image(dtype):
    from distributed_sigmoid_loss_b200 import SigLipLoss

    B, D = B1, D1
    g = torch.Generator().manual_seed(41)
    img, txt = _spoil(_unit(g, B, D), 5, "nan").to(dtype), _unit(g, B, D).to(dtype)
    a, b = img.to(_dev()).requires_grad_(True), txt.to(_dev()).requires_grad_(True)
    tp = torch.tensor(TP, device=_dev(), requires_grad=True)
    bias = torch.tensor(BIAS, device=_dev(), requires_grad=True)
    loss = SigLipLoss()(a, b, tp, bias)
    loss.backward()
    ref = _reference(operand_values(img), [operand_values(txt)], _labels(B, B, [B], 0), TP, BIAS, B)
    tol = 4e-3 if dtype == torch.bfloat16 else TOL
    _contract("siglip loss", loss.detach(), ref["loss"])
    _contract("siglip dimg", a.grad, ref["dimg"], tol)
    _contract("siglip dtxt", b.grad, ref["contrib"][0], tol)
    _contract("siglip dt'", tp.grad, ref["dtp"])
    _contract("siglip dbias", bias.grad, ref["db"])


# ---------------------------------------------------------------------------------------------------------------------
# 5. metrics and top-K armed on a NaN step; zero rows
# ---------------------------------------------------------------------------------------------------------------------
def _grid(seed, n, D):
    """Small-integer vectors / 8: exact in bf16, every logit an exact fp32 number (ties are real ties)."""
    return torch.from_numpy(np.random.default_rng(seed).integers(-2, 3, (n, D)) / 8.0).float()


def _metrics_step(eng, img, txt, k):
    top1 = torch.zeros(2, device=_dev())
    i2t = torch.zeros(eng.metric_images, dtype=torch.int64, device=_dev())
    t2i = torch.zeros(eng.metric_texts, dtype=torch.int64, device=_dev())
    recall = torch.zeros(2 * k, device=_dev())
    i2t_k = torch.zeros(eng.metric_images, k, dtype=torch.int64, device=_dev())
    t2i_k = torch.zeros(eng.metric_texts, k, dtype=torch.int64, device=_dev())
    eng.request_metrics(top1, i2t, t2i)
    eng.request_topk(k, recall, i2t_k, t2i_k)
    out = _run(eng, _operand(eng, img, False), [_operand(eng, txt, False)], TP, BIAS, "fused")
    torch.cuda.synchronize()
    return out, top1.cpu(), i2t.cpu(), t2i.cpu(), recall.cpu(), i2t_k.cpu(), t2i_k.cpu()


def test_metrics_and_topk_on_a_nan_step():
    """A NaN text: the step finishes, every index is in range, the rates lie in [0, 1], and the t2i lists of every text
    whose column has no non-finite logit are the float64 oracle's exactly."""
    eng = _engine("w1")
    k, j = 5, 42
    img, txt = _grid(1, B1 + E1, D1), _spoil(_grid(2, B1 + K1, D1), j, "nan")
    out, top1, i2t, t2i, recall, i2t_k, t2i_k = _metrics_step(eng, img, txt, k)
    assert not bool(torch.isfinite(out["loss"]).all())
    R, T = B1 + E1, B1 + K1
    assert bool(((i2t >= 0) & (i2t < T)).all()) and bool(((t2i >= 0) & (t2i < R)).all())
    assert bool(((i2t_k >= -1) & (i2t_k < T)).all()) and bool(((t2i_k >= -1) & (t2i_k < R)).all())
    assert bool(((top1 >= 0) & (top1 <= 1)).all()) and bool(((recall >= 0) & (recall <= 1)).all())
    ref = topk_retrieval([img.double().numpy()], [txt.double().numpy()], [B1], k)[0]
    finite_cols = [m for m in range(B1) if m != j]
    assert torch.equal(t2i_k[finite_cols], torch.from_numpy(ref["t2i_topk"][finite_cols])), "t2i top-K lists"
    assert torch.equal(t2i[finite_cols], torch.from_numpy(ref["t2i_topk"][finite_cols, 0])), "t2i top-1"


def test_zero_rows():
    """A zero image row is finite and degenerate: its logits are exact zeros, so its i2t match and top-K list are the
    lowest indices; under normalize_inputs its gradient is dxhat / 1e-12, as with F.normalize."""
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss

    eng = _engine("w1")
    k, i = 5, 9
    img, txt = _grid(3, B1 + E1, D1), _grid(4, B1 + K1, D1)
    img[i] = 0.0
    out, _, i2t, _, _, i2t_k, _ = _metrics_step(eng, img, txt, k)
    assert bool(torch.isfinite(out["dimg"]).all())
    assert int(i2t[i]) == 0 and i2t_k[i].tolist() == list(range(k))
    g = torch.Generator().manual_seed(51)
    x, t = _unit(g, B1, D1) * 3, _unit(g, B1, D1) * 3
    x[i] = 0.0
    for fused in (True, False):
        mod = DDPSigmoidLoss(B1, normalize_inputs=True, fused_step=fused).to(_dev())
        a, b = x.to(_dev()).requires_grad_(True), t.to(_dev()).requires_grad_(True)
        mod(a, b).backward()
        ref = _reference(x.double(), [t.double()], _labels(B1, B1, [B1], 0), math.log(10), -10.0, B1, normalize=True)
        assert float(ref["dimg"][i].abs().max()) > 1e9
        _contract(f"zero row fused={fused} dimg", a.grad, ref["dimg"])
        _contract(f"zero row fused={fused} dimg row {i}", a.grad[i], ref["dimg"][i])
        _contract(f"zero row fused={fused} dtxt", b.grad, ref["contrib"][0])


# ---------------------------------------------------------------------------------------------------------------------
# 6. GradScaler end to end
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fused", [True, False])
def test_grad_scaler_skips_the_step_of_overflowing_fp16_towers(fused):
    """Two linear towers under fp16 autocast, the image tower's output overflowing to inf in one column (a bias beyond
    the fp16 range): the loss's text gradients carry the non-finite values back, so GradScaler skips the step
    (parameters unchanged) and halves the scale, as it does with the torch restatement as the loss. Without the overflow
    both take the step."""
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss

    B, Din, D = 64, 32, 128
    y = _labels(B, B, [B], 0).float().to(_dev())

    def restated(a, b, tp, bias):
        return torch_loss(a.float(), b.float(), tp.float(), bias, y, batch=B)

    def run(loss_kind, overflow):
        torch.manual_seed(0)
        towers = [torch.nn.Linear(Din, D).to(_dev()) for _ in range(2)]
        if overflow:
            with torch.no_grad():   # beyond the fp16 range: output column 5 of the image tower is +inf under autocast
                towers[0].bias[5] = 7e4
        mod = DDPSigmoidLoss(B, fused_step=fused).to(_dev())
        params = [p for t in towers for p in t.parameters()] + list(mod.parameters())
        opt = torch.optim.SGD(params, lr=0.1)
        # a small scale: a loss that saturated the inf to a finite value would leave every gradient finite in fp16
        scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** -8)
        g = torch.Generator().manual_seed(1)
        xi, xt = torch.randn(B, Din, generator=g).to(_dev()), torch.randn(B, Din, generator=g).to(_dev())
        before = [p.detach().clone() for p in params]
        with torch.autocast("cuda", dtype=torch.float16):
            a, b = towers[0](xi), towers[1](xt)
            assert a.dtype == torch.float16 and bool(torch.isinf(a).any()) == overflow
            if loss_kind == "kernel":
                loss = mod(a, b)
            else:
                with torch.autocast("cuda", enabled=False):
                    loss = restated(a, b, mod.t_prime, mod.bias)
        scaler.scale(loss).backward()
        scaler.step(opt)
        scaler.update()
        stepped = any(not torch.equal(p0, p.detach()) for p0, p in zip(before, params))
        return stepped, scaler.get_scale()

    for overflow in (True, False):
        want = run("restated", overflow)
        assert want == ((False, 2.0 ** -9) if overflow else (True, 2.0 ** -8))
        assert run("kernel", overflow) == want, f"overflow={overflow} fused={fused}"
