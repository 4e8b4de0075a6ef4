"""Multi-positive labels from sample ids (SIGLIP_OPT_SAMPLE_IDS) on the H100: unique ids reproduce the positional labels
bit for bit, duplicates (within and across text chunks) match the float64 oracle with the id label matrix, through the C
ABI (fused, split and forward-only), the loopback W-rank schedules, the modules and a captured CUDA graph."""
import math

import numpy as np
import pytest
import torch

from sample_ids_oracle import closed_form_ids

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


def _check(name, got, ref, tol=TOL):
    if np.ndim(ref) == 0 and not torch.is_tensor(ref):
        err = abs(float(got) - float(ref)) / (abs(float(ref)) + 1e-30)
        assert err <= tol, f"{name}: {float(got)} vs {float(ref)} (rel {err:.3e})"
    else:
        ef, em = _rel_f(got, ref), _max_rel(got, ref)
        assert ef <= tol and em <= tol, f"{name}: rel-Frobenius {ef:.3e}, max-abs/max {em:.3e}"


def _engine(B, D, cg=2, ids=True, **kw):
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi

    eng = SigmoidLossEngine(B, D, _dev(), cta_group=cg, **kw)
    if ids:
        eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 1)
    return eng


def _scal(x):
    return torch.tensor([x], device=_dev(), dtype=torch.float32)


def _blocks(Bs, D, seed):
    g = torch.Generator().manual_seed(seed)
    imgs = [torch.nn.functional.normalize(torch.randn(b, D, generator=g)).to(torch.bfloat16) for b in Bs]
    txts = [torch.nn.functional.normalize(torch.randn(b, D, generator=g)).to(torch.bfloat16) for b in Bs]
    return imgs, txts


def _unique_ids(Bs, seed):
    g = torch.Generator().manual_seed(seed)
    total = sum(Bs)
    ids = (torch.randperm(total, generator=g).to(torch.int64) - total // 2) * 8589934597   # negatives, beyond 2^32
    return list(torch.split(ids, list(Bs)))


def _oracle(imgs, txts, ids, tp, bias):
    return closed_form_ids([x.float().numpy() for x in imgs], [x.float().numpy() for x in txts],
                           [x.numpy() for x in ids], tp, bias)


def _step(eng, sched, img, txt, tp, b, gdt, ids=None, chunk_ids=None):
    """One step of rank eng.rank; returns every output including this rank's per-owner text contributions."""
    if ids is not None:
        for k, x in enumerate(chunk_ids or []):
            if k != eng.rank:
                eng.debug_set_chunk_ids(k, x.to(_dev()))
        eng.set_sample_ids(ids.to(_dev()))
    if sched == "fused":
        loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, tp, b, gdt)
    elif sched == "split":
        loss = eng.forward(img, txt, tp, b, True)
        dimg, dtxt, dtp, db = eng.backward(img, txt, tp, None, gdt)
    else:
        return [eng.fwd(img, txt, tp, b)]
    outs = [loss, dimg, dtxt, dtp, db]
    if eng.world > 1:
        outs += [eng.debug_get_slot(k) for k in range(eng.world) if k != eng.rank]
    return [x.clone() for x in outs]


# ---------------------------------------------------------------------------------------------------------------------
# 1. unique ids == positional labels, bit for bit
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("W", [1, 3])
def test_unique_ids_are_bit_identical_to_no_ids(W, cg):
    B, D = 300, 136
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    imgs, txts = _blocks([B] * W, D, 3)
    ids = _unique_ids([B] * W, 4)
    for r in range(W):
        kw = dict(rank_world=(r, W), loopback=True) if W > 1 else {}
        plain = _engine(B, D, cg, ids=False, **kw)
        with_ids = _engine(B, D, cg, ids=True, **kw)
        for eng in (plain, with_ids):
            for k in range(W):
                if W > 1:
                    eng.debug_set_text_chunk(k, txts[k].to(_dev()))
        img, txt = imgs[r].to(_dev()), txts[r].to(_dev())
        for sched in ("fused", "split", "fwd"):
            for gdt in ((torch.float32, torch.bfloat16) if sched != "fwd" else (torch.float32,)):
                a = _step(plain, sched, img, txt, tp, b, gdt)
                c = _step(with_ids, sched, img, txt, tp, b, gdt, ids[r], ids)
                torch.cuda.synchronize()
                for i, (x, y) in enumerate(zip(a, c)):
                    assert torch.equal(x, y), f"W={W} r={r} {sched} {gdt} output {i} differs"
        plain.close()
        with_ids.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. duplicates within one chunk against the float64 oracle
# ---------------------------------------------------------------------------------------------------------------------
def _single_rank_case(B, D, ids, tp, bias, img=None, txt=None, cg=2):
    if img is None:
        (img,), (txt,) = _blocks([B], D, 21)
    ref = _oracle([img], [txt], [ids], tp, bias)[0]
    eng = _engine(B, D, cg)
    for sched in ("fused", "split", "fwd"):
        out = _step(eng, sched, img.to(_dev()), txt.to(_dev()), _scal(tp), _scal(bias), torch.float32, ids)
        torch.cuda.synchronize()
        _check(f"{sched} loss", out[0], ref["loss"])
        if sched == "fwd":
            continue
        _check(f"{sched} dimg", out[1], ref["dimg"])
        _check(f"{sched} dtxt", out[2], ref["contrib"][0])
        _check(f"{sched} dt_prime", out[3], ref["dt_prime"])
        _check(f"{sched} dbias", out[4], ref["dbias"])
    eng.close()


@pytest.mark.parametrize("B,D", [(300, 136), (4096, 768)])
@pytest.mark.parametrize("kind", ["groups4", "classes10"])
def test_duplicate_ids_single_rank_match_the_oracle(B, D, kind):
    g = torch.Generator().manual_seed(B + D)
    ids = torch.arange(B) // 4 if kind == "groups4" else torch.randint(0, 10, (B,), generator=g)
    _single_rank_case(B, D, ids.to(torch.int64) - 2 ** 36, math.log(10.0), -10.0)


def test_warm_groups_share_content():
    """Members of a group share content (text = normalize(group mean of the images + noise)): the positive logits are
    large, so their slabs leave the fast series path and the labels decide the sign of large terms."""
    B, D = 512, 256
    g = torch.Generator().manual_seed(8)
    ids = torch.arange(B) // 4
    img = torch.nn.functional.normalize(torch.randn(B, D, generator=g))
    means = img.reshape(B // 4, 4, D).mean(1).repeat_interleave(4, 0)
    txt = torch.nn.functional.normalize(means + 0.3 * torch.randn(B, D, generator=g) / math.sqrt(D))
    img, txt = img.to(torch.bfloat16), txt.to(torch.bfloat16)
    tp, bias = math.log(20.0), -10.0
    z_pos = math.exp(tp) * float((img.float() * txt.float()).sum(1).mean()) + bias
    assert z_pos > -4.2                                   # the fast path's bound (kFastZ): these slabs go general
    _single_rank_case(B, D, ids, tp, bias, img, txt)


def test_all_equal_ids_make_every_pair_positive():
    B, D = 384, 128
    _single_rank_case(B, D, torch.full((B,), 7, dtype=torch.int64), math.log(10.0), -10.0)


# ---------------------------------------------------------------------------------------------------------------------
# 3. positives across chunks: loopback W-rank schedules
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Bs,bidir", [((160, 160, 160), False), ((128, 128, 128, 128), True), ((40, 24, 33), False)])
def test_cross_chunk_positives_loopback(Bs, bidir):
    from distributed_sigmoid_loss_b200 import _capi

    W, D = len(Bs), 72
    tp, bias = math.log(10.0), -8.0
    imgs, txts = _blocks(Bs, D, 41)
    g = torch.Generator().manual_seed(42)
    ids = list(torch.split(torch.randint(-5, 12, (sum(Bs),), generator=g), list(Bs)))    # 17 classes over all ranks
    ref = _oracle(imgs, txts, ids, tp, bias)
    uneven = len(set(Bs)) > 1
    for sched in ("fused", "split"):
        dtxt_sum = [torch.zeros(b, D, device=_dev()) for b in Bs]
        for r in range(W):
            eng = _engine(Bs[r], D, 2, rank_world=(r, W), loopback=True, batch_per_rank=Bs if uneven else None)
            if bidir:
                eng.set_option(_capi.SIGLIP_OPT_BIDIR, 1)
            for k in range(W):
                eng.debug_set_text_chunk(k, txts[k].to(_dev()))
            out = _step(eng, sched, imgs[r].to(_dev()), txts[r].to(_dev()), _scal(tp), _scal(bias), torch.float32,
                        ids[r], ids)
            torch.cuda.synchronize()
            _check(f"{sched} loss r{r}", out[0], ref[r]["loss"])
            _check(f"{sched} dimg r{r}", out[1], ref[r]["dimg"])
            _check(f"{sched} dt_prime r{r}", out[3], ref[r]["dt_prime"])
            _check(f"{sched} dbias r{r}", out[4], ref[r]["dbias"])
            slots = iter(out[5:])
            for k in range(W):
                got = out[2].float() if k == r else next(slots)
                _check(f"{sched} contribution r{r} -> owner {k}", got, ref[r]["contrib"][k])
                dtxt_sum[k] += got
            eng.close()
        for k in range(W):
            _check(f"{sched} dtxt owner {k}", dtxt_sum[k], sum(ref[r]["contrib"][k] for r in range(W)))


# ---------------------------------------------------------------------------------------------------------------------
# 4. the modules
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("inputs", ["bf16", "fp32", "normalize"])
@pytest.mark.parametrize("id_dtype", [torch.int32, torch.int64])
def test_modules_with_sample_ids(inputs, id_dtype):
    """DDPSigmoidLoss / SigLipLoss(multi_positive=True), both schedules, against the oracle. bf16 leaves get bf16
    gradients (2^-9 rounding of the result: 4e-3); fp32 leaves take the fp16 x 16 operand path (1e-3)."""
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    B, D = 256, 96
    tp, bias = math.log(10.0), -10.0
    g = torch.Generator().manual_seed(55)
    raw_i, raw_t = torch.randn(B, D, generator=g), torch.randn(B, D, generator=g)
    ids = (torch.arange(B) // 4).to(id_dtype)
    if inputs == "normalize":
        x_i, x_t = raw_i, raw_t
        ref_i, ref_t = torch.nn.functional.normalize(raw_i.double()), torch.nn.functional.normalize(raw_t.double())
    else:
        x_i, x_t = torch.nn.functional.normalize(raw_i), torch.nn.functional.normalize(raw_t)
        if inputs == "bf16":
            x_i, x_t = x_i.to(torch.bfloat16), x_t.to(torch.bfloat16)
        ref_i, ref_t = x_i.double(), x_t.double()
    ref = closed_form_ids([ref_i.numpy()], [ref_t.numpy()], [ids.to(torch.int64).numpy()], tp, bias)[0]
    if inputs == "normalize":
        # the leaves are the raw embeddings: F.normalize's backward, dx = (dxhat - xhat <xhat, dxhat>) / ||x||
        def proj(raw, xhat, d):
            d = torch.from_numpy(d)
            return ((d - xhat * (xhat * d).sum(1, keepdim=True)) / raw.double().norm(dim=1, keepdim=True)).numpy()
        ref["dimg"] = proj(raw_i, ref_i, ref["dimg"])
        ref["contrib"] = [proj(raw_t, ref_t, ref["contrib"][0])]
    gtol = 4e-3 if inputs == "bf16" else TOL
    for fused in (False, True):
        for kind in ("ddp", "siglip"):
            a = x_i.to(_dev()).requires_grad_(True)
            b = x_t.to(_dev()).requires_grad_(True)
            if kind == "ddp":
                mod = DDPSigmoidLoss(B, normalize_inputs=(inputs == "normalize"), fused_step=fused,
                                     multi_positive=True).to(_dev())
                loss = mod(a, b, sample_ids=ids.to(_dev()))
                sc = (mod.t_prime, mod.bias)
            else:
                if inputs == "normalize":
                    continue
                mod = SigLipLoss(fused_step=fused, multi_positive=True)
                sc = (torch.tensor(tp, device=_dev(), requires_grad=True),
                      torch.tensor(bias, device=_dev(), requires_grad=True))
                loss = mod(a, b, sc[0], sc[1], sample_ids=ids.to(_dev()))
            loss.backward()
            torch.cuda.synchronize()
            tag = f"{kind} fused={fused} {inputs} {id_dtype}"
            _check(f"{tag} loss", loss.detach(), ref["loss"])
            _check(f"{tag} dimg", a.grad.float(), ref["dimg"], gtol)
            _check(f"{tag} dtxt", b.grad.float(), ref["contrib"][0], gtol)
            _check(f"{tag} dt_prime", sc[0].grad, ref["dt_prime"])
            _check(f"{tag} dbias", sc[1].grad, ref["dbias"])


def test_split_schedule_generation_guard_sets_the_ids_again():
    """Two forwards with different ids, then the backward of the FIRST: the engine's saved state belongs to the second,
    so the backward re-runs the first forward — with the first call's ids."""
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss

    B, D = 256, 64
    tp, bias = math.log(10.0), -10.0
    (img,), (txt,) = _blocks([B], D, 77)
    ids1, ids2 = torch.arange(B) // 4, torch.arange(B) // 2
    ref1 = _oracle([img], [txt], [ids1], tp, bias)[0]
    mod = DDPSigmoidLoss(B, fused_step=False, multi_positive=True).to(_dev())
    a1, b1 = img.float().to(_dev()).requires_grad_(True), txt.float().to(_dev()).requires_grad_(True)
    a2, b2 = img.float().to(_dev()).requires_grad_(True), txt.float().to(_dev()).requires_grad_(True)
    l1 = mod(a1, b1, sample_ids=ids1.to(_dev()))
    l2 = mod(a2, b2, sample_ids=ids2.to(_dev()))
    l1.backward()
    torch.cuda.synchronize()
    assert float(l1) != float(l2)
    _check("loss 1", l1.detach(), ref1["loss"])
    _check("dimg 1", a1.grad, ref1["dimg"])
    _check("dtxt 1", b1.grad, ref1["contrib"][0])
    _check("dbias 1", mod.bias.grad, ref1["dbias"])


# ---------------------------------------------------------------------------------------------------------------------
# 5. CUDA graph
# ---------------------------------------------------------------------------------------------------------------------
def test_captured_step_follows_the_ids_buffer():
    B, D = 512, 128
    eng = _engine(B, D, 2)
    (img,), (txt,) = _blocks([B], D, 91)
    img, txt = img.to(_dev()), txt.to(_dev())
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    ids1 = (torch.arange(B) // 4).to(_dev())
    ids2 = torch.randint(0, 10, (B,), generator=torch.Generator().manual_seed(5)).to(_dev())
    eager = []
    for ids in (ids1, ids2):
        eng.set_sample_ids(ids)
        eager.append([x.clone() for x in eng.fwd_bwd(img, txt, tp, b)])
    assert not torch.equal(eager[0][1], eager[1][1])
    ids_s = ids1.clone()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        eng.set_sample_ids(ids_s)
        eng.fwd_bwd(img, txt, tp, b)
        with torch.cuda.graph(g, stream=side):
            eng.set_sample_ids(ids_s)
            outs = eng.fwd_bwd(img, txt, tp, b)
    torch.cuda.current_stream().wait_stream(side)
    g.replay()
    torch.cuda.synchronize()
    for x, e in zip(outs, eager[0]):
        assert torch.equal(x, e)
    ids_s.copy_(ids2)
    g.replay()
    torch.cuda.synchronize()
    for x, e in zip(outs, eager[1]):
        assert torch.equal(x, e)
    del g
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. errors
# ---------------------------------------------------------------------------------------------------------------------
def test_ids_mode_errors_have_the_documented_status():
    from distributed_sigmoid_loss_b200 import _capi

    B, D = 128, 64
    (img,), (txt,) = _blocks([B], D, 13)
    img, txt = img.to(_dev()), txt.to(_dev())
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    ids = torch.arange(B, device=_dev())
    plain = _engine(B, D, ids=False)
    with pytest.raises(_capi.SiglipError) as e:
        plain.set_sample_ids(ids)
    assert e.value.code == _capi.SIGLIP_ERR_STATE
    eng = _engine(B, D)
    launches = eng.launch_count
    for call in (lambda: eng.fwd_bwd(img, txt, tp, b), lambda: eng.forward(img, txt, tp, b, True),
                 lambda: eng.fwd(img, txt, tp, b)):
        with pytest.raises(_capi.SiglipError) as e:
            call()
        assert e.value.code == _capi.SIGLIP_ERR_STATE and "siglip_set_sample_ids" in str(e.value)
    assert eng.launch_count == launches                   # refused before launching anything
    eng.set_sample_ids(ids)
    eng.fwd_bwd(img, txt, tp, b)
    with pytest.raises(_capi.SiglipError) as e:           # the ids were consumed by that step
        eng.fwd_bwd(img, txt, tp, b)
    assert e.value.code == _capi.SIGLIP_ERR_STATE
    hi, ht = img.cpu(), txt.cpu()
    for call in (lambda: eng.fwd_bwd_host(hi, ht, math.log(10.0), -10.0),
                 lambda: eng.host_submit(hi, ht, math.log(10.0), -10.0)):
        with pytest.raises(_capi.SiglipError) as e:
            call()
        assert e.value.code == _capi.SIGLIP_ERR_STATE
    with pytest.raises(RuntimeError):
        eng.set_sample_ids(ids.to(torch.int32))
    torch.cuda.synchronize()
    eng.close()
    plain.close()
