"""Hard-negative captions (siglip_ctx_create_texts, DDPSigmoidLoss(hard_negatives=K)) on the H100: each rank's text chunk
is [paired captions; extras], the extras are negatives for every image of the global batch. Checked against the float64
oracle through the C ABI (fused, split, forward-only; cta_group 1 / 2, mcast 2), against an existing schedule (a W=2
loopback context whose second chunk holds the extras), in loopback W=3 / W=4 with uneven batches and a different K per
chunk, with sample ids, with the retrieval metrics, in a captured CUDA graph and through both modules."""
import math

import numpy as np
import pytest
import torch

from hard_negatives_oracle import closed_form_hard_negatives, retrieval_metrics_hard_negatives

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


def _scal(x):
    return torch.tensor([x], device=_dev(), dtype=torch.float32)


def _unit(n, D, g):
    return torch.nn.functional.normalize(torch.randn(n, D, generator=g)).to(torch.bfloat16)


def _blocks(Bs, Ks, D, seed):
    g = torch.Generator().manual_seed(seed)
    return [_unit(b, D, g) for b in Bs], [_unit(b, D, g) for b in Bs], [_unit(k, D, g) for k in Ks]


def _oracle(imgs, txts, extras, tp, bias, ids=None):
    f = lambda xs: [x.float().numpy() for x in xs]  # noqa: E731
    return closed_form_hard_negatives(f(imgs), f(txts), f(extras), tp, bias,
                                      None if ids is None else [x.numpy() for x in ids])


def _engine(B, T, D, cg=2, mcast=1, ids=False, Bs=None, Ts=None, **kw):
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi

    eng = SigmoidLossEngine(B, D, _dev(), cta_group=cg, batch_per_rank=Bs if Bs is not None else None,
                            texts_per_rank=Ts if Ts is not None else [T], **kw)
    if mcast != 1:
        eng.set_option(_capi.SIGLIP_OPT_MCAST, mcast)
    if ids:
        eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 1)
    return eng


def _step(eng, sched, img, txt, tp, b, gdt=torch.float32, ids=None):
    if ids is not None:
        eng.set_sample_ids(ids.to(_dev()))
    if sched == "fused":
        loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, tp, b, gdt)
    elif sched == "split":
        loss = eng.forward(img, txt, tp, b, True)
        dimg, dtxt, dtp, db = eng.backward(img, txt, tp, None, gdt)
    else:
        return [eng.fwd(img, txt, tp, b).clone()]
    outs = [loss, dimg, dtxt, dtp, db]
    if eng.world > 1:
        outs += [eng.debug_get_slot(k) for k in range(eng.world) if k != eng.rank]
    return [x.clone() for x in outs]


def _check_rank(tag, out, ref, own_contrib, tol=TOL):
    _check(f"{tag} loss", out[0], ref["loss"], tol)
    if len(out) == 1:
        return
    _check(f"{tag} dimg", out[1], ref["dimg"], tol)
    _check(f"{tag} dtxt", out[2], own_contrib, tol)
    _check(f"{tag} dt_prime", out[3], ref["dt_prime"], tol)
    _check(f"{tag} dbias", out[4], ref["dbias"], tol)


# ---------------------------------------------------------------------------------------------------------------------
# 1. one rank against the float64 oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,K,D", [(300, 37, 136), (4096, 4096, 768)])
@pytest.mark.parametrize("cg,mcast", [(1, 1), (2, 1), (2, 2)])
def test_single_rank_matches_the_oracle(B, K, D, cg, mcast):
    if B > 1000 and (cg, mcast) != (2, 1):
        pytest.skip("the large shape runs at the default cluster shape only")
    tp, bias = math.log(10.0), -10.0
    (img,), (txt,), (ext,) = _blocks([B], [K], D, B + K + D)
    ref = _oracle([img], [txt], [ext], tp, bias)[0]
    eng = _engine(B, B + K, D, cg, mcast)
    full = torch.cat([txt, ext]).to(_dev())
    for sched in ("fused", "split", "fwd"):
        out = _step(eng, sched, img.to(_dev()), full, _scal(tp), _scal(bias))
        torch.cuda.synchronize()
        _check_rank(f"{sched} cg={cg} mcast={mcast}", out, ref, ref["contrib"][0])
        if sched != "fwd":
            _check(f"{sched} dtxt of the extras", out[2][B:], ref["contrib"][0][B:])
    eng.close()


def test_planted_extras_near_their_image_take_the_general_path():
    """Extras that lie close to an image (a perturbed copy of it): their logits are far above the fast path's bound, so
    the slabs that hold them run the general path with label -1 on a large z."""
    B, K, D = 512, 200, 256
    g = torch.Generator().manual_seed(3)
    img = torch.nn.functional.normalize(torch.randn(B, D, generator=g))
    txt = torch.nn.functional.normalize(img + 0.3 * torch.randn(B, D, generator=g) / math.sqrt(D))
    ext = torch.nn.functional.normalize(img[:K] + 0.2 * torch.randn(K, D, generator=g) / math.sqrt(D))
    img, txt, ext = (x.to(torch.bfloat16) for x in (img, txt, ext))
    tp, bias = math.log(20.0), -10.0
    z_ext = math.exp(tp) * float((img[:K].float() * ext.float()).sum(1).mean()) + bias
    assert z_ext > 5.0                                    # far above the fast path's bound (kFastZ)
    ref = _oracle([img], [txt], [ext], tp, bias)[0]
    eng = _engine(B, B + K, D)
    for sched in ("fused", "split", "fwd"):
        out = _step(eng, sched, img.to(_dev()), torch.cat([txt, ext]).to(_dev()), _scal(tp), _scal(bias))
        torch.cuda.synchronize()
        _check_rank(f"planted {sched}", out, ref, ref["contrib"][0])
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. the same numbers as an existing schedule: W=1 with K extras == rank 0 of a loopback W=2 [B, K] context
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,K", [(300, 37), (256, 640)])
def test_extras_match_a_second_chunk_of_a_loopback_context(B, K):
    D = 136
    tp, b = _scal(math.log(10.0)), _scal(-9.0)
    (img,), (txt,), (ext,) = _blocks([B], [K], D, 17)
    img, txt, ext = img.to(_dev()), txt.to(_dev()), ext.to(_dev())
    one = _engine(B, B + K, D)
    two = _engine(B, B, D, rank_world=(0, 2), loopback=True, Bs=[B, K], Ts=[B, K])
    two.debug_set_text_chunk(0, txt)
    two.debug_set_text_chunk(1, ext)
    for sched in ("fused", "split"):
        a = _step(one, sched, img, torch.cat([txt, ext]), tp, b)
        c = _step(two, sched, img, txt, tp, b)
        torch.cuda.synchronize()
        for i, name in ((0, "loss"), (1, "dimg"), (3, "dt_prime"), (4, "dbias")):
            _check(f"{sched} {name}", a[i], c[i], 1e-5)
        _check(f"{sched} dtxt of the paired texts", a[2][:B], c[2], 1e-5)
        _check(f"{sched} dtxt of the extras vs slot 1", a[2][B:], c[5], 1e-5)
    one.close()
    two.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. loopback W-rank schedules: uneven batches, a different K per chunk
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Bs,Ks,bidir,with_ids", [((160, 96, 130), (40, 0, 200), False, False),
                                                  ((128, 128, 128, 128), (16, 300, 5, 64), True, False),
                                                  ((40, 24, 33), (9, 30, 1), False, True)])
def test_loopback_schedules_with_extras(Bs, Ks, bidir, with_ids):
    from distributed_sigmoid_loss_b200 import _capi

    W, D = len(Bs), 72
    tp, bias = math.log(10.0), -8.0
    imgs, txts, extras = _blocks(Bs, Ks, D, 41)
    Ts = [b + k for b, k in zip(Bs, Ks)]
    ids = None
    if with_ids:
        g = torch.Generator().manual_seed(42)
        ids = list(torch.split(torch.randint(-5, 12, (sum(Bs),), generator=g), list(Bs)))
        extras[0][0] = txts[1][0]                         # an extra that copies another rank's caption stays negative
    ref = _oracle(imgs, txts, extras, tp, bias, ids)
    full = [torch.cat([t, e]) for t, e in zip(txts, extras)]
    for sched in ("fused", "split"):
        dtxt_sum = [torch.zeros(t, D, device=_dev()) for t in Ts]
        for r in range(W):
            eng = _engine(Bs[r], Ts[r], D, ids=with_ids, rank_world=(r, W), loopback=True, Bs=list(Bs), Ts=Ts)
            if bidir:
                eng.set_option(_capi.SIGLIP_OPT_BIDIR, 1)
            for k in range(W):
                eng.debug_set_text_chunk(k, full[k].to(_dev()))
                if with_ids and k != r:
                    eng.debug_set_chunk_ids(k, ids[k].to(_dev()))
            out = _step(eng, sched, imgs[r].to(_dev()), full[r].to(_dev()), _scal(tp), _scal(bias),
                        ids=ids[r] if with_ids else None)
            torch.cuda.synchronize()
            _check_rank(f"{sched} r{r}", out, ref[r], ref[r]["contrib"][r])
            slots = iter(out[5:])
            for k in range(W):
                got = out[2].float() if k == r else next(slots)
                _check(f"{sched} contribution r{r} -> owner {k}", got, ref[r]["contrib"][k])
                dtxt_sum[k] += got
            eng.close()
        for k in range(W):
            _check(f"{sched} dtxt owner {k}", dtxt_sum[k], sum(ref[r]["contrib"][k] for r in range(W)))


def test_ids_with_duplicates_never_make_an_extra_positive():
    B, K, D = 384, 96, 128
    g = torch.Generator().manual_seed(5)
    (img,), (txt,), (ext,) = _blocks([B], [K], D, 6)
    ext[:K] = txt[:K]                                     # every extra a copy of a caption, same content
    ids = (torch.arange(B) // 4).to(torch.int64)
    ref = _oracle([img], [txt], [ext], math.log(10.0), -10.0, [ids])[0]
    eng = _engine(B, B + K, D, ids=True)
    for sched in ("fused", "split", "fwd"):
        out = _step(eng, sched, img.to(_dev()), torch.cat([txt, ext]).to(_dev()), _scal(math.log(10.0)),
                    _scal(-10.0), ids=ids)
        torch.cuda.synchronize()
        _check_rank(f"ids {sched}", out, ref, ref["contrib"][0])
    del g
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. retrieval metrics
# ---------------------------------------------------------------------------------------------------------------------
def _planted(B, K, D, seed):
    """Captions are perturbed images; extra j is a closer copy of image 2j, so images 0, 2, 4, ... (up to 2K) rank their
    hard negative first: a miss at global index B + j."""
    g = torch.Generator().manual_seed(seed)
    img = torch.nn.functional.normalize(torch.randn(B, D, generator=g))
    txt = torch.nn.functional.normalize(img + 0.5 * torch.randn(B, D, generator=g) / math.sqrt(D))
    ext = torch.nn.functional.normalize(img[0:2 * K:2] + 0.1 * torch.randn(K, D, generator=g) / math.sqrt(D))
    return img.to(torch.bfloat16), txt.to(torch.bfloat16), ext.to(torch.bfloat16)


@pytest.mark.parametrize("B,K,D", [(300, 37, 136), (4096, 1024, 768)])
def test_metrics_count_a_winning_extra_as_a_miss(B, K, D):
    img, txt, ext = _planted(B, K, D, B)
    res = retrieval_metrics_hard_negatives([img.float().numpy()], [txt.float().numpy()], [ext.float().numpy()])[0]
    assert (res["i2t_index"][0:2 * K:2] == B + np.arange(K)).all()       # the plant: every extra wins its image
    eng, plain = _engine(B, B + K, D), _engine(B, B + K, D)
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    full, im = torch.cat([txt, ext]).to(_dev()), img.to(_dev())
    for sched in ("fused", "split", "fwd"):
        top1 = torch.empty(2, device=_dev())
        i2t = torch.empty(B, device=_dev(), dtype=torch.int64)
        t2i = torch.empty(B, device=_dev(), dtype=torch.int64)
        eng.request_metrics(top1, i2t, t2i)
        armed = _step(eng, sched, im, full, tp, b)
        unarmed = _step(plain, sched, im, full, tp, b)
        torch.cuda.synchronize()
        for i, (x, y) in enumerate(zip(armed, unarmed)):
            assert torch.equal(x, y), f"{sched}: output {i} of the armed step differs"
        assert torch.equal(i2t.cpu(), torch.from_numpy(res["i2t_index"])), sched
        assert torch.equal(t2i.cpu(), torch.from_numpy(res["t2i_index"])), sched
        assert int(i2t.max()) < B + K and int(i2t.min()) >= 0
        assert abs(float(top1[0]) - res["i2t_top1"]) < 1e-6 and abs(float(top1[1]) - res["t2i_top1"]) < 1e-6
        assert float(top1[0]) <= 1.0 - K / B + 1e-6                       # every planted extra is a miss
    eng.close()
    plain.close()


def test_metrics_loopback_index_over_every_rank_texts():
    """W=3 loopback, uneven batches and K: i2t indexes the concatenation [paired_0, extras_0, paired_1, ...]."""
    Bs, Ks, D = (96, 64, 80), (20, 30, 7), 128
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    imgs, txts, extras = [], [], []
    for r, (B, K) in enumerate(zip(Bs, Ks)):
        i, t, e = _planted(B, K, D, 100 + r)
        imgs.append(i), txts.append(t), extras.append(e)
    # rank 1's extras are near rank 0's images: a cross-rank hard negative
    extras[1][:10] = torch.nn.functional.normalize(imgs[0][1:21:2].float() + 0.01).to(torch.bfloat16)
    res = retrieval_metrics_hard_negatives([x.float().numpy() for x in imgs], [x.float().numpy() for x in txts],
                                           [x.float().numpy() for x in extras])
    Ts = [b_ + k for b_, k in zip(Bs, Ks)]
    full = [torch.cat([t, e]) for t, e in zip(txts, extras)]
    for r in range(3):
        eng = _engine(Bs[r], Ts[r], D, rank_world=(r, 3), loopback=True, Bs=list(Bs), Ts=Ts)
        for k in range(3):
            eng.debug_set_text_chunk(k, full[k].to(_dev()))
        top1 = torch.empty(2, device=_dev())
        i2t = torch.empty(Bs[r], device=_dev(), dtype=torch.int64)
        eng.request_metrics(top1, i2t, None)
        eng.fwd_bwd(imgs[r].to(_dev()), full[r].to(_dev()), tp, b)
        torch.cuda.synchronize()
        assert torch.equal(i2t.cpu(), torch.from_numpy(res[r]["i2t_index"])), r
        assert abs(float(top1[0]) - res[r]["i2t_top1"]) < 1e-6, r
        eng.close()
    assert (res[0]["i2t_index"][1:21:2] >= Ts[0] + Bs[1]).all()          # the plant crossed ranks


# ---------------------------------------------------------------------------------------------------------------------
# 5. CUDA graph, modules, errors
# ---------------------------------------------------------------------------------------------------------------------
def test_captured_step_with_extras_replays_the_eager_step():
    B, K, D = 512, 256, 128
    (img,), (txt,), (ext,) = _blocks([B], [K], D, 91)
    img, full = img.to(_dev()), torch.cat([txt, ext]).to(_dev())
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    eng = _engine(B, B + K, D)
    eager = [x.clone() for x in eng.fwd_bwd(img, full, tp, b)]
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        eng.fwd_bwd(img, full, tp, b)
        with torch.cuda.graph(g, stream=side):
            outs = eng.fwd_bwd(img, full, tp, b)
    torch.cuda.current_stream().wait_stream(side)
    g.replay()
    torch.cuda.synchronize()
    for x, e in zip(outs, eager):
        assert torch.equal(x, e)
    del g
    eng.close()


@pytest.mark.parametrize("inputs", ["bf16", "fp32", "normalize"])
def test_modules_return_the_negatives_gradient(inputs):
    """DDPSigmoidLoss / SigLipLoss(hard_negatives=K): negative_text.grad (and the rest) against the oracle, fused and
    split, with metrics and sample ids composed in. bf16 leaves get bf16 gradients (4e-3)."""
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    B, K, D = 256, 48, 96
    tp, bias = math.log(10.0), -10.0
    g = torch.Generator().manual_seed(55)
    raw = [torch.randn(n, D, generator=g) for n in (B, B, K)]
    ids = (torch.arange(B) // 2).to(torch.int64)
    if inputs == "normalize":
        xs = raw
        refs = [torch.nn.functional.normalize(x.double()) for x in raw]
    else:
        xs = [torch.nn.functional.normalize(x) for x in raw]
        if inputs == "bf16":
            xs = [x.to(torch.bfloat16) for x in xs]
        refs = [x.double() for x in xs]
    gtol = 4e-3 if inputs == "bf16" else TOL
    for with_ids in (False, True):
        ref = closed_form_hard_negatives([refs[0].numpy()], [refs[1].numpy()], [refs[2].numpy()], tp, bias,
                                         [ids.numpy()] if with_ids else None)[0]
        dimg_ref, dtxt_ref = ref["dimg"], ref["contrib"][0]
        if inputs == "normalize":
            def proj(r, xhat, d):
                d = torch.from_numpy(d)
                return ((d - xhat * (xhat * d).sum(1, keepdim=True)) / r.double().norm(dim=1, keepdim=True)).numpy()
            dimg_ref = proj(raw[0], refs[0], dimg_ref)
            dtxt_ref = proj(torch.cat(raw[1:]), torch.cat(refs[1:]), dtxt_ref)
        for fused in (False, True):
            for kind in ("ddp", "siglip"):
                if kind == "siglip" and inputs == "normalize":
                    continue
                a, b_, e = (x.to(_dev()).requires_grad_(True) for x in xs)
                kw = dict(negative_text=e, sample_ids=ids.to(_dev()) if with_ids else None, return_metrics=True)
                if kind == "ddp":
                    mod = DDPSigmoidLoss(B, normalize_inputs=(inputs == "normalize"), fused_step=fused,
                                         multi_positive=with_ids, hard_negatives=K).to(_dev())
                    loss, met = mod(a, b_, **kw)
                    sc = (mod.t_prime, mod.bias)
                else:
                    mod = SigLipLoss(fused_step=fused, multi_positive=with_ids, hard_negatives=K)
                    sc = (torch.tensor(tp, device=_dev(), requires_grad=True),
                          torch.tensor(bias, device=_dev(), requires_grad=True))
                    loss, met = mod(a, b_, sc[0], sc[1], **kw)
                loss.backward()
                torch.cuda.synchronize()
                tag = f"{kind} fused={fused} {inputs} ids={with_ids}"
                _check(f"{tag} loss", loss.detach(), ref["loss"])
                _check(f"{tag} dimg", a.grad.float(), dimg_ref, gtol)
                _check(f"{tag} dtxt", b_.grad.float(), dtxt_ref[:B], gtol)
                _check(f"{tag} negative_text.grad", e.grad.float(), dtxt_ref[B:], gtol)
                assert e.grad.dtype == e.dtype and e.grad.shape == e.shape
                _check(f"{tag} dt_prime", sc[0].grad, ref["dt_prime"])
                _check(f"{tag} dbias", sc[1].grad, ref["dbias"])
                assert met["i2t_index"].shape == (B,) and int(met["i2t_index"].max()) < B + K


def test_split_schedule_generation_guard_with_extras():
    """Two forwards with different extras, then the backward of the FIRST: the re-run forward takes the first call's
    [txt; negative_text] operand again."""
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss

    B, K, D = 256, 40, 64
    tp, bias = math.log(10.0), -10.0
    (img,), (txt,), (e1,) = _blocks([B], [K], D, 77)
    e2 = torch.nn.functional.normalize(img[:K].float()).to(torch.bfloat16)
    ref1 = _oracle([img], [txt], [e1], tp, bias)[0]
    mod = DDPSigmoidLoss(B, fused_step=False, hard_negatives=K).to(_dev())
    leaves1 = [x.float().to(_dev()).requires_grad_(True) for x in (img, txt, e1)]
    leaves2 = [x.float().to(_dev()).requires_grad_(True) for x in (img, txt, e2)]
    l1 = mod(leaves1[0], leaves1[1], negative_text=leaves1[2])
    l2 = mod(leaves2[0], leaves2[1], negative_text=leaves2[2])
    l1.backward()
    torch.cuda.synchronize()
    assert float(l1) != float(l2)
    _check("loss 1", l1.detach(), ref1["loss"])
    _check("dimg 1", leaves1[0].grad, ref1["dimg"])
    _check("negative_text.grad 1", leaves1[2].grad, ref1["contrib"][0][B:])


def test_host_entries_refuse_a_context_with_extras():
    from distributed_sigmoid_loss_b200 import _capi

    B, K, D = 128, 16, 64
    eng = _engine(B, B + K, D)
    hi, ht = torch.zeros(B, D, dtype=torch.bfloat16), torch.zeros(B, D, dtype=torch.bfloat16)
    launches = eng.launch_count
    for call in (lambda: eng.fwd_bwd_host(hi, ht, math.log(10.0), -10.0),
                 lambda: eng.host_submit(hi, ht, math.log(10.0), -10.0)):
        with pytest.raises(_capi.SiglipError) as e:
            call()
        assert e.value.code == _capi.SIGLIP_ERR_STATE and "hard negatives" in str(e.value)
    assert eng.launch_count == launches
    with pytest.raises(RuntimeError, match=r"\[144, 64\]"):
        eng.fwd_bwd(torch.zeros(B, D, dtype=torch.bfloat16, device=_dev()),
                    torch.zeros(B, D, dtype=torch.bfloat16, device=_dev()), _scal(0.0), _scal(0.0))
    eng.close()
