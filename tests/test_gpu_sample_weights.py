"""Per-sample loss weights (SIGLIP_OPT_SAMPLE_WEIGHTS, DDPSigmoidLoss / SigLipLoss(sample_weights=True)) on the H100.
Unit weights are checked bit for bit against the unweighted step, zero weights against the float64 oracle on the batch
without those samples, random weights against the weighted float64 oracle (W = 1, loopback W = 3 and W = 4 bidir,
uneven batches); then clamping, a captured CUDA graph, the modules with their metrics, and the error statuses."""
import math

import pytest
import torch

from sample_weights_oracle import closed_form_weighted, label_blocks

pytestmark = pytest.mark.gpu

TOL = 1e-3
CLUSTERS = [(1, 1), (2, 1), (2, 2)]


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


def _unit(g, n, D):
    return torch.nn.functional.normalize(torch.randn(n, D, generator=g)).to(torch.bfloat16)


def _engine(B, D, cg=2, mcast=1, Bs=None, Ts=None, ids=False, extra_ids=False, weights=True, **kw):
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi

    eng = SigmoidLossEngine(B, D, _dev(), cta_group=cg, batch_per_rank=Bs, texts_per_rank=Ts, **kw)
    if mcast != 1:
        eng.set_option(_capi.SIGLIP_OPT_MCAST, mcast)
    if ids:
        eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 1)
    if extra_ids:
        eng.set_option(_capi.SIGLIP_OPT_EXTRA_TEXT_IDS, 1)
    if weights:
        eng.set_option(_capi.SIGLIP_OPT_SAMPLE_WEIGHTS, 1)
    eng.weighted = weights
    return eng


def _dv(x):
    return None if x is None else x.to(_dev())


def _step(eng, sched, img, txt, tp, b, ids=None, eids=None, iw=None, tw=None):
    """One step; returns its outputs (fwd: the loss only) and, at W > 1, this rank's contribution slots to the peers."""
    if ids is not None:
        eng.set_sample_ids(_dv(ids))
    if eids is not None and eng.extra_text_ids:
        eng.set_extra_text_ids(_dv(eids))
    if eng.weighted:
        eng.set_sample_weights(_dv(iw), _dv(tw))
    if sched == "fused":
        loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, tp, b)
    elif sched == "split":
        loss = eng.forward(img, txt, tp, b, True)
        dimg, dtxt, dtp, db = eng.backward(img, txt, tp, None)
    else:
        return [eng.fwd(img, txt, tp, b).clone()]
    outs = [loss, dimg, dtxt, dtp, db]
    if eng.world > 1:
        outs += [eng.debug_get_slot(k) for k in range(eng.world) if k != eng.rank]
    return [x.clone() for x in outs]


def _loopback(eng, r, texts, ids=None, eids=None, tws=None):
    """Stand-ins of the peers' published chunks: text, ids and (weighted engines) text weights."""
    for k in range(eng.world):
        eng.debug_set_text_chunk(k, texts[k].to(_dev()))
        if k == r:
            continue
        if ids is not None:
            eng.debug_set_chunk_ids(k, (torch.cat([ids[k], eids[k]]) if eng.extra_text_ids else ids[k]).to(_dev()))
        if eng.weighted:
            eng.debug_set_chunk_weights(k, None if tws is None else tws[k].to(_dev()))


def _contribs(out, r, W):
    """This rank's contribution to every chunk's text gradient: dtxt for its own chunk, the slots for the others."""
    slots = iter(out[5:])
    return [out[2].float() if k == r else next(slots) for k in range(W)]


def _check_step(tag, out, ref, r, W, tol=TOL):
    _check(f"{tag} loss", out[0], ref["loss"], tol)
    if len(out) == 1:
        return
    _check(f"{tag} dimg", out[1], ref["dimg"], tol)
    _check(f"{tag} dt_prime", out[3], ref["dt_prime"], tol)
    _check(f"{tag} dbias", out[4], ref["dbias"], tol)
    for k, got in enumerate(_contribs(out, r, W)):
        _check(f"{tag} contribution to chunk {k}", got, ref["contrib"][k], tol)


def _problem(Bs, Ks, D, seed, mode):
    """Inputs of a W-rank problem. mode: pos (positional labels), ids (duplicated sample ids), hn (hard negatives with
    ids), extra (extra texts with ids, some captioning images of other ranks)."""
    g = torch.Generator().manual_seed(seed)
    imgs = [_unit(g, b, D) for b in Bs]
    texts = [_unit(g, b + k, D) for b, k in zip(Bs, Ks)]
    ids = eids = None
    if mode != "pos":
        ids = list(torch.split(torch.randint(0, max(Bs), (sum(Bs),), generator=g), list(Bs)))
        eids = [torch.randint(0, 2 * max(Bs), (k,), generator=g) for k in Ks]
    return imgs, texts, ids, eids


def _labels(Bs, Ks, ids, eids, mode):
    Ts = [b + k for b, k in zip(Bs, Ks)]
    f = (lambda xs: None if xs is None else [x.numpy() for x in xs])  # noqa: E731
    return label_blocks(Bs, Ts, f(ids), f(eids) if mode == "extra" else None)


def _oracle(imgs, texts, tp, bias, iws, tws, labels):
    f = (lambda xs: None if xs is None else [x.double().numpy() for x in xs])  # noqa: E731
    return closed_form_weighted(f(imgs), f(texts), tp, bias, f(iws), f(tws), labels)


# ---------------------------------------------------------------------------------------------------------------------
# 1. unit weights: bit for bit the unweighted step
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["pos", "ids", "hn", "extra"])
@pytest.mark.parametrize("cg,mcast", CLUSTERS)
@pytest.mark.parametrize("W", [1, 3])
def test_unit_weights_are_bitwise_the_unweighted_step(W, cg, mcast, mode):
    Bs = (300,) if W == 1 else (96, 64, 80)
    Ks = tuple(0 for _ in Bs) if mode in ("pos", "ids") else ((37,) if W == 1 else (40, 0, 130))
    D = 136 if W == 1 else 72
    Ts = [b + k for b, k in zip(Bs, Ks)]
    imgs, texts, ids, eids = _problem(Bs, Ks, D, W * 100 + cg * 10 + mcast, mode)
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    for r in range(W):
        kw = dict(rank_world=(r, W), loopback=True) if W > 1 else {}
        opts = dict(ids=mode != "pos", extra_ids=mode == "extra", Bs=list(Bs), Ts=Ts, **kw)
        wt, plain = _engine(Bs[r], D, cg, mcast, weights=True, **opts), _engine(Bs[r], D, cg, mcast, weights=False, **opts)
        ones = [torch.ones(t) for t in Ts]
        if W > 1:
            _loopback(wt, r, texts, ids, eids, ones)
            _loopback(plain, r, texts, ids, eids)
        for sched in ("fused", "split", "fwd"):
            # explicit ones, and None (ones written by the copy) on the forward-only step
            iw, tw = (None, None) if sched == "fwd" else (torch.ones(Bs[r]), ones[r])
            a = _step(wt, sched, imgs[r].to(_dev()), texts[r].to(_dev()), tp, b, ids and ids[r], eids and eids[r], iw, tw)
            c = _step(plain, sched, imgs[r].to(_dev()), texts[r].to(_dev()), tp, b, ids and ids[r], eids and eids[r])
            torch.cuda.synchronize()
            for i, (x, y) in enumerate(zip(a, c)):
                assert torch.equal(x, y), f"W={W} r={r} {sched} {mode}: output {i} differs from the unweighted step"
        wt.close()
        plain.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. zero weights: the step of the batch without those samples (x (B - m) / B), masked rows exactly 0
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W", [1, 3])
def test_zero_weights_equal_the_batch_without_the_samples(W):
    Bs = (300,) if W == 1 else (96, 64, 80)
    D = 136 if W == 1 else 72
    imgs, texts, _, _ = _problem(Bs, (0,) * W, D, 40 + W, "pos")
    tp, bias = math.log(10.0), -10.0
    g = torch.Generator().manual_seed(W)
    drop = [torch.randperm(b, generator=g)[: b // 10] for b in Bs]    # 10 % of every rank's samples, peers' too
    ws = []
    for b, d in zip(Bs, drop):
        w = torch.ones(b)
        w[d] = 0.0
        ws.append(w)
    keep = [torch.nonzero(w).flatten() for w in ws]
    kB = [len(k) for k in keep]
    ref = _oracle([x[k] for x, k in zip(imgs, keep)], [x[k] for x, k in zip(texts, keep)], tp, bias, None, None,
                  label_blocks(kB, kB))
    for r in range(W):
        eng = _engine(Bs[r], D, Bs=list(Bs), **(dict(rank_world=(r, W), loopback=True) if W > 1 else {}))
        if W > 1:
            _loopback(eng, r, texts, tws=ws)
        f = kB[r] / Bs[r]
        for sched in ("fused", "split", "fwd"):
            out = _step(eng, sched, imgs[r].to(_dev()), texts[r].to(_dev()), _scal(tp), _scal(bias), iw=ws[r], tw=ws[r])
            torch.cuda.synchronize()
            tag = f"W={W} r={r} {sched}"
            _check(f"{tag} loss", out[0], ref[r]["loss"] * f)
            if sched == "fwd":
                continue
            _check(f"{tag} dt_prime", out[3], ref[r]["dt_prime"] * f)
            _check(f"{tag} dbias", out[4], ref[r]["dbias"] * f)
            _check(f"{tag} dimg", out[1][keep[r]], ref[r]["dimg"] * f)
            assert not out[1][drop[r]].any(), f"{tag}: dimg rows of dropped images are not 0"
            for k, got in enumerate(_contribs(out, r, W)):
                _check(f"{tag} contribution to chunk {k}", got[keep[k]], ref[r]["contrib"][k] * f)
                assert not got[drop[k]].any(), f"{tag}: rows of dropped texts of chunk {k} are not 0"
        eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. random weights in [0, 1] against the weighted float64 oracle
# ---------------------------------------------------------------------------------------------------------------------
def _random_weights(g, n):
    w = torch.rand(n, generator=g)
    w[torch.rand(n, generator=g) < 0.1] = 0.0
    w[torch.rand(n, generator=g) < 0.1] = 1.0
    return w


@pytest.mark.parametrize("B,K,D,mode", [(300, 37, 136, "hn"), (300, 0, 136, "ids"), (4096, 0, 768, "pos")])
@pytest.mark.parametrize("cg,mcast", CLUSTERS)
def test_single_rank_random_weights_match_the_oracle(B, K, D, mode, cg, mcast):
    if B > 1000 and (cg, mcast) != (2, 1):
        pytest.skip("the large shape runs at the default cluster shape only")
    tp, bias = math.log(10.0), -10.0
    (img,), (txt,), ids, eids = _problem((B,), (K,), D, B + K + cg, mode)
    g = torch.Generator().manual_seed(5)
    iw, tw = _random_weights(g, B), _random_weights(g, B + K)
    ref = _oracle([img], [txt], tp, bias, [iw], [tw], _labels((B,), (K,), ids, eids, mode))[0]
    eng = _engine(B, D, cg, mcast, ids=mode != "pos", Ts=[B + K])
    for sched in ("fused", "split", "fwd"):
        out = _step(eng, sched, img.to(_dev()), txt.to(_dev()), _scal(tp), _scal(bias), ids and ids[0],
                    eids and eids[0], iw, tw)
        torch.cuda.synchronize()
        _check_step(f"{sched} B={B} K={K} {mode} cg={cg} mcast={mcast}", out, ref, 0, 1)
    eng.close()


@pytest.mark.parametrize("Bs,Ks,mode,bidir", [((160, 96, 130), (0, 0, 0), "pos", False),
                                              ((160, 96, 130), (40, 0, 200), "extra", False),
                                              ((128, 128, 128, 128), (0, 0, 0, 0), "ids", True),
                                              ((128, 128, 128, 128), (16, 300, 5, 64), "hn", True)])
def test_loopback_random_weights_match_the_oracle(Bs, Ks, mode, bidir):
    from distributed_sigmoid_loss_b200 import _capi

    W, D = len(Bs), 72
    Ts = [b + k for b, k in zip(Bs, Ks)]
    tp, bias = math.log(10.0), -8.0
    imgs, texts, ids, eids = _problem(Bs, Ks, D, sum(Ts), mode)
    g = torch.Generator().manual_seed(W)
    iws, tws = [_random_weights(g, b) for b in Bs], [_random_weights(g, t) for t in Ts]
    ref = _oracle(imgs, texts, tp, bias, iws, tws, _labels(Bs, Ks, ids, eids, mode))
    for sched in ("fused", "split"):
        for r in range(W):
            eng = _engine(Bs[r], D, Bs=list(Bs), Ts=Ts, ids=mode != "pos", extra_ids=mode == "extra",
                          rank_world=(r, W), loopback=True)
            if bidir:
                eng.set_option(_capi.SIGLIP_OPT_BIDIR, 1)
            _loopback(eng, r, texts, ids, eids, tws)
            out = _step(eng, sched, imgs[r].to(_dev()), texts[r].to(_dev()), _scal(tp), _scal(bias), ids and ids[r],
                        eids and eids[r], iws[r], tws[r])
            torch.cuda.synchronize()
            _check_step(f"{sched} {mode} r{r}", out, ref[r], r, W)
            eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. clamping, CUDA graph, errors
# ---------------------------------------------------------------------------------------------------------------------
def test_out_of_range_weights_are_clamped():
    """-1, 2 and NaN behave as 0, 1 and 0: bit for bit the step with the clamped weights."""
    B, D = 300, 136
    (img,), (txt,), _, _ = _problem((B,), (0,), D, 9, "pos")
    g = torch.Generator().manual_seed(9)
    w = torch.rand(B, generator=g)
    raw, clamped = w.clone(), w.clone()
    for idx, v, c in ((slice(0, 300, 7), -1.0, 0.0), (slice(3, 300, 11), 2.0, 1.0), (slice(5, 300, 13), float("nan"), 0.0)):
        raw[idx], clamped[idx] = v, c
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    eng = _engine(B, D)
    for sched in ("fused", "split"):
        x = _step(eng, sched, img.to(_dev()), txt.to(_dev()), tp, b, iw=raw, tw=raw.flip(0))
        y = _step(eng, sched, img.to(_dev()), txt.to(_dev()), tp, b, iw=clamped, tw=clamped.flip(0))
        torch.cuda.synchronize()
        for i, (p, q) in enumerate(zip(x, y)):
            assert torch.equal(p, q), f"{sched}: output {i} differs"
        assert all(torch.isfinite(t).all() for t in x)
    eng.close()


def test_captured_step_follows_the_weight_buffers():
    B, D = 512, 128
    (img,), (txt,), _, _ = _problem((B,), (0,), D, 91, "pos")
    img, txt = img.to(_dev()), txt.to(_dev())
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    eng = _engine(B, D)
    iw_buf, tw_buf = torch.ones(B, device=_dev()), torch.ones(B, device=_dev())
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        eng.set_sample_weights(iw_buf, tw_buf)
        eng.fwd_bwd(img, txt, tp, b)
        with torch.cuda.graph(g, stream=side):
            eng.set_sample_weights(iw_buf, tw_buf)
            outs = eng.fwd_bwd(img, txt, tp, b)
    torch.cuda.current_stream().wait_stream(side)
    gen = torch.Generator().manual_seed(3)
    for _ in range(2):
        new_i, new_t = _random_weights(gen, B), _random_weights(gen, B)
        iw_buf.copy_(new_i.to(_dev()))
        tw_buf.copy_(new_t.to(_dev()))
        g.replay()
        torch.cuda.synchronize()
        replay = [x.clone() for x in outs]
        eager = _step(eng, "fused", img, txt, tp, b, iw=new_i, tw=new_t)
        torch.cuda.synchronize()
        for x, e in zip(replay, eager):
            assert torch.equal(x, e)
    del g
    eng.close()


def test_error_statuses():
    from distributed_sigmoid_loss_b200 import _capi

    B, D = 128, 64
    img = torch.zeros(B, D, dtype=torch.bfloat16, device=_dev())
    txt = torch.zeros(B, D, dtype=torch.bfloat16, device=_dev())
    tp, b = _scal(0.0), _scal(0.0)
    w = torch.ones(B, device=_dev())
    eng = _engine(B, D, weights=False)
    with pytest.raises(_capi.SiglipError) as e:            # the setter outside the mode
        eng.set_sample_weights(w, w)
    assert e.value.code == _capi.SIGLIP_ERR_STATE
    eng.set_option(_capi.SIGLIP_OPT_SAMPLE_WEIGHTS, 1)
    launches = eng.launch_count
    for call in (lambda: eng.fwd_bwd(img, txt, tp, b), lambda: eng.forward(img, txt, tp, b, True),
                 lambda: eng.fwd(img, txt, tp, b)):
        with pytest.raises(_capi.SiglipError) as e:        # a step without weights set since the previous step
            call()
        assert e.value.code == _capi.SIGLIP_ERR_STATE and "siglip_set_sample_weights" in str(e.value)
    assert eng.launch_count == launches
    eng.set_sample_weights(w, None)
    eng.set_option(_capi.SIGLIP_OPT_SAMPLE_WEIGHTS, 1)     # setting the option forgets the weights
    with pytest.raises(_capi.SiglipError) as e:
        eng.fwd(img, txt, tp, b)
    assert e.value.code == _capi.SIGLIP_ERR_STATE
    eng.set_sample_weights(None, w)
    eng.fwd(img, txt, tp, b)
    with pytest.raises(_capi.SiglipError) as e:            # consumed by that step
        eng.fwd(img, txt, tp, b)
    assert e.value.code == _capi.SIGLIP_ERR_STATE
    hb = torch.zeros(B, D, dtype=torch.bfloat16)
    with pytest.raises(_capi.SiglipError) as e:            # the host-buffer entries refuse the mode
        eng.fwd_bwd_host(hb, hb, 0.0, 0.0)
    assert e.value.code == _capi.SIGLIP_ERR_STATE
    with pytest.raises(RuntimeError, match="contiguous fp32"):
        eng.set_sample_weights(w.double(), None)
    eng.set_option(_capi.SIGLIP_OPT_SAMPLE_WEIGHTS, 0)
    eng.fwd(img, txt, tp, b)                                # no weights needed outside the mode
    torch.cuda.synchronize()
    eng.close()
    lb = _engine(B, D, Bs=[B, B], rank_world=(0, 2), loopback=True)
    with pytest.raises(_capi.SiglipError) as e:
        _capi.check(lb._L.siglip_debug_set_chunk_weights(lb._h, 2, None, lb._stream()))
    assert e.value.code == _capi.SIGLIP_ERR_INVALID
    lb.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. modules
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("inputs", ["bf16", "fp32", "normalize"])
def test_modules_match_the_oracle(inputs):
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    B, K, D = 256, 24, 96
    tp, bias = math.log(10.0), -10.0
    g = torch.Generator().manual_seed(17)
    img, txt, neg = torch.randn(B, D, generator=g), torch.randn(B, D, generator=g), torch.randn(K, D, generator=g)
    if inputs != "normalize":
        img, txt, neg = (torch.nn.functional.normalize(x) for x in (img, txt, neg))
    if inputs == "bf16":
        img, txt, neg = (x.to(torch.bfloat16) for x in (img, txt, neg))
    iw, tw = _random_weights(g, B), _random_weights(g, B + K)
    f = (lambda x: torch.nn.functional.normalize(x.double()) if inputs == "normalize" else x.double())  # noqa: E731
    ref = _oracle([f(img)], [torch.cat([f(txt), f(neg)])], tp, bias, [iw], [tw], label_blocks([B], [B + K]))[0]
    tol = 5e-3 if inputs == "bf16" else 2e-3
    for fused in (False, True):
        for kind in ("ddp", "siglip"):
            if kind == "siglip" and inputs == "normalize":
                continue
            leaves = [x.to(_dev()).requires_grad_(True) for x in (img, txt, neg)]
            kw = dict(negative_text=leaves[2], image_weights=iw.to(_dev()), text_weights=tw.to(_dev()))
            if kind == "ddp":
                mod = DDPSigmoidLoss(B, normalize_inputs=inputs == "normalize", fused_step=fused, hard_negatives=K,
                                     sample_weights=True).to(_dev())
                with torch.no_grad():
                    mod.t_prime.fill_(tp)
                    mod.bias.fill_(bias)
                loss, metrics = mod(leaves[0], leaves[1], return_metrics=True, **kw)
                sc = (mod.t_prime, mod.bias)
                plain = DDPSigmoidLoss(B, normalize_inputs=inputs == "normalize", fused_step=fused,
                                       hard_negatives=K).to(_dev())
                with torch.no_grad():
                    plain.t_prime.fill_(tp)
                    plain.bias.fill_(bias)
                _, m_plain = plain(leaves[0].detach(), leaves[1].detach(), negative_text=leaves[2].detach(),
                                   return_metrics=True)
            else:
                mod = SigLipLoss(fused_step=fused, hard_negatives=K, sample_weights=True)
                sc = (torch.tensor(tp, device=_dev(), requires_grad=True),
                      torch.tensor(bias, device=_dev(), requires_grad=True))
                loss, metrics = mod(leaves[0], leaves[1], sc[0], sc[1], return_metrics=True, **kw)
                _, m_plain = SigLipLoss(fused_step=fused, hard_negatives=K)(
                    leaves[0].detach(), leaves[1].detach(), sc[0].detach(), sc[1].detach(),
                    negative_text=leaves[2].detach(), return_metrics=True)
            loss.backward()
            torch.cuda.synchronize()
            tag = f"{kind} fused={fused} {inputs}"
            _check(f"{tag} loss", loss.detach(), ref["loss"], tol)
            _check(f"{tag} t_prime.grad", sc[0].grad, ref["dt_prime"], tol)
            _check(f"{tag} bias.grad", sc[1].grad, ref["dbias"], tol)
            if inputs != "normalize":   # the oracle's gradients are w.r.t. the normalised embeddings
                _check(f"{tag} img.grad", leaves[0].grad, ref["dimg"], tol)
                _check(f"{tag} txt.grad", leaves[1].grad, ref["contrib"][0][:B], tol)
                _check(f"{tag} negative_text.grad", leaves[2].grad, ref["contrib"][0][B:], tol)
            for k in metrics:                    # the retrieval metrics ignore the weights
                assert torch.equal(metrics[k], m_plain[k]), f"{tag}: metric {k} differs from the unweighted step"


def test_split_schedule_generation_guard_sets_the_weights_again():
    """Two forwards with different weights, then the backward of the FIRST: the re-run forward takes its weights."""
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss

    B, D = 256, 64
    tp, bias = math.log(10.0), -10.0
    (img,), (txt,), _, _ = _problem((B,), (0,), D, 77, "pos")
    g = torch.Generator().manual_seed(77)
    iw1, tw1 = _random_weights(g, B), _random_weights(g, B)
    ref1 = _oracle([img], [txt], tp, bias, [iw1], [tw1], label_blocks([B], [B]))[0]
    mod = DDPSigmoidLoss(B, fused_step=False, sample_weights=True).to(_dev())
    l1 = [x.float().to(_dev()).requires_grad_(True) for x in (img, txt)]
    l2 = [x.float().to(_dev()).requires_grad_(True) for x in (img, txt)]
    loss1 = mod(l1[0], l1[1], image_weights=iw1.to(_dev()), text_weights=tw1.to(_dev()))
    loss2 = mod(l2[0], l2[1], image_weights=None, text_weights=torch.rand(B, generator=g).to(_dev()))
    loss1.backward()
    torch.cuda.synchronize()
    assert float(loss1.detach()) != float(loss2.detach())
    _check("loss 1", loss1.detach(), ref1["loss"])
    _check("dimg 1", l1[0].grad, ref1["dimg"])
    _check("dtxt 1", l1[1].grad, ref1["contrib"][0])
