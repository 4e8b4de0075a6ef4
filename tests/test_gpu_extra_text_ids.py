"""Extra texts with ids (SIGLIP_OPT_EXTRA_TEXT_IDS, DDPSigmoidLoss(multi_positive=True, extra_texts=K)) on the H100:
several captions per image without repeating the image. Checked bit for bit against hard negatives + sample ids when
no extra id matches an image, against the float64 oracle (W = 1 and loopback W = 3 / W = 4 with cross-rank positives),
against multi_positive on repeated images through both modules, with the retrieval metrics, in a captured CUDA graph,
and for the error statuses."""
import math

import numpy as np
import pytest
import torch

from extra_text_ids_oracle import closed_form_extra_text_ids, retrieval_metrics_extra_text_ids
from retrieval_metrics_oracle import key_as_int64, metric_key

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


def _captions(Bs, M, D, seed, noise=0.5, extra_noise=0.3):
    """Per rank: images, their first captions (perturbed images) and M - 1 further captions each as extras (caption-major:
    extra m * B + i captions image i, with noise (m + 1) * extra_noise, so an image's captions are clearly ranked). With
    extra_noise < noise the first extra is the closest caption and wins i2t."""
    g = torch.Generator().manual_seed(seed)
    imgs, txts, extras = [], [], []
    for b in Bs:
        img = torch.nn.functional.normalize(torch.randn(b, D, generator=g))
        txt = torch.nn.functional.normalize(img + noise * torch.randn(b, D, generator=g) / math.sqrt(D))
        ext = torch.cat([torch.nn.functional.normalize(img + (m + 1) * extra_noise * torch.randn(b, D, generator=g) /
                                                       math.sqrt(D)) for m in range(M - 1)]) if M > 1 else torch.zeros(0, D)
        imgs.append(img.to(torch.bfloat16)), txts.append(txt.to(torch.bfloat16)), extras.append(ext.to(torch.bfloat16))
    return imgs, txts, extras


def _ids(Bs, M):
    """Sample ids 3 * global index; extra ids of rank r: its images' ids repeated M - 1 times."""
    ids = list(torch.split(torch.arange(sum(Bs), dtype=torch.int64) * 3, list(Bs)))
    return ids, [x.repeat(M - 1) for x in ids]


def _oracle(imgs, txts, extras, ids, eids, tp, bias):
    f = lambda xs: [x.float().numpy() for x in xs]  # noqa: E731
    return closed_form_extra_text_ids(f(imgs), f(txts), f(extras), [x.numpy() for x in ids],
                                      [x.numpy() for x in eids], tp, bias)


def _engine(B, T, D, cg=2, mcast=1, extra=True, Bs=None, Ts=None, **kw):
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi

    eng = SigmoidLossEngine(B, D, _dev(), cta_group=cg, batch_per_rank=Bs, texts_per_rank=Ts if Ts is not None else [T],
                            **kw)
    if mcast != 1:
        eng.set_option(_capi.SIGLIP_OPT_MCAST, mcast)
    eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 1)
    if extra:
        eng.set_option(_capi.SIGLIP_OPT_EXTRA_TEXT_IDS, 1)
    return eng


def _step(eng, sched, img, txt, tp, b, ids, eids, gdt=torch.float32):
    eng.set_sample_ids(ids.to(_dev()))
    if eng.extra_text_ids:
        eng.set_extra_text_ids(eids.to(_dev()))
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


def _loopback(eng, r, full, ids, eids, extra=True):
    for k in range(eng.world):
        eng.debug_set_text_chunk(k, full[k].to(_dev()))
        if k != r:
            eng.debug_set_chunk_ids(k, (torch.cat([ids[k], eids[k]]) if extra else ids[k]).to(_dev()))


CLUSTERS = [(1, 1), (2, 1), (2, 2)]


def _margin(S, axis):
    """Best minus second best similarity along `axis` (float64): the gap the kernel's fp32 ranking must not cross."""
    part = -np.partition(-S, 1, axis=axis)
    return np.take(part, 0, axis=axis) - np.take(part, 1, axis=axis)


def _check_index(what, got, want, margin, min_gap=1e-4):
    """Indices agree wherever the oracle's best beats its second best by more than fp32 rounding can move; nearly all
    rows qualify on these planted inputs."""
    got = got.cpu().numpy()
    ok = margin > min_gap
    assert ok.mean() > 0.95, f"{what}: only {ok.mean():.3f} of the rows have a clear best"
    bad = np.nonzero(ok & (got != want))[0]
    assert len(bad) == 0, f"{what}: {len(bad)} rows differ, first {bad[:5]}: got {got[bad[:5]]} want {want[bad[:5]]}"


def _hit_rate(index, row_ids, cand_ids):
    """The kernel's top-1 rate of a list of returned indices: integer hits over the count, in fp32."""
    index = index.cpu().numpy()
    return np.float32((cand_ids[index] == row_ids).sum()) / np.float32(len(index))


# ---------------------------------------------------------------------------------------------------------------------
# 1. extras whose ids match no image: bit for bit the step of hard negatives + sample ids (same slab classes)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cg,mcast", CLUSTERS)
@pytest.mark.parametrize("W", [1, 3])
def test_unmatched_extra_ids_are_bitwise_hard_negatives(W, cg, mcast):
    Bs, Ks, D = ((300,), (170,), 136) if W == 1 else ((96, 64, 80), (40, 0, 130), 72)
    Ts = [b + k for b, k in zip(Bs, Ks)]
    g = torch.Generator().manual_seed(W * 10 + cg + mcast)
    unit = lambda n: torch.nn.functional.normalize(torch.randn(n, D, generator=g)).to(torch.bfloat16)  # noqa: E731
    imgs, full = [unit(b) for b in Bs], [unit(t) for t in Ts]
    ids = list(torch.split(torch.randint(0, 40, (sum(Bs),), generator=g), list(Bs)))   # duplicates across ranks
    eids = [-1 - torch.arange(k, dtype=torch.int64) for k in Ks]                        # no image has a negative id
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    for r in range(W):
        kw = dict(rank_world=(r, W), loopback=True) if W > 1 else {}
        ext = _engine(Bs[r], Ts[r], D, cg, mcast, True, Bs=list(Bs), Ts=Ts, **kw)
        hn = _engine(Bs[r], Ts[r], D, cg, mcast, False, Bs=list(Bs), Ts=Ts, **kw)
        if W > 1:
            _loopback(ext, r, full, ids, eids, True)
            _loopback(hn, r, full, ids, eids, False)
        for sched in ("fused", "split", "fwd"):
            a = _step(ext, sched, imgs[r].to(_dev()), full[r].to(_dev()), tp, b, ids[r], eids[r])
            c = _step(hn, sched, imgs[r].to(_dev()), full[r].to(_dev()), tp, b, ids[r], eids[r])
            torch.cuda.synchronize()
            for i, (x, y) in enumerate(zip(a, c)):
                assert torch.equal(x, y), f"W={W} r={r} {sched}: output {i} differs from hard negatives + ids"
        ext.close()
        hn.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. one rank against the float64 oracle, several captions per image, planted so that extra captions win
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,M,D", [(300, 3, 136), (4096, 4, 768)])
@pytest.mark.parametrize("cg,mcast", CLUSTERS)
def test_single_rank_matches_the_oracle(B, M, D, cg, mcast):
    if B > 1000 and (cg, mcast) != (2, 1):
        pytest.skip("the large shape runs at the default cluster shape only")
    tp, bias = math.log(10.0), -10.0
    (img,), (txt,), (ext,) = _captions([B], M, D, B + M)
    ids, eids = _ids([B], M)
    ref = _oracle([img], [txt], [ext], ids, eids, tp, bias)[0]
    eng = _engine(B, M * B, D, cg, mcast)
    full = torch.cat([txt, ext]).to(_dev())
    for sched in ("fused", "split", "fwd"):
        out = _step(eng, sched, img.to(_dev()), full, _scal(tp), _scal(bias), ids[0], eids[0])
        torch.cuda.synchronize()
        _check_rank(f"{sched} B={B} M={M} cg={cg} mcast={mcast}", out, ref, ref["contrib"][0])
        if sched != "fwd":
            _check(f"{sched} dtxt of the extra captions", out[2][B:], ref["contrib"][0][B:])
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. loopback W-rank schedules: extras that caption images of other chunks, uneven batches and K
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Bs,Ks,bidir", [((160, 96, 130), (40, 0, 200), False),
                                         ((128, 128, 128, 128), (16, 300, 5, 64), True)])
def test_loopback_cross_rank_extra_captions(Bs, Ks, bidir):
    from distributed_sigmoid_loss_b200 import _capi

    W, D = len(Bs), 72
    tp, bias = math.log(10.0), -8.0
    g = torch.Generator().manual_seed(sum(Ks))
    unit = lambda n: torch.nn.functional.normalize(torch.randn(n, D, generator=g)).to(torch.bfloat16)  # noqa: E731
    imgs, txts = [unit(b) for b in Bs], [unit(b) for b in Bs]
    ids, _ = _ids(Bs, 1)
    # extra j of rank r: a caption of image j of rank r + 1 (a near copy of it, so the positive carries weight), every
    # third one an id that no image has
    extras, eids = [], []
    for r, k in enumerate(Ks):
        o = (r + 1) % W
        sel = torch.arange(k) % Bs[o]
        e = torch.nn.functional.normalize(imgs[o][sel].float() + 0.05 * torch.randn(k, D, generator=g))
        extras.append(e.to(torch.bfloat16))
        x = ids[o][sel].clone()
        x[::3] = 1 + 3 * torch.arange(len(x[::3]))
        eids.append(x)
    ref = _oracle(imgs, txts, extras, ids, eids, tp, bias)
    Ts = [b + k for b, k in zip(Bs, Ks)]
    full = [torch.cat([t, e]) for t, e in zip(txts, extras)]
    for sched in ("fused", "split"):
        dtxt_sum = [torch.zeros(t, D, device=_dev()) for t in Ts]
        for r in range(W):
            eng = _engine(Bs[r], Ts[r], D, rank_world=(r, W), loopback=True, Bs=list(Bs), Ts=Ts)
            if bidir:
                eng.set_option(_capi.SIGLIP_OPT_BIDIR, 1)
            _loopback(eng, r, full, ids, eids)
            out = _step(eng, sched, imgs[r].to(_dev()), full[r].to(_dev()), _scal(tp), _scal(bias), ids[r], eids[r])
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


# ---------------------------------------------------------------------------------------------------------------------
# 4. modules: extra_texts on B images == multi_positive on M·B repeated images
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("inputs", ["bf16", "fp32", "normalize"])
def test_modules_equal_repeated_images(inputs):
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    B, M, D = 256, 3, 96
    tp, bias = math.log(10.0), -10.0
    g = torch.Generator().manual_seed(71)
    img = torch.randn(B, D, generator=g)
    caps = [img + 0.5 * torch.randn(B, D, generator=g) for _ in range(M)]
    if inputs != "normalize":
        img, caps = torch.nn.functional.normalize(img), [torch.nn.functional.normalize(c) for c in caps]
    if inputs == "bf16":
        img, caps = img.to(torch.bfloat16), [c.to(torch.bfloat16) for c in caps]
    ids = torch.arange(B, dtype=torch.int64) * 5
    # bf16 leaves: both sides round their gradients to bf16 (2^-9), and the repeated side also sums its M bf16 copies
    tol = 8e-3 if inputs == "bf16" else TOL
    for fused in (False, True):
        for kind in ("ddp", "siglip"):
            if kind == "siglip" and inputs == "normalize":
                continue
            res = {}
            for mode in ("extra", "repeat"):
                a = img.to(_dev()).requires_grad_(True)
                t = torch.cat(caps).to(_dev()).requires_grad_(True)
                if mode == "extra":
                    kw = dict(sample_ids=ids.to(_dev()), extra_text=t[B:], extra_text_ids=ids.repeat(M - 1).to(_dev()))
                    x_img, x_txt, n = a, t[:B], B
                    mk = dict(multi_positive=True, extra_texts=(M - 1) * B)
                else:
                    kw = dict(sample_ids=ids.repeat(M).to(_dev()))
                    x_img, x_txt, n = a.repeat(M, 1), t, M * B
                    mk = dict(multi_positive=True)
                if kind == "ddp":
                    mod = DDPSigmoidLoss(n, normalize_inputs=(inputs == "normalize"), fused_step=fused, **mk).to(_dev())
                    with torch.no_grad():
                        mod.t_prime.fill_(tp)
                        mod.bias.fill_(bias)
                    loss = mod(x_img, x_txt, **kw)
                    sc = (mod.t_prime, mod.bias)
                else:
                    mod = SigLipLoss(fused_step=fused, **mk)
                    sc = (torch.tensor(tp, device=_dev(), requires_grad=True),
                          torch.tensor(bias, device=_dev(), requires_grad=True))
                    loss = mod(x_img, x_txt, sc[0], sc[1], **kw)
                loss.backward()
                torch.cuda.synchronize()
                res[mode] = (loss.detach().float(), a.grad.float(), t.grad.float(), sc[0].grad.float(), sc[1].grad.float())
            tag = f"{kind} fused={fused} {inputs}"
            for i, name in enumerate(("loss", "img.grad (summed over copies)", "txt.grad", "dt_prime", "dbias")):
                _check(f"{tag} {name}", res["extra"][i], res["repeat"][i], tol)


def test_split_schedule_generation_guard_sets_both_id_buffers():
    """Two forwards with different ids, then the backward of the FIRST: the re-run forward takes the first call's
    sample ids and extra ids again."""
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss

    B, M, D = 256, 3, 64
    tp, bias = math.log(10.0), -10.0
    (img,), (txt,), (ext,) = _captions([B], M, D, 77)
    ids, eids = _ids([B], M)
    ids2, eids2 = ids[0] + 1, -eids[0] - 1            # second call: no extra matches an image
    ref1 = _oracle([img], [txt], [ext], ids, eids, tp, bias)[0]
    mod = DDPSigmoidLoss(B, fused_step=False, multi_positive=True, extra_texts=(M - 1) * B).to(_dev())
    leaves1 = [x.float().to(_dev()).requires_grad_(True) for x in (img, txt, ext)]
    leaves2 = [x.float().to(_dev()).requires_grad_(True) for x in (img, txt, ext)]
    l1 = mod(leaves1[0], leaves1[1], sample_ids=ids[0].to(_dev()), extra_text=leaves1[2],
             extra_text_ids=eids[0].to(_dev()))
    l2 = mod(leaves2[0], leaves2[1], sample_ids=ids2.to(_dev()), extra_text=leaves2[2], extra_text_ids=eids2.to(_dev()))
    l1.backward()
    torch.cuda.synchronize()
    assert float(l1) != float(l2)
    _check("loss 1", l1.detach(), ref1["loss"])
    _check("dimg 1", leaves1[0].grad, ref1["dimg"])
    _check("extra_text.grad 1", leaves1[2].grad, ref1["contrib"][0][B:])


# ---------------------------------------------------------------------------------------------------------------------
# 5. retrieval metrics
# ---------------------------------------------------------------------------------------------------------------------
def _arm(eng, B, T):
    top1 = torch.empty(2, device=_dev())
    i2t = torch.empty(B, device=_dev(), dtype=torch.int64)
    t2i = torch.empty(T, device=_dev(), dtype=torch.int64)
    eng.request_metrics(top1, i2t, t2i)
    return top1, i2t, t2i


@pytest.mark.parametrize("B,M,D", [(300, 3, 136), (4096, 4, 768)])
def test_metrics_winning_extra_caption_is_a_hit(B, M, D):
    """The extras are the closer captions: most images rank one of them first, a hit. A quarter of the extras carry an
    id that no image has: where one wins i2t it is a miss, and as a text it is always a t2i miss."""
    (img,), (txt,), (ext,) = _captions([B], M, D, B + 1, noise=1.0, extra_noise=0.2)
    ids, eids = _ids([B], M)
    eids[0][::4] = -7 - torch.arange(len(eids[0][::4]))
    res = retrieval_metrics_extra_text_ids([img.float().numpy()], [txt.float().numpy()], [ext.float().numpy()],
                                           [ids[0].numpy()], [eids[0].numpy()])[0]
    extra_wins = res["i2t_index"] >= B
    assert extra_wins.mean() > 0.5 and 0.0 < res["i2t_top1"] < 1.0          # the plant: extras win, some are misses
    T = M * B
    tid = np.concatenate([ids[0].numpy(), eids[0].numpy()])
    eng, plain = _engine(B, T, D), _engine(B, T, D)
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    full, im = torch.cat([txt, ext]).to(_dev()), img.to(_dev())
    for sched in ("fused", "split", "fwd"):
        top1, i2t, t2i = _arm(eng, B, T)
        armed = _step(eng, sched, im, full, tp, b, ids[0], eids[0])
        unarmed = _step(plain, sched, im, full, tp, b, ids[0], eids[0])
        torch.cuda.synchronize()
        for i, (x, y) in enumerate(zip(armed, unarmed)):
            assert torch.equal(x, y), f"{sched}: output {i} of the armed step differs"
        _check_index(f"{sched} i2t", i2t, res["i2t_index"], _margin(res["S"], 1))
        _check_index(f"{sched} t2i", t2i, res["t2i_index"], _margin(res["S"], 0))
        assert float(top1[0]) == _hit_rate(i2t, ids[0].numpy(), tid), sched
        assert float(top1[1]) == _hit_rate(t2i, tid, ids[0].numpy()), sched
        assert abs(float(top1[0]) - res["i2t_top1"]) < 0.01 and abs(float(top1[1]) - res["t2i_top1"]) < 0.01, sched
        n_neg = len(eids[0][::4])
        assert float(top1[1]) <= (T - n_neg) / T + 1e-6                      # every pure negative is a t2i miss
    eng.close()
    plain.close()


def test_metrics_loopback_t2i_over_every_text_with_seeded_peer_keys():
    """W = 3 loopback, uneven: t2i_index is [T_r] and combines this rank's column partials with seeded stand-ins for the
    peers' (keys of their best images from the oracle, some raised above any real similarity)."""
    Bs, M, D = (96, 64, 80), 2, 128
    imgs, txts, extras = _captions(Bs, M, D, 5, noise=0.6, extra_noise=0.2)
    ids, eids = _ids(Bs, M)
    eids[1][:10] = ids[0][:10]                         # rank 1's first extras caption rank 0's images
    extras[1][:10] = torch.nn.functional.normalize(imgs[0][:10].float() + 0.01).to(torch.bfloat16)
    f = lambda xs: [x.float().numpy() for x in xs]  # noqa: E731
    res = retrieval_metrics_extra_text_ids(f(imgs), f(txts), f(extras), [x.numpy() for x in ids],
                                           [x.numpy() for x in eids])
    Ts = [b * M for b in Bs]
    full = [torch.cat([t, e]) for t, e in zip(txts, extras)]
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    for r in range(3):
        eng = _engine(Bs[r], Ts[r], D, rank_world=(r, 3), loopback=True, Bs=list(Bs), Ts=Ts)
        _loopback(eng, r, full, ids, eids)
        S, off, toff = res[r]["S"], res[r]["off"], res[r]["toff"]
        want = res[r]["t2i_index"].copy()
        for p in range(3):
            if p == r:
                continue
            blk = S[off[p]:off[p + 1], toff[r]:toff[r + 1]]
            best = np.argmax(blk, axis=0)
            keys = [metric_key(np.float32(blk[best[j], j]), off[p] + best[j]) for j in range(Ts[r])]
            for j in range(p, Ts[r], 7):                # this peer's image j % B_p beats every real candidate
                keys[j] = metric_key(np.float32(1e4), off[p] + j % Bs[p])
                want[j] = off[p] + j % Bs[p]
            eng.debug_set_peer_metric_keys(p, torch.tensor([key_as_int64(k) for k in keys], dtype=torch.int64,
                                                           device=_dev()))
        top1, i2t, t2i = _arm(eng, Bs[r], Ts[r])
        _step(eng, "fused", imgs[r].to(_dev()), full[r].to(_dev()), tp, b, ids[r], eids[r])
        torch.cuda.synchronize()
        gid = np.concatenate([x.numpy() for x in ids])
        tid = np.concatenate([x.numpy() for pair in zip(ids, eids) for x in pair])
        mine = np.concatenate([ids[r].numpy(), eids[r].numpy()])
        _check_index(f"r{r} i2t", i2t, res[r]["i2t_index"], _margin(S[off[r]:off[r + 1]], 1))
        t_margin = _margin(S[:, toff[r]:toff[r + 1]], 0)
        t_margin[want != res[r]["t2i_index"]] = np.inf      # a raised key wins by far
        _check_index(f"r{r} t2i", t2i, want, t_margin)
        assert float(top1[0]) == _hit_rate(i2t, ids[r].numpy(), tid), r
        assert float(top1[1]) == _hit_rate(t2i, mine, gid), r
        eng.close()
    assert (res[0]["i2t_index"][:10] >= Ts[0] + Bs[1]).all()     # rank 0's images chose rank 1's extras: hits
    assert res[0]["i2t_top1"] > 0.9


# ---------------------------------------------------------------------------------------------------------------------
# 6. CUDA graph, errors
# ---------------------------------------------------------------------------------------------------------------------
def test_captured_step_follows_both_id_buffers():
    B, M, D = 512, 2, 128
    (img,), (txt,), (ext,) = _captions([B], M, D, 91)
    img, full = img.to(_dev()), torch.cat([txt, ext]).to(_dev())
    ids, eids = _ids([B], M)
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    eng = _engine(B, M * B, D)
    ids_buf, eids_buf = ids[0].to(_dev()), eids[0].to(_dev())
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        eng.set_sample_ids(ids_buf)
        eng.set_extra_text_ids(eids_buf)
        eng.fwd_bwd(img, full, tp, b)
        with torch.cuda.graph(g, stream=side):
            eng.set_sample_ids(ids_buf)
            eng.set_extra_text_ids(eids_buf)
            outs = eng.fwd_bwd(img, full, tp, b)
    torch.cuda.current_stream().wait_stream(side)
    # new contents of both buffers: no extra matches, then every extra matches the image of the next row
    for new_ids, new_eids in ((ids[0], -1 - eids[0]), (ids[0] + 1, torch.roll(ids[0] + 1, 1).repeat(M - 1))):
        ids_buf.copy_(new_ids.to(_dev()))
        eids_buf.copy_(new_eids.to(_dev()))
        g.replay()
        torch.cuda.synchronize()
        replay = [x.clone() for x in outs]
        eager = _step(eng, "fused", img, full, tp, b, new_ids, new_eids)
        torch.cuda.synchronize()
        for x, e in zip(replay, eager):
            assert torch.equal(x, e)
    del g
    eng.close()


def test_error_statuses():
    from distributed_sigmoid_loss_b200 import _capi

    B, K, D = 128, 64, 64
    img = torch.zeros(B, D, dtype=torch.bfloat16, device=_dev())
    txt = torch.zeros(B + K, D, dtype=torch.bfloat16, device=_dev())
    tp, b = _scal(0.0), _scal(0.0)
    ids, eids = torch.arange(B, device=_dev()), torch.arange(K, device=_dev())
    eng = _engine(B, B + K, D, extra=False)
    eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 0)
    with pytest.raises(_capi.SiglipError) as e:            # the option needs the sample ids on
        eng.set_option(_capi.SIGLIP_OPT_EXTRA_TEXT_IDS, 1)
    assert e.value.code == _capi.SIGLIP_ERR_STATE and not eng.extra_text_ids
    eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 1)
    with pytest.raises(_capi.SiglipError) as e:            # the setter outside the mode
        eng.set_extra_text_ids(eids)
    assert e.value.code == _capi.SIGLIP_ERR_STATE
    eng.set_option(_capi.SIGLIP_OPT_EXTRA_TEXT_IDS, 1)
    launches = eng.launch_count
    for call in (lambda: eng.fwd_bwd(img, txt, tp, b), lambda: eng.forward(img, txt, tp, b, True),
                 lambda: eng.fwd(img, txt, tp, b)):
        eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 1)      # setting the option forgets both id buffers
        eng.set_sample_ids(ids)                             # sample ids without extra ids
        with pytest.raises(_capi.SiglipError) as e:
            call()
        assert e.value.code == _capi.SIGLIP_ERR_STATE and "siglip_set_extra_text_ids" in str(e.value)
        eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 1)
        assert eng.extra_text_ids
        eng.set_extra_text_ids(eids)                        # extra ids without sample ids
        with pytest.raises(_capi.SiglipError) as e:
            call()
        assert e.value.code == _capi.SIGLIP_ERR_STATE and "siglip_set_sample_ids" in str(e.value)
    assert eng.launch_count == launches
    eng.set_sample_ids(ids)
    eng.set_extra_text_ids(eids)
    eng.fwd(img, txt, tp, b)
    torch.cuda.synchronize()
    assert eng.launch_count > launches
    eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 0)         # clears the extras' ids too
    assert not eng.extra_text_ids
    with pytest.raises(_capi.SiglipError) as e:
        eng.set_extra_text_ids(eids)
    assert e.value.code == _capi.SIGLIP_ERR_STATE
    eng.fwd(img, txt, tp, b)                                # plain labels again: no ids needed
    torch.cuda.synchronize()
    eng.close()
    # accepted with T == B, where it changes nothing
    same = _engine(B, B, D)
    same.set_sample_ids(ids)
    same.set_extra_text_ids(eids[:0])
    same.fwd(img, txt[:B], tp, b)
    torch.cuda.synchronize()
    same.close()
