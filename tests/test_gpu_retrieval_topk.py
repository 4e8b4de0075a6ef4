"""Top-K in-batch retrieval (siglip_request_topk, return_metrics=True with metrics_topk=K) on the H100.

Planted data: every embedding is a small-integer vector / 8, so that the bf16 operands are exact and every logit is an
exact fp32 number: the kernel's accumulator then equals the float64 oracle of tests/retrieval_topk_oracle.py, and the
lists (ties to the lower index included) and recall@k are compared exactly. Captions are noisy copies of their image,
so a positive is often, but not always, first. Covered: one rank at (300, 136) and (4096, 768); loopback W = 3 with
seeded peer lists, uneven batches and bidir; ids with duplicates; COCO-style 5 captions per image through extra_texts
under torch.no_grad(); extra images with ids; loss and gradients bit-identical to the unarmed step; recall[0] and
column 0 against the top-1 metrics bit for bit; K = 5 a prefix of K = 10; the same bits across cluster shapes, stage
counts, schedules and row panels; no stale lists across steps; CUDA-graph replay with the first request inside the
capture; the modules with bf16, fp32 and normalize_inputs; the error statuses."""
import ctypes
import math

import numpy as np
import pytest
import torch

from retrieval_metrics_oracle import key_as_int64, metric_key
from retrieval_topk_oracle import recall_counts, topk_retrieval

pytestmark = pytest.mark.gpu

TP, BIAS = math.log(10.0), -10.0
KMAX = 10


def _dev():
    return torch.device("cuda", 0)


def _scal(x):
    return torch.tensor([x], device=_dev(), dtype=torch.float32)


def _grid(g, n, D):
    return g.integers(-2, 3, (n, D)).astype(np.float64)


def _planted(seed, Bs, Rs, Ts, D):
    """Per rank: R images (B paired, then extras near a paired image), T texts (B captions near their image, then
    extras near a random paired image). Integers / 8: exact in bf16."""
    g = np.random.default_rng(seed)
    imgs, txts = [], []
    for b, r, t in zip(Bs, Rs, Ts):
        base = _grid(g, b, D)
        noise = lambda n: g.choice([-1, 0, 1], (n, D), p=[0.3, 0.4, 0.3])  # noqa: E731
        xi = base[np.arange(r - b) % b] + noise(r - b)
        cap = base + noise(b)
        xt = base[g.integers(0, b, t - b)] + noise(t - b)
        imgs.append(torch.from_numpy(np.concatenate([base, xi]) / 8).to(torch.bfloat16))
        txts.append(torch.from_numpy(np.concatenate([cap, xt]) / 8).to(torch.bfloat16))
    return imgs, txts


def _engine(r, Bs, Rs, Ts, D, cg=2, mcast=1, ids=False, ximg_ids=False, xtxt_ids=False):
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi

    W = len(Bs)
    eng = SigmoidLossEngine(Bs[r], D, _dev(), cta_group=cg, rank_world=(r, W), loopback=W > 1, batch_per_rank=Bs,
                            texts_per_rank=Ts, images_per_rank=Rs)
    if mcast != 1:
        eng.set_option(_capi.SIGLIP_OPT_MCAST, mcast)
    for on, opt in ((ids, _capi.SIGLIP_OPT_SAMPLE_IDS), (xtxt_ids, _capi.SIGLIP_OPT_EXTRA_TEXT_IDS),
                    (ximg_ids, _capi.SIGLIP_OPT_EXTRA_IMAGE_IDS)):
        if on:
            eng.set_option(opt, 1)
    return eng


def _prepare(eng, r, txts, ids=None, xt=None, xi=None):
    dev = _dev()
    if eng.world > 1:
        for k in range(eng.world):
            eng.debug_set_text_chunk(k, txts[k].to(dev))
            if k != r and ids is not None:
                cid = np.concatenate([ids[k], xt[k]]) if eng.extra_text_ids else ids[k]
                eng.debug_set_chunk_ids(k, torch.from_numpy(cid).to(dev))
    if ids is not None:
        eng.set_sample_ids(torch.from_numpy(ids[r]).to(dev))
        if eng.extra_text_ids:
            eng.set_extra_text_ids(torch.from_numpy(xt[r]).to(dev))
        if eng.extra_image_ids:
            eng.set_extra_image_ids(torch.from_numpy(xi[r]).to(dev))


def _tbufs(eng, k):
    return (torch.full((2 * k,), -1.0, device=_dev()),
            torch.full((eng.metric_images, k), -7, device=_dev(), dtype=torch.int64),
            torch.full((eng.metric_texts, k), -7, device=_dev(), dtype=torch.int64))


def _mbufs(eng):
    return (torch.full((2,), -1.0, device=_dev()), torch.full((eng.metric_images,), -7, device=_dev(), dtype=torch.int64),
            torch.full((eng.metric_texts,), -7, device=_dev(), dtype=torch.int64))


def _step(eng, sched, img, txt, topk=None, metrics=None):
    tp, b = _scal(TP), _scal(BIAS)
    if metrics is not None:
        eng.request_metrics(*metrics)
    if topk is not None:
        eng.request_topk(*topk)
    if sched == "fused":
        outs = list(eng.fwd_bwd(img, txt, tp, b, torch.float32))
    elif sched == "split":
        outs = [eng.forward(img, txt, tp, b, True)] + list(eng.backward(img, txt, tp, None, torch.float32))
    else:
        outs = [eng.fwd(img, txt, tp, b)]
    return [x.clone() for x in outs]


def _check(tag, k, bufs, ref):
    recall, i2t, t2i = (x.cpu() for x in bufs)
    assert np.array_equal(i2t.numpy(), ref["i2t_topk"]), f"{tag}: i2t lists differ from the oracle"
    assert np.array_equal(t2i.numpy(), ref["t2i_topk"]), f"{tag}: t2i lists differ from the oracle"
    want = np.concatenate([recall_counts(ref["i2t_first"], k), recall_counts(ref["t2i_first"], k)])
    assert np.array_equal(recall.numpy(), want), f"{tag}: recall {recall.numpy()} vs {want}"


def _oracle(imgs, txts, Bs, k, **kw):
    return topk_retrieval([x.double().numpy() for x in imgs], [x.double().numpy() for x in txts], Bs, k, **kw)


# ---------------------------------------------------------------------------------------------------------------------
# 1. one rank against the oracle; arming changes no bit of the step; the top-1 outputs are columns / entries 0
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,D,sched,k", [(300, 136, "fused", 5), (300, 136, "split", 10), (300, 136, "fwd", 2),
                                         (4096, 768, "fused", 10)])
def test_single_rank_matches_oracle_and_changes_no_bit(B, D, sched, k):
    imgs, txts = _planted(B + D, (B,), (B,), (B,), D)
    img, txt = imgs[0].to(_dev()), txts[0].to(_dev())
    plain, armed = _engine(0, (B,), (B,), (B,), D), _engine(0, (B,), (B,), (B,), D)
    a = _step(plain, sched, img, txt)
    m = _mbufs(armed)
    bufs = _tbufs(armed, k)
    c = _step(armed, sched, img, txt, topk=(k, *bufs), metrics=m)
    torch.cuda.synchronize()
    for x, y in zip(a, c):
        assert torch.equal(x, y), f"{sched}: the armed step differs from the plain one"
    _check(f"W=1 B={B} D={D} {sched} K={k}", k, bufs, _oracle(imgs, txts, (B,), k)[0])
    recall, i2t, t2i = bufs
    assert torch.equal(recall[0], m[0][0]) and torch.equal(recall[k], m[0][1]), "recall@1 is not the top-1 rate"
    assert torch.equal(i2t[:, 0], m[1]) and torch.equal(t2i[:, 0], m[2]), "column 0 is not the top-1 index"
    plain.close()
    armed.close()


def test_k1_is_the_metrics_path_and_k5_a_prefix_of_k10():
    B, D = 300, 136
    imgs, txts = _planted(5, (B,), (B,), (B,), D)
    img, txt = imgs[0].to(_dev()), txts[0].to(_dev())
    eng = _engine(0, (B,), (B,), (B,), D)
    m = _mbufs(eng)
    b1 = _tbufs(eng, 1)
    n = eng.launch_count
    _step(eng, "fused", img, txt, metrics=m)
    plain_metrics = eng.launch_count - n
    n = eng.launch_count
    _step(eng, "fused", img, txt, topk=(1, *b1))
    assert eng.launch_count - n == plain_metrics   # K = 1: the metrics kernels, nothing else
    assert torch.equal(b1[0], m[0]) and torch.equal(b1[1][:, 0], m[1]) and torch.equal(b1[2][:, 0], m[2])
    b5, b10 = _tbufs(eng, 5), _tbufs(eng, 10)
    _step(eng, "fused", img, txt, topk=(5, *b5))
    _step(eng, "fused", img, txt, topk=(10, *b10))
    torch.cuda.synchronize()
    assert torch.equal(b5[1], b10[1][:, :5]) and torch.equal(b5[2], b10[2][:, :5])
    assert torch.equal(b5[0][:5], b10[0][:5]) and torch.equal(b5[0][5:], b10[0][10:15])
    eng.close()


def test_ids_with_duplicates():
    B, D, k = 300, 136, 5
    imgs, txts = _planted(17, (B,), (B,), (B,), D)
    ids = [np.random.default_rng(17).integers(0, B // 3, B).astype(np.int64)]
    eng = _engine(0, (B,), (B,), (B,), D, ids=True)
    _prepare(eng, 0, txts, ids)
    bufs = _tbufs(eng, k)
    _step(eng, "fused", imgs[0].to(_dev()), txts[0].to(_dev()), topk=(k, *bufs))
    torch.cuda.synchronize()
    _check("ids with duplicates", k, bufs, _oracle(imgs, txts, (B,), k, img_ids=ids, txt_ids=ids)[0])
    eng.close()


def test_extra_images_with_ids():
    Bs, Rs, Ts, D, k = (300,), (420,), (340,), 136, 10
    imgs, txts = _planted(23, Bs, Rs, Ts, D)
    rng = np.random.default_rng(23)
    ids = [np.arange(300, dtype=np.int64) * 3]
    xt = [rng.choice(ids[0], 40).astype(np.int64)]
    xi = [np.where(rng.random(120) < 0.8, ids[0][np.arange(120) % 300], 7_000_001 + np.arange(120)).astype(np.int64)]
    eng = _engine(0, Bs, Rs, Ts, D, ids=True, xtxt_ids=True, ximg_ids=True)
    _prepare(eng, 0, txts, ids, xt, xi)
    bufs = _tbufs(eng, k)
    _step(eng, "split", imgs[0].to(_dev()), txts[0].to(_dev()), topk=(k, *bufs))
    torch.cuda.synchronize()
    ref = _oracle(imgs, txts, Bs, k, img_ids=[np.concatenate([ids[0], xi[0]])],
                  txt_ids=[np.concatenate([ids[0], xt[0]])], rank_all_images=True, rank_all_texts=True)[0]
    _check("extra images with ids", k, bufs, ref)
    eng.close()


def test_coco_style_five_captions_under_no_grad():
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss

    B, D, k = 512, 136, 10
    g = np.random.default_rng(31)
    base = _grid(g, B, D)
    caps = [base + g.choice([-1, 0, 1], (B, D), p=[0.35, 0.3, 0.35]) for _ in range(5)]
    img = torch.from_numpy(base / 8).to(torch.bfloat16)
    txt = torch.from_numpy(caps[0] / 8).to(torch.bfloat16)
    extra = torch.from_numpy(np.concatenate(caps[1:]) / 8).to(torch.bfloat16)
    ids = torch.arange(B, dtype=torch.int64)
    xids = ids.repeat(4)
    mod = DDPSigmoidLoss(B, multi_positive=True, extra_texts=4 * B).to(_dev())
    with torch.no_grad():
        loss, met = mod(img.to(_dev()), txt.to(_dev()), sample_ids=ids.to(_dev()), extra_text=extra.to(_dev()),
                        extra_text_ids=xids.to(_dev()), return_metrics=True, metrics_topk=k)
    torch.cuda.synchronize()
    assert met["i2t_topk"].shape == (B, k) and met["t2i_topk"].shape == (5 * B, k)
    assert met["i2t_recall"].shape == (k,) and met["i2t_recall"].dtype == torch.float32
    ref = _oracle([img], [torch.cat([txt, extra])], (B,), k, img_ids=[ids.numpy()], txt_ids=[torch.cat([ids, xids]).numpy()],
                  rank_all_texts=True)[0]
    _check("COCO-style", k, (torch.cat([met["i2t_recall"], met["t2i_recall"]]), met["i2t_topk"], met["t2i_topk"]), ref)
    r = met["i2t_recall"].cpu()
    print(f"COCO-style i2t R@1 {r[0]:.3f} R@5 {r[4]:.3f} R@10 {r[9]:.3f}")
    assert torch.equal(met["i2t_recall"][0], met["i2t_top1"]) and torch.equal(met["t2i_recall"][0], met["t2i_top1"])


# ---------------------------------------------------------------------------------------------------------------------
# 2. loopback W = 3 with seeded peer lists
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Bs,r,bidir,sched", [((300, 200, 264), 1, False, "fused"), ((300, 200, 264), 0, True, "fwd"),
                                              ((128, 256, 200), 2, True, "fused")])
def test_loopback_with_seeded_peer_lists(Bs, r, bidir, sched):
    from distributed_sigmoid_loss_b200 import _capi

    D, k = 136, 10
    imgs, txts = _planted(len(Bs) * 13 + r, Bs, Bs, Bs, D)
    eng = _engine(r, Bs, Bs, Bs, D)
    if bidir:
        eng.set_option(_capi.SIGLIP_OPT_BIDIR, 1)
    _prepare(eng, r, txts)
    ref = _oracle(imgs, txts, Bs, k)
    S, off, toff = ref[r]["S"], ref[r]["off"], ref[r]["toff"]
    for p in range(len(Bs)):
        if p == r:
            continue
        keys = np.zeros((Bs[r], KMAX), np.int64)
        for j in range(Bs[r]):
            col = S[off[p]:off[p + 1], toff[r] + j]
            order = np.lexsort((np.arange(len(col)), -col))[:KMAX]
            keys[j, :len(order)] = [key_as_int64(metric_key(col[i], off[p] + i)) for i in order]
        eng.debug_set_peer_topk_keys(p, torch.from_numpy(keys).to(_dev()))
    bufs = _tbufs(eng, k)
    _step(eng, sched, imgs[r].to(_dev()), txts[r].to(_dev()), topk=(k, *bufs))
    torch.cuda.synchronize()
    _check(f"loopback W={len(Bs)} r={r} bidir={bidir} {sched}", k, bufs, ref[r])
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. the same bits across configurations and repeated steps; no stale lists
# ---------------------------------------------------------------------------------------------------------------------
def test_bitwise_reproducible_across_configurations():
    from distributed_sigmoid_loss_b200 import _capi

    B, D, k = 2048, 136, 10
    imgs, txts = _planted(41, (B,), (B,), (B,), D)
    img, txt = imgs[0].to(_dev()), txts[0].to(_dev())
    first = None
    for cg, mcast, stages, budget in [(2, 1, 0, 0), (1, 1, 0, 0), (2, 2, 0, 0), (1, 2, 4, 0), (2, 1, 4, 0),
                                      (2, 1, 0, 2), (1, 1, 4, 2)]:
        eng = _engine(0, (B,), (B,), (B,), D, cg=cg, mcast=mcast)
        if stages:
            eng.set_option(_capi.SIGLIP_OPT_STAGES_LOSS, stages)
        if budget:
            eng.set_sigma_budget(budget << 20)
        for sched in (("fused", "fwd") if budget else ("fused", "split", "fwd")):
            for with_losses in (False, True):
                for rep in range(2):
                    bufs = _tbufs(eng, k)
                    if with_losses:
                        eng.request_sample_losses(torch.empty(B, device=_dev()), torch.empty(B, device=_dev()))
                    _step(eng, sched, img, txt, topk=(k, *bufs))
                    torch.cuda.synchronize()
                    if first is None:
                        first = [x.clone() for x in bufs]
                        _check("reference configuration", k, bufs, _oracle(imgs, txts, (B,), k)[0])
                    tag = f"cg={cg} mcast={mcast} stages={stages} budget={budget} {sched} losses={with_losses} rep={rep}"
                    for x, y in zip(bufs, first):
                        assert torch.equal(x, y), f"{tag}: differs from the first configuration"
        eng.close()


def test_no_stale_lists_across_steps():
    B, D, k = 300, 136, 10
    eng = _engine(0, (B,), (B,), (B,), D)
    for seed in (51, 52, 53):
        imgs, txts = _planted(seed, (B,), (B,), (B,), D)
        bufs = _tbufs(eng, k)
        _step(eng, "fused", imgs[0].to(_dev()), txts[0].to(_dev()), topk=(k, *bufs))
        _step(eng, "fused", imgs[0].to(_dev()), txts[0].to(_dev()))   # unarmed steps in between
        torch.cuda.synchronize()
        _check(f"step seed={seed}", k, bufs, _oracle(imgs, txts, (B,), k)[0])
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. capture, the modules, errors
# ---------------------------------------------------------------------------------------------------------------------
def test_first_request_inside_a_capture_allocates_the_workspace():
    B, D, k = 256, 128, 5
    eng = _engine(0, (B,), (B,), (B,), D)
    imgs, txts = _planted(61, (B,), (B,), (B,), D)
    img, txt = imgs[0].to(_dev()).clone(), txts[0].to(_dev()).clone()
    tp, b = _scal(TP), _scal(BIAS)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eng.fwd_bwd(img, txt, tp, b, torch.float32)
        torch.cuda.synchronize()
        ws = eng.workspace_bytes
        bufs = _tbufs(eng, k)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            eng.request_topk(k, *bufs)
            eng.fwd_bwd(img, txt, tp, b, torch.float32)
    assert eng.workspace_bytes == ws + 2 * (B + B) * KMAX * 8
    for seed in (62, 63):
        i1, t1 = _planted(seed, (B,), (B,), (B,), D)
        img.copy_(i1[0].to(_dev()))
        txt.copy_(t1[0].to(_dev()))
        graph.replay()
        torch.cuda.synchronize()
        _check(f"graph replay {seed}", k, bufs, _oracle(i1, t1, (B,), k)[0])
    eng.close()


@pytest.mark.parametrize("fp32,normalize", [(False, False), (True, False), (True, True), (False, True)])
def test_modules_return_topk(fp32, normalize):
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    B, D, k = 300, 136, 5
    imgs, txts = _planted(71, (B,), (B,), (B,), D)
    dt = torch.float32 if fp32 else torch.bfloat16
    a = imgs[0].to(dt).to(_dev()).requires_grad_(True)
    t = txts[0].to(dt).to(_dev()).requires_grad_(True)
    mod = DDPSigmoidLoss(B, normalize_inputs=normalize).to(_dev())
    loss0, m0 = mod(a, t, return_metrics=True)
    assert set(m0) == {"i2t_top1", "t2i_top1", "i2t_index", "t2i_index"}
    g0 = torch.autograd.grad(loss0, [a, t])
    loss, met = mod(a, t, return_metrics=True, metrics_topk=k)
    g1 = torch.autograd.grad(loss, [a, t])
    assert torch.equal(loss, loss0) and all(torch.equal(x, y) for x, y in zip(g0, g1))
    assert set(met) == set(m0) | {"i2t_topk", "t2i_topk", "i2t_recall", "t2i_recall"}
    assert met["i2t_topk"].shape == (B, k) and met["i2t_topk"].dtype == torch.int64
    for key in m0:
        assert torch.equal(met[key], m0[key]), key
    assert torch.equal(met["i2t_topk"][:, 0], met["i2t_index"]) and torch.equal(met["i2t_recall"][0], met["i2t_top1"])
    assert torch.equal(met["t2i_topk"][:, 0], met["t2i_index"]) and torch.equal(met["t2i_recall"][0], met["t2i_top1"])
    if not normalize:   # exact operands (bf16 values; fp32 inputs become fp16 x 16, also exact here)
        _check(f"module fp32={fp32}", k, (torch.cat([met["i2t_recall"], met["t2i_recall"]]), met["i2t_topk"],
                                          met["t2i_topk"]), _oracle(imgs, txts, (B,), k)[0])
        with torch.no_grad():
            _, m2 = SigLipLoss()(a.detach(), t.detach(), torch.tensor(TP, device=_dev()),
                                 torch.tensor(BIAS, device=_dev()), return_metrics=True, metrics_topk=k)
        assert torch.equal(m2["i2t_topk"], met["i2t_topk"]) and torch.equal(m2["t2i_recall"], met["t2i_recall"])
    with pytest.raises(RuntimeError, match="metrics_topk"):
        mod(a, t, return_metrics=True, metrics_topk=0)


def test_error_statuses():
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi

    B, D = 64, 64
    L = _capi.lib()
    eng = _engine(0, (B,), (B,), (B,), D)
    recall, i2t, t2i = _tbufs(eng, 5)
    assert L.siglip_request_topk(eng._h, 0, recall.data_ptr(), None, None) == _capi.SIGLIP_ERR_INVALID
    assert L.siglip_request_topk(eng._h, 11, recall.data_ptr(), None, None) == _capi.SIGLIP_ERR_INVALID
    assert L.siglip_request_topk(eng._h, 5, None, i2t.data_ptr(), t2i.data_ptr()) == _capi.SIGLIP_ERR_INVALID
    assert L.siglip_request_topk(None, 5, recall.data_ptr(), None, None) == _capi.SIGLIP_ERR_INVALID
    assert L.siglip_request_topk(eng._h, 5, recall.data_ptr(), i2t.data_ptr(), None) == _capi.SIGLIP_OK
    h = torch.zeros(B, D, dtype=torch.bfloat16)
    ticket = ctypes.c_ulonglong(0)
    rc = L.siglip_host_submit(eng._h, h.data_ptr(), h.data_ptr(), 0.0, 0.0, ctypes.byref(ticket),
                              torch.cuda.current_stream().cuda_stream)
    assert rc == _capi.SIGLIP_ERR_STATE and b"top-K" in L.siglip_last_error()
    eng.close()
    dis = SigmoidLossEngine(B, D, _dev(), teacher_dim=D)
    dis.set_option(_capi.SIGLIP_OPT_DISTILL, 1)
    assert L.siglip_request_topk(dis._h, 5, recall.data_ptr(), None, None) == _capi.SIGLIP_ERR_STATE
    dis.close()
    dis = SigmoidLossEngine(B, D, _dev(), teacher_dim=D)
    assert L.siglip_request_topk(dis._h, 5, recall.data_ptr(), None, None) == _capi.SIGLIP_OK
    dis.set_option(_capi.SIGLIP_OPT_DISTILL, 1)   # armed before the option: refused at the step
    x = torch.zeros(B, D, dtype=torch.bfloat16, device=_dev())
    with pytest.raises(RuntimeError, match="top-K"):
        dis.fwd(x, x, _scal(TP), _scal(BIAS))
    dis.close()
