"""Extra images per rank (siglip_ctx_create_extras, DDPSigmoidLoss(extra_images=K)) on the H100: hard-negative images
and several images per caption, scored against every text of the global batch. Checked against the float64 oracle of
tests/extra_images_oracle.py on the single-rank fused / split / forward-only schedules, loopback W = 2 and 3 with uneven
B / R / T, R = 300, extras on both sides of the own chunk, extra-image ids that match paired and extra texts of other
chunks, weights (weight-0 extras against no extras), the retrieval metrics (with the loopback peers' extra-image ids),
normalize_inputs, fp32 inputs, bf16 gradients, both gradient tile widths and split-K (same bits), a CUDA-graph capture,
and the error statuses."""
import math

import numpy as np
import pytest
import torch

from extra_images_oracle import closed_form_extras, label_blocks, retrieval_metrics_extras
from retrieval_metrics_oracle import key_as_int64, metric_key

pytestmark = pytest.mark.gpu

TOL = 1e-3
TP, BIAS = math.log(10.0), -10.0


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


def _data(Bs, Rs, Ts, D, seed):
    """Per rank: R images (B paired, then extras that are noisy copies of paired images: further photos of a caption),
    T texts (B captions of the paired images, then extras near random paired images)."""
    g = torch.Generator().manual_seed(seed)
    n = lambda x: torch.nn.functional.normalize(x)  # noqa: E731
    imgs, txts = [], []
    for b, r, t in zip(Bs, Rs, Ts):
        base = n(torch.randn(b, D, generator=g))
        xi = n(base[torch.arange(r - b) % b] + 0.4 * torch.randn(r - b, D, generator=g) / math.sqrt(D) * 8)
        cap = n(base + 0.5 * torch.randn(b, D, generator=g) / math.sqrt(D) * 8)
        xt = n(base[torch.randint(0, b, (t - b,), generator=g)] + 0.6 * torch.randn(t - b, D, generator=g) / math.sqrt(D) * 8)
        imgs.append(torch.cat([base, xi]).to(torch.bfloat16))
        txts.append(torch.cat([cap, xt]).to(torch.bfloat16))
    return imgs, txts


def _ids(Bs, Rs, Ts, seed, cross=True):
    """Sample ids 3 * global paired index; extra texts' ids: ids of paired samples of any rank or fresh ones; extra
    images' ids: ids of paired texts and of extra texts of OTHER ranks (cross) or of their own rank, and fresh ones."""
    rng = np.random.default_rng(seed)
    off = np.concatenate([[0], np.cumsum(Bs)])
    ids = [np.arange(off[p], off[p + 1], dtype=np.int64) * 3 for p in range(len(Bs))]
    allids = np.concatenate(ids)
    xt = [np.where(rng.random(t - b) < 0.7, rng.choice(allids, t - b), 1_000_000 + rng.integers(0, 10**6, t - b))
          .astype(np.int64) for b, t in zip(Bs, Ts)]
    xi = []
    for p, (b, r) in enumerate(zip(Bs, Rs)):
        e = r - b
        own = ids[p][np.arange(e) % b]
        # W = 1: the own rank's captions and extra texts are the only candidates
        src = [q for q in range(len(Bs)) if q != p] or [p]
        pool = np.concatenate([ids[q] for q in src] + [xt[q] for q in src])
        if cross and len(pool):
            pick = np.where(rng.random(e) < 0.5, rng.choice(pool, e) if e else own, own)
        else:
            pick = own
        fresh = rng.random(e) < 0.2
        xi.append(np.where(fresh, 7_000_001 + 2 * np.arange(e), pick).astype(np.int64))
    return ids, xt, xi


def _engine(r, Bs, Rs, Ts, D, cg=2, mcast=1, ids=False, ximg_ids=False, xtxt_ids=False, weights=False):
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi

    W = len(Bs)
    eng = SigmoidLossEngine(Bs[r], D, _dev(), cta_group=cg, rank_world=(r, W), loopback=W > 1, batch_per_rank=Bs,
                            texts_per_rank=Ts, images_per_rank=Rs)
    if mcast != 1:
        eng.set_option(_capi.SIGLIP_OPT_MCAST, mcast)
    if ids:
        eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 1)
    if xtxt_ids:
        eng.set_option(_capi.SIGLIP_OPT_EXTRA_TEXT_IDS, 1)
    if ximg_ids:
        eng.set_option(_capi.SIGLIP_OPT_EXTRA_IMAGE_IDS, 1)
    if weights:
        eng.set_option(_capi.SIGLIP_OPT_SAMPLE_WEIGHTS, 1)
    return eng


def _prepare(eng, r, txts, ids, xt, xi, wi, wt):
    """Per-step inputs of rank r, and (loopback) what the other ranks would have published."""
    dev = _dev()
    if eng.world > 1:
        for k in range(eng.world):
            eng.debug_set_text_chunk(k, txts[k].to(dev))
            if k == r:
                continue
            if ids is not None:
                cid = np.concatenate([ids[k], xt[k]]) if eng.extra_text_ids else ids[k]
                eng.debug_set_chunk_ids(k, torch.from_numpy(cid).to(dev))
            if wt is not None:
                eng.debug_set_chunk_weights(k, wt[k].to(dev))
    if ids is not None:
        eng.set_sample_ids(torch.from_numpy(ids[r]).to(dev))
        if eng.extra_text_ids:
            eng.set_extra_text_ids(torch.from_numpy(xt[r]).to(dev))
        if eng.extra_image_ids:
            eng.set_extra_image_ids(torch.from_numpy(xi[r]).to(dev))
    if wi is not None:
        eng.set_sample_weights(wi[r].to(dev), wt[r].to(dev))


def _step(eng, sched, img, txt, gdt=torch.float32):
    tp, b = _scal(TP), _scal(BIAS)
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


def _oracle(imgs, txts, Bs, ids=None, xt=None, xi=None, wi=None, wt=None):
    Rs, Ts = [len(x) for x in imgs], [len(x) for x in txts]
    labels = label_blocks(Bs, Rs, Ts, ids, xt, xi)
    f = lambda xs: [x.float().numpy() for x in xs]  # noqa: E731
    w = lambda xs: None if xs is None else [x.numpy() for x in xs]  # noqa: E731
    return closed_form_extras(f(imgs), f(txts), Bs, TP, BIAS, labels, w(wi), w(wt))


def _check_rank(tag, eng, r, out, ref, tol=TOL):
    res = ref[r]
    _check(f"{tag} loss", out[0], res["loss"], tol)
    if len(out) == 1:
        return
    _check(f"{tag} dimg", out[1], res["dimg"], tol)
    _check(f"{tag} dtxt (own contribution)", out[2], res["contrib"][r], tol)
    _check(f"{tag} dt_prime", out[3], res["dt_prime"], tol)
    _check(f"{tag} dbias", out[4], res["dbias"], tol)
    others = [k for k in range(eng.world) if k != r]
    for n, k in enumerate(others):
        _check(f"{tag} contribution to chunk {k}", out[5 + n], res["contrib"][k], tol)


def _run(Bs, Rs, Ts, r=0, D=136, sched="fused", mode="pos", weights=False, cg=2, mcast=1, gdt=torch.float32, seed=0,
         tol=TOL, bidir=False):
    imgs, txts = _data(Bs, Rs, Ts, D, seed)
    ids = xt = xi = None
    if mode != "pos":
        ids, xt, xi = _ids(Bs, Rs, Ts, seed)
    wi = wt = None
    if weights:
        g = torch.Generator().manual_seed(seed + 1)
        wi = [torch.rand(x, generator=g) for x in Rs]
        wt = [torch.rand(x, generator=g) for x in Ts]
    eng = _engine(r, Bs, Rs, Ts, D, cg, mcast, ids=mode != "pos", ximg_ids="ximg" in mode, xtxt_ids="xtxt" in mode,
                  weights=weights)
    if bidir:
        from distributed_sigmoid_loss_b200 import _capi
        eng.set_option(_capi.SIGLIP_OPT_BIDIR, 1)
    _prepare(eng, r, txts, ids, xt, xi if "ximg" in mode else None, wi, wt)
    out = _step(eng, sched, imgs[r].to(_dev()), txts[r].to(_dev()), gdt)
    ref = _oracle(imgs, txts, Bs, ids, xt if "xtxt" in mode else None, xi if "ximg" in mode else None, wi, wt)
    _check_rank(f"{Bs}/{Rs}/{Ts} r={r} {sched} {mode} w={weights}", eng, r, out, ref, tol)
    eng.close()


CLUSTERS = [(1, 1), (2, 1), (2, 2)]
MODES = ["pos", "ids", "ids+ximg", "ids+ximg+xtxt"]


# ---------------------------------------------------------------------------------------------------------------------
# 1. single rank: fused, split and forward-only against the oracle; R not a multiple of 128; both extras on the own chunk
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cg,mcast", CLUSTERS)
@pytest.mark.parametrize("sched", ["fused", "split", "fwd"])
@pytest.mark.parametrize("mode", MODES)
def test_single_rank_against_oracle(cg, mcast, sched, mode):
    # R = 300 (not a multiple of 128), T = 300 > B = 260: rows >= B and columns >= B of the own chunk meet on the diagonal
    _run([260], [300], [300], sched=sched, mode=mode, cg=cg, mcast=mcast)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("RT", [(300, 260), (260 + 128, 260 + 37), (1000, 640)])
def test_single_rank_shapes(mode, RT):
    R, T = RT
    _run([260 if R < 1000 else 512], [R], [max(T, 260 if R < 1000 else 512)], mode=mode, D=264, seed=3)


# ---------------------------------------------------------------------------------------------------------------------
# 2. loopback W = 2 / 3 with uneven B / R / T; ids that match paired and extra texts of other chunks
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sched", ["fused", "split"])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("shape", [
    ([96, 160], [130, 160], [96, 200]),
    ([150, 40, 200], [190, 300, 200], [170, 90, 260]),
])
def test_loopback_against_oracle(sched, mode, shape):
    Bs, Rs, Ts = shape
    for r in range(len(Bs)):
        _run(Bs, Rs, Ts, r=r, sched=sched, mode=mode, seed=10 + r)


@pytest.mark.parametrize("sched", ["fused", "split"])
@pytest.mark.parametrize("mode", ["pos", "ids+ximg+xtxt"])
def test_loopback_bidir_against_oracle(sched, mode):
    Bs, Rs, Ts = [150, 40, 200, 64], [190, 300, 200, 64], [170, 90, 260, 100]
    for r in range(len(Bs)):
        _run(Bs, Rs, Ts, r=r, sched=sched, mode=mode, seed=30 + r, bidir=True)


# ---------------------------------------------------------------------------------------------------------------------
# 3. weights, including weight-0 extras against the context without them
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("W", [1, 3])
def test_weights_against_oracle(mode, W):
    shape = ([260], [300], [300]) if W == 1 else ([150, 40, 200], [190, 300, 200], [170, 90, 260])
    for r in range(W):
        _run(*shape, r=r, mode=mode, weights=True, seed=20 + r)


@pytest.mark.parametrize("mode", ["pos", "ids", "ids+ximg"])
@pytest.mark.parametrize("sched", ["fused", "split"])
@pytest.mark.parametrize("T", [200, 240])
def test_weight_zero_extras_equal_no_extras(mode, sched, T):
    B, E, D = 200, 88, 136
    # T == B: the same per-element terms in another CTA / slab layout, equal up to fp32 summation order. T > B: the own
    # chunk of the context with extra images takes its positives through the fp16 sigma operand (own_pos_ids), so the
    # two agree to that operand's rounding
    tol = 1e-5 if T == B else TOL
    imgs, txts = _data([B], [B + E], [T], D, 5)
    ids, xt, xi = _ids([B], [B + E], [T], 5)
    g = torch.Generator().manual_seed(6)
    wt = torch.rand(T, generator=g)
    wi_paired = torch.rand(B, generator=g)
    outs = []
    for with_extras in (True, False):
        R = B + E if with_extras else B
        eng = _engine(0, [B], [R], [T], D, ids=mode != "pos", ximg_ids=with_extras and "ximg" in mode, weights=True)
        wi = torch.cat([wi_paired, torch.zeros(E)]) if with_extras else wi_paired
        _prepare(eng, 0, txts, ids if mode != "pos" else None, xt, xi, [wi], [wt])
        img = imgs[0][:R].to(_dev())
        outs.append(_step(eng, sched, img, txts[0].to(_dev())))
        eng.close()
    a, b = outs
    _check("loss", a[0], b[0].cpu(), tol)
    _check("dtxt", a[2], b[2].cpu(), tol)
    _check("dt_prime", a[3], b[3].cpu(), tol)
    _check("dbias", a[4], b[4].cpu(), tol)
    assert torch.equal(a[1][B:], torch.zeros_like(a[1][B:]))
    _check("dimg paired rows", a[1][:B], b[1].cpu(), tol)


# ---------------------------------------------------------------------------------------------------------------------
# 4. gradient tiles: 128 / 256 columns and split-K give the same bits on a partial last row block
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["pos", "ids+ximg"])
def test_grad_tile_widths_same_bits(mode):
    from distributed_sigmoid_loss_b200 import _capi

    B, R, T, D = 520, 700, 600, 1024   # 700 rows: a partial last 128-row block in dimg and a partial last k block in dtxt
    imgs, txts = _data([B], [R], [T], D, 7)
    ids, xt, xi = _ids([B], [R], [T], 7)
    res = {}
    for tag, opts in (("128", {_capi.SIGLIP_OPT_GRAD_TILE_N: 128}), ("256", {_capi.SIGLIP_OPT_GRAD_TILE_N: 256}),
                      ("splitk", {_capi.SIGLIP_OPT_GRAD_TILE_N: 128, _capi.SIGLIP_OPT_SPLIT_K: -1})):
        eng = _engine(0, [B], [R], [T], D, cg=1, ids=mode != "pos", ximg_ids="ximg" in mode)
        for k, v in opts.items():
            eng.set_option(k, v)
        _prepare(eng, 0, txts, ids if mode != "pos" else None, xt, xi, None, None)
        res[tag] = _step(eng, "fused", imgs[0].to(_dev()), txts[0].to(_dev()))
        eng.close()
    for tag in ("256", "splitk"):
        for n, (a, b) in enumerate(zip(res["128"], res[tag])):
            assert torch.equal(a, b), f"{tag}: output {n} differs from the 128-column tiles"
    ref = _oracle(imgs, txts, [B], ids if mode != "pos" else None, None, xi if "ximg" in mode else None)
    _check_rank("tiles", type("E", (), {"world": 1})(), 0, res["128"], ref)


# ---------------------------------------------------------------------------------------------------------------------
# 5. bf16 gradients, fp32 inputs and normalize_inputs through the module; autograd of extra_image
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("kind", ["bf16", "fp32", "normalize"])
@pytest.mark.parametrize("multi", [False, True])
def test_module_against_oracle(fused, kind, multi):
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss

    B, K, D = 256, 70, 96
    imgs, txts = _data([B], [B + K], [B], D, 9)
    ids, _, xi = _ids([B], [B + K], [B], 9)
    dt = torch.bfloat16 if kind == "bf16" else torch.float32
    img_in = imgs[0].to(dt)
    if kind == "normalize":
        img_in = img_in * 3.0
    a = img_in[:B].to(_dev()).clone().requires_grad_(True)
    e = img_in[B:].to(_dev()).clone().requires_grad_(True)
    t = txts[0].to(dt).to(_dev()).clone().requires_grad_(True)
    mod = DDPSigmoidLoss(B, fused_step=fused, normalize_inputs=kind == "normalize", multi_positive=multi,
                         extra_images=K).to(_dev())
    kw = dict(extra_image=e)
    if multi:
        kw.update(sample_ids=torch.from_numpy(ids[0]).to(_dev()), extra_image_ids=torch.from_numpy(xi[0]).to(_dev()))
    loss = mod(a, t, **kw)
    loss.backward()
    if kind == "normalize":   # the oracle on the normalised inputs; gradients projected back through F.normalize
        xi_f = [torch.nn.functional.normalize(img_in.double())]
        xt_f = [torch.nn.functional.normalize(txts[0].double())]
    else:
        xi_f, xt_f = [imgs[0].double()], [txts[0].double()]
    labels = label_blocks([B], [B + K], [B], ids if multi else None, None, xi if multi else None)
    ref = closed_form_extras([x.numpy() for x in xi_f], [x.numpy() for x in xt_f], [B], TP, BIAS, labels)[0]
    tol = TOL if kind != "bf16" else TOL + 2.0 ** -8

    def back(raw, g):
        if kind != "normalize":
            return g
        raw = raw.double()
        xn = torch.nn.functional.normalize(raw)
        g = torch.from_numpy(g)
        return (g - xn * (xn * g).sum(1, keepdim=True)) / raw.norm(dim=1, keepdim=True)

    _check("loss", loss.detach(), ref["loss"], tol)
    _check("dimg", torch.cat([a.grad, e.grad]).float(), back(img_in, ref["dimg"]), tol)
    assert e.grad.dtype == e.dtype and e.grad.shape == e.shape
    _check("dtxt", t.grad.float(), back(txts[0], ref["contrib"][0]), tol)
    _check("t_prime.grad", mod.t_prime.grad, ref["dt_prime"], tol)
    _check("bias.grad", mod.bias.grad, ref["dbias"], tol)


def test_siglip_loss_and_composition():
    """SigLipLoss with extra images, extra texts with ids, weights and metrics in one forward."""
    from distributed_sigmoid_loss_b200 import SigLipLoss

    B, K, Kt, D = 192, 40, 24, 64
    imgs, txts = _data([B], [B + K], [B + Kt], D, 11)
    ids, xt, xi = _ids([B], [B + K], [B + Kt], 11)
    g = torch.Generator().manual_seed(12)
    wi, wt = torch.rand(B + K, generator=g), torch.rand(B + Kt, generator=g)
    mod = SigLipLoss(multi_positive=True, extra_texts=Kt, extra_images=K, sample_weights=True, fused_step=True)
    a = imgs[0][:B].to(_dev()).requires_grad_(True)
    e = imgs[0][B:].to(_dev()).requires_grad_(True)
    t = txts[0][:B].to(_dev()).requires_grad_(True)
    x = txts[0][B:].to(_dev()).requires_grad_(True)
    d = lambda v: torch.from_numpy(v).to(_dev())  # noqa: E731
    loss, m = mod(a, t, _scal(TP).reshape(()), _scal(BIAS).reshape(()), sample_ids=d(ids[0]), extra_text=x,
                  extra_text_ids=d(xt[0]), extra_image=e, extra_image_ids=d(xi[0]), image_weights=wi.to(_dev()),
                  text_weights=wt.to(_dev()), return_metrics=True)
    loss.backward()
    ref = _oracle(imgs, txts, [B], ids, xt, xi, [wi], [wt])[0]
    _check("loss", loss.detach(), ref["loss"], TOL + 2.0 ** -8)
    _check("dimg", torch.cat([a.grad, e.grad]).float(), ref["dimg"], TOL + 2.0 ** -8)
    _check("dtxt", torch.cat([t.grad, x.grad]).float(), ref["contrib"][0], TOL + 2.0 ** -8)
    assert m["i2t_index"].shape == (B + K,) and m["t2i_index"].shape == (B + Kt,)


# ---------------------------------------------------------------------------------------------------------------------
# 6. retrieval metrics: exact indices where no near-tie exists; loopback peers' extra-image ids
# ---------------------------------------------------------------------------------------------------------------------
def _metrics_step(eng, r, imgs, txts, ids, xt, xi):
    dev = _dev()
    top1 = torch.empty(2, device=dev)
    i2t = torch.empty(eng.metric_images, device=dev, dtype=torch.int64)
    t2i = torch.empty(eng.metric_texts, device=dev, dtype=torch.int64)
    eng.request_metrics(top1, i2t, t2i)
    out = _step(eng, "fused", imgs[r].to(dev), txts[r].to(dev))
    torch.cuda.synchronize()
    return top1.cpu(), i2t.cpu().numpy(), t2i.cpu().numpy(), out


@pytest.mark.parametrize("mode", MODES)
def test_metrics_single_rank(mode):
    Bs, Rs, Ts, D = [260], [300], [300], 136
    imgs, txts = _data(Bs, Rs, Ts, D, 13)
    ids, xt, xi = _ids(Bs, Rs, Ts, 13) if mode != "pos" else (None, None, None)
    eng = _engine(0, Bs, Rs, Ts, D, ids=mode != "pos", ximg_ids="ximg" in mode, xtxt_ids="xtxt" in mode)
    _prepare(eng, 0, txts, ids, xt, xi, None, None)
    top1, i2t, t2i, out = _metrics_step(eng, 0, imgs, txts, ids, xt, xi)
    want = retrieval_metrics_extras([x.float().numpy() for x in imgs], [x.float().numpy() for x in txts], Bs, ids,
                                    xt if "xtxt" in mode else None, xi if "ximg" in mode else None)[0]
    for name, got, idx, mg in (("i2t", i2t, want["i2t_index"], want["i2t_margin"]),
                               ("t2i", t2i, want["t2i_index"], want["t2i_margin"])):
        assert got.shape == idx.shape, (name, got.shape, idx.shape)
        clear = mg > 1e-4
        assert clear.mean() > 0.95 and np.array_equal(got[clear], idx[clear]), name
    # the rates from the returned indices, with the oracle's hit rule
    if clear.all():
        assert abs(float(top1[0]) - want["i2t_top1"]) < 1e-6 and abs(float(top1[1]) - want["t2i_top1"]) < 1e-6
    # loss and gradients are the step's without metrics
    ref = _oracle(imgs, txts, Bs, ids, xt if "xtxt" in mode else None, xi if "ximg" in mode else None)
    _check_rank("metrics step", eng, 0, out, ref)
    eng.close()


@pytest.mark.parametrize("ximg", [False, True])
def test_metrics_loopback_peer_extra_image_ids(ximg):
    """W = 2 loopback, rank 0. Peer 1's column partials of my texts are seeded so that text j's best image is peer 1's
    extra image j (s = 10, beyond any real logit), and peer 1's published extra-image ids are seeded too: under
    SIGLIP_OPT_EXTRA_IMAGE_IDS the even texts get their own id (hits), the odd ones a foreign id (misses); without the
    option every such text is a miss."""
    Bs, Rs, Ts, D = [64, 64], [100, 164], [64, 64], 64
    imgs, txts = _data(Bs, Rs, Ts, D, 17)
    ids, xt, xi = _ids(Bs, Rs, Ts, 17)
    eng = _engine(0, Bs, Rs, Ts, D, ids=True, ximg_ids=ximg)
    _prepare(eng, 0, txts, ids, xt, xi if ximg else None, None, None)
    off1 = Rs[0]   # global index of peer 1's first image
    keys = [key_as_int64(metric_key(10.0, off1 + Bs[1] + j)) for j in range(Bs[0])]
    eng.debug_set_peer_metric_keys(1, torch.tensor(keys, dtype=torch.int64, device=_dev()))
    peer_x = np.full(Rs[1] - Bs[1], 9_999_999, np.int64)
    peer_x[: Bs[0]: 2] = ids[0][::2]
    eng.debug_set_peer_extra_image_ids(1, torch.from_numpy(peer_x).to(_dev()))
    top1, i2t, t2i, _ = _metrics_step(eng, 0, imgs, txts, ids, xt, xi)
    assert np.array_equal(t2i, off1 + Bs[1] + np.arange(Bs[0]))
    want = (Bs[0] + 1) // 2 / Bs[0] if ximg else 0.0
    assert abs(float(top1[1]) - want) < 1e-6, (float(top1[1]), want)
    assert i2t.shape == ((Rs[0],) if ximg else (Bs[0],))
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# 7. CUDA graph of a single-rank step with ids, and the error statuses
# ---------------------------------------------------------------------------------------------------------------------
def test_cuda_graph_capture_with_ids():
    Bs, Rs, Ts, D = [256], [320], [288], 128
    imgs, txts = _data(Bs, Rs, Ts, D, 19)
    ids, xt, xi = _ids(Bs, Rs, Ts, 19)
    eng = _engine(0, Bs, Rs, Ts, D, ids=True, ximg_ids=True, xtxt_ids=True)
    dev = _dev()
    img, txt = imgs[0].to(dev), txts[0].to(dev)
    sid, tid, iid = (torch.from_numpy(x[0]).to(dev) for x in (ids, xt, xi))
    tp, b = _scal(TP), _scal(BIAS)

    def step():
        eng.set_sample_ids(sid)
        eng.set_extra_text_ids(tid)
        eng.set_extra_image_ids(iid)
        return eng.fwd_bwd(img, txt, tp, b)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()   # warm-up: allocations and module loads outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    iid.copy_(torch.from_numpy(xi[0][::-1].copy()).to(dev))   # the replay copies the ids it finds then
    graph.replay()
    torch.cuda.synchronize()
    xr = [xi[0][::-1].copy()]
    ref = _oracle(imgs, txts, Bs, ids, xt, xr)
    _check_rank("graph", eng, 0, [x.clone() for x in out], ref)
    eng.close()


def test_error_statuses():
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi
    from distributed_sigmoid_loss_b200._capi import SiglipError

    L = _capi.lib()
    import ctypes
    h = ctypes.c_void_p()
    one = lambda v: (ctypes.c_int * 1)(v)  # noqa: E731
    assert L.siglip_ctx_create_extras(ctypes.byref(h), 0, 0, 1, one(64), one(63), one(64), 64) == _capi.SIGLIP_ERR_INVALID
    assert L.siglip_ctx_create_extras(ctypes.byref(h), 0, 0, 1, one(64), one(64), one(63), 64) == _capi.SIGLIP_ERR_INVALID
    eng = SigmoidLossEngine(64, 64, _dev(), batch_per_rank=[64], texts_per_rank=[64], images_per_rank=[80])
    # the option needs the sample ids first; the setter needs the option
    with pytest.raises(SiglipError):
        eng.set_option(_capi.SIGLIP_OPT_EXTRA_IMAGE_IDS, 1)
    with pytest.raises(SiglipError):
        eng.set_extra_image_ids(torch.zeros(16, dtype=torch.int64, device=_dev()))
    eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 1)
    eng.set_option(_capi.SIGLIP_OPT_EXTRA_IMAGE_IDS, 1)
    img = torch.zeros(80, 64, dtype=torch.bfloat16, device=_dev())
    txt = torch.zeros(64, 64, dtype=torch.bfloat16, device=_dev())
    eng.set_sample_ids(torch.arange(64, device=_dev()))
    launches = eng.launch_count
    with pytest.raises(SiglipError) as ei:   # ids of the extra images missing: refused before any launch
        eng.fwd_bwd(img, txt, _scal(TP), _scal(BIAS))
    assert ei.value.code == _capi.SIGLIP_ERR_STATE and eng.launch_count == launches
    # the host-buffer entries refuse a context with extra images
    eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 0)
    with pytest.raises(SiglipError) as ei:
        eng.fwd_bwd_host(torch.zeros(64, 64, dtype=torch.bfloat16), torch.zeros(64, 64, dtype=torch.bfloat16), TP, BIAS)
    assert ei.value.code == _capi.SIGLIP_ERR_STATE
    eng.close()
