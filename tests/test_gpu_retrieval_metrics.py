"""In-batch retrieval metrics (siglip_request_metrics) on the H100: arming them changes no loss or gradient bit, the
indices match the float64 oracle (one rank, loopback W-rank schedules with seeded peer partials, uneven batches, sample
ids), no key survives into a later step, a CUDA graph follows its inputs, and the modules return them."""
import ctypes
import math

import numpy as np
import pytest
import torch

from retrieval_metrics_oracle import hits, key_as_int64, metric_key, retrieval_metrics

pytestmark = pytest.mark.gpu

MARGIN = 1e-3


def _dev():
    return torch.device("cuda", 0)


def _scal(x):
    return torch.tensor([x], device=_dev(), dtype=torch.float32)


def _engine(B, D, cg=2, ids=False, **kw):
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi

    eng = SigmoidLossEngine(B, D, _dev(), cta_group=cg, **kw)
    if ids:
        eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 1)
    return eng


def _planted(Bs, D, seed, miss=0.2, eps=0.3):
    """Texts are perturbed images under a permutation: a `miss` fraction of the samples form a cyclic derangement
    (text j is close to image perm[j] != j), the rest are positional. Each image has exactly one close text, so the
    top-1 margins are large and the accuracy is about 1 - miss in both directions."""
    g = torch.Generator().manual_seed(seed)
    n = sum(Bs)
    img = torch.nn.functional.normalize(torch.randn(n, D, generator=g))
    perm = torch.arange(n)
    sel = torch.randperm(n, generator=g)[: max(2, int(miss * n))]
    perm[sel] = sel.roll(1)
    txt = torch.nn.functional.normalize(img[perm] + eps * torch.randn(n, D, generator=g) / math.sqrt(D) * 3)
    img, txt = img.to(torch.bfloat16), txt.to(torch.bfloat16)
    return list(torch.split(img, list(Bs))), list(torch.split(txt, list(Bs)))


def _oracle(imgs, txts, ids=None):
    return retrieval_metrics([x.float().numpy() for x in imgs], [x.float().numpy() for x in txts],
                             [x.numpy() for x in ids] if ids is not None else None)


def _bufs(B):
    return (torch.full((2,), -1.0, device=_dev()), torch.full((B,), -7, device=_dev(), dtype=torch.int64),
            torch.full((B,), -7, device=_dev(), dtype=torch.int64))


def _step(eng, sched, img, txt, tp, b, metrics=None, gdt=torch.float32):
    if metrics is not None:
        eng.request_metrics(*metrics)
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


def _check_indices(got, want, margin, what):
    got = got.cpu().numpy()
    ok = margin > MARGIN
    assert ok.mean() >= 0.95, f"{what}: only {ok.mean():.3f} of the rows have a clear top-1"
    bad = np.nonzero(ok & (got != want))[0]
    assert len(bad) == 0, f"{what}: {len(bad)} rows differ, first {bad[:5]}: got {got[bad[:5]]} want {want[bad[:5]]}"


def _check_top1(top1, i2t, t2i, gid, first):
    """top-1 rates are the hit fractions of the returned indices (exactly: integer counts over B)."""
    B = len(i2t)
    hi = hits(i2t.cpu().numpy(), gid, first).sum()
    ht = hits(t2i.cpu().numpy(), gid, first).sum()
    t = top1.cpu()
    assert float(t[0]) == np.float32(hi) / np.float32(B) and float(t[1]) == np.float32(ht) / np.float32(B), (t, hi, ht)


def _seed_peer_keys(eng, ref, imgs_f, txt_r, W, r, beat=()):
    """Stand-in partials of my chunk for every peer p: the key of p's best image for each of my texts (float64 max,
    rounded to fp32). `beat`: (peer, text) pairs whose key is raised above any real similarity."""
    off = ref["off"]
    S = ref["S"]
    want = np.empty(len(txt_r), np.int64)
    for p in range(W):
        if p == r:
            continue
        blk = S[off[p]:off[p + 1], off[r]:off[r + 1]]
        best = np.argmax(blk, axis=0)
        keys = [metric_key(np.float32(blk[best[j], j]), off[p] + best[j]) for j in range(len(best))]
        for (bp, j) in beat:
            if bp == p:
                keys[j] = metric_key(np.float32(1e4), off[p] + (j % (off[p + 1] - off[p])))
        eng.debug_set_peer_metric_keys(p, torch.tensor([key_as_int64(k) for k in keys], dtype=torch.int64,
                                                       device=_dev()))
    want[:] = ref["t2i_index"]
    margin = ref["t2i_margin"].copy()
    for (bp, j) in beat:
        want[j] = off[bp] + (j % (off[bp + 1] - off[bp]))
        margin[j] = np.inf
    return want, margin


# ---------------------------------------------------------------------------------------------------------------------
# 1. arming the metrics changes no output bit
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cg,mcast", [(1, 1), (2, 1), (1, 2)])
@pytest.mark.parametrize("W", [1, 3])
def test_metrics_leave_loss_and_gradients_bit_identical(W, cg, mcast):
    from distributed_sigmoid_loss_b200 import _capi

    B, D = 300, 136
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    imgs, txts = _planted([B] * W, D, 5)
    r = W - 1
    kw = dict(rank_world=(r, W), loopback=True) if W > 1 else {}
    plain, armed = _engine(B, D, cg, **kw), _engine(B, D, cg, **kw)
    for eng in (plain, armed):
        eng.set_option(_capi.SIGLIP_OPT_MCAST, mcast)
        for k in range(W if W > 1 else 0):
            eng.debug_set_text_chunk(k, txts[k].to(_dev()))
    img, txt = imgs[r].to(_dev()), txts[r].to(_dev())
    ref = _oracle(imgs, txts)[r]
    for sched in ("fused", "split", "fwd"):
        for gdt in ((torch.float32, torch.bfloat16) if sched != "fwd" else (torch.float32,)):
            m = _bufs(B)
            a = _step(plain, sched, img, txt, tp, b, None, gdt)
            c = _step(armed, sched, img, txt, tp, b, m, gdt)
            torch.cuda.synchronize()
            for i, (x, y) in enumerate(zip(a, c)):
                assert torch.equal(x, y), f"W={W} cg={cg} mcast={mcast} {sched} {gdt}: output {i} differs"
            _check_indices(m[1], ref["i2t_index"], ref["i2t_margin"], f"{sched} i2t")
            if W == 1:
                _check_indices(m[2], ref["t2i_index"], ref["t2i_margin"], f"{sched} t2i")
    plain.close()
    armed.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. one rank: indices and rates against the oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,D", [(300, 136), (4096, 768)])
def test_single_rank_matches_oracle(B, D):
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    (img,), (txt,) = _planted([B], D, 11)
    ref = _oracle([img], [txt])[0]
    assert 0.5 < ref["i2t_top1"] < 0.95 and 0.5 < ref["t2i_top1"] < 0.95
    eng = _engine(B, D)
    for sched in ("fused", "split", "fwd"):
        m = _bufs(B)
        _step(eng, sched, img.to(_dev()), txt.to(_dev()), tp, b, m)
        torch.cuda.synchronize()
        _check_indices(m[1], ref["i2t_index"], ref["i2t_margin"], f"{sched} i2t")
        _check_indices(m[2], ref["t2i_index"], ref["t2i_margin"], f"{sched} t2i")
        _check_top1(m[0], m[1], m[2], ref["gid"], 0)
        assert abs(float(m[0][0]) - ref["i2t_top1"]) <= 0.05 and abs(float(m[0][1]) - ref["t2i_top1"]) <= 0.05
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. loopback W-rank schedules: i2t over every chunk, t2i combined with seeded peer partials
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Bs,bidir", [([96, 96, 96], False), ([64] * 4, True), ([40, 24, 33], False),
                                      ([384, 256, 130], False)])
def test_loopback_matches_oracle(Bs, bidir):
    from distributed_sigmoid_loss_b200 import _capi

    D = 64
    W = len(Bs)
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    imgs, txts = _planted(Bs, D, 17)
    res = _oracle(imgs, txts)
    for r in range(W):
        ref = res[r]
        eng = _engine(Bs[r], D, rank_world=(r, W), loopback=True, batch_per_rank=Bs)
        if bidir:
            eng.set_option(_capi.SIGLIP_OPT_BIDIR, 1)
        for k in range(W):
            eng.debug_set_text_chunk(k, txts[k].to(_dev()))
        peer = (r + 1) % W
        beat = [(peer, j) for j in range(0, Bs[r], 5)]
        want_t2i, m_t2i = _seed_peer_keys(eng, ref, imgs, txts[r], W, r, beat)
        for sched in ("fused", "split", "fwd"):
            m = _bufs(Bs[r])
            _step(eng, sched, imgs[r].to(_dev()), txts[r].to(_dev()), tp, b, m)
            torch.cuda.synchronize()
            _check_indices(m[1], ref["i2t_index"], ref["i2t_margin"], f"r={r} {sched} i2t")
            _check_indices(m[2], want_t2i, m_t2i, f"r={r} {sched} t2i")
            _check_top1(m[0], m[1], m[2], ref["gid"], ref["off"][r])
        eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. sample ids: a duplicate that wins off the diagonal is a hit
# ---------------------------------------------------------------------------------------------------------------------
def test_ids_duplicate_off_diagonal_is_a_hit():
    B, D = 256, 128
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    (img,), (txt,) = _planted([B], D, 23, miss=0.3)
    ref_pos = _oracle([img], [txt])[0]
    # give every missed pair (image i, its best text j != i) the same id: under ids those become hits
    ids = torch.arange(B, dtype=torch.int64) * 3 + 1
    i2t = ref_pos["i2t_index"]
    for i in range(B):
        j = int(i2t[i])
        if j != i and ref_pos["i2t_margin"][i] > MARGIN:
            ids[j] = ids[i]
    ref = _oracle([img], [txt], [ids])[0]
    assert ref["i2t_top1"] > ref_pos["i2t_top1"]
    eng = _engine(B, D, ids=True)
    for sched in ("fused", "split", "fwd"):
        eng.set_sample_ids(ids.to(_dev()))
        m = _bufs(B)
        _step(eng, sched, img.to(_dev()), txt.to(_dev()), tp, b, m)
        torch.cuda.synchronize()
        _check_indices(m[1], ref["i2t_index"], ref["i2t_margin"], f"{sched} i2t")
        _check_top1(m[0], m[1], m[2], ref["gid"], 0)
        ok = ref["i2t_margin"] > MARGIN
        got_hits = hits(m[1].cpu().numpy(), ref["gid"], 0)
        want_hits = hits(ref["i2t_index"], ref["gid"], 0)
        assert np.array_equal(got_hits[ok], want_hits[ok])
    eng.close()


def test_ids_loopback_maps_peer_indices_to_their_ids():
    Bs, D = [48, 40, 56], 64
    W, r = 3, 1
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    imgs, txts = _planted(Bs, D, 29)
    # ids repeat across ranks: global sample g has id g % 50
    ids = [torch.arange(sum(Bs[:p]), sum(Bs[:p + 1]), dtype=torch.int64) % 50 for p in range(W)]
    ref = _oracle(imgs, txts, ids)[r]
    eng = _engine(Bs[r], D, ids=True, rank_world=(r, W), loopback=True, batch_per_rank=Bs)
    for k in range(W):
        eng.debug_set_text_chunk(k, txts[k].to(_dev()))
    beat = [(0, j) for j in range(0, Bs[r], 3)]
    want_t2i, m_t2i = _seed_peer_keys(eng, ref, imgs, txts[r], W, r, beat)
    for sched in ("fused", "split", "fwd"):
        for k in range(W):
            if k != r:
                eng.debug_set_chunk_ids(k, ids[k].to(_dev()))
        eng.set_sample_ids(ids[r].to(_dev()))
        m = _bufs(Bs[r])
        _step(eng, sched, imgs[r].to(_dev()), txts[r].to(_dev()), tp, b, m)
        torch.cuda.synchronize()
        _check_indices(m[1], ref["i2t_index"], ref["i2t_margin"], f"{sched} i2t")
        _check_indices(m[2], want_t2i, m_t2i, f"{sched} t2i")
        _check_top1(m[0], m[1], m[2], ref["gid"], ref["off"][r])
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. no stale keys, launch count
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W", [1, 3])
def test_no_stale_keys_and_two_extra_launches(W):
    B, D = 200, 64
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    r = 0
    kw = dict(rank_world=(r, W), loopback=True) if W > 1 else {}
    eng = _engine(B, D, **kw)
    # inputs whose similarities shrink from one step to the next: a surviving max of an earlier step would win
    cases = []
    for seed, scale in ((31, 1.0), (32, 0.25), (33, 1.0), (34, 0.1)):
        imgs, txts = _planted([B] * W, D, seed)
        imgs = [(x.float() * scale).to(torch.bfloat16) for x in imgs]
        cases.append((imgs, txts, _oracle(imgs, txts)[r]))
    for sched in ("fused", "fwd"):
        plan = [True, True, False, True]   # two metrics steps in a row, then plain, then metrics
        for (imgs, txts, ref), arm in zip(cases, plan):
            for k in range(W if W > 1 else 0):
                eng.debug_set_text_chunk(k, txts[k].to(_dev()))
            n0 = eng.launch_count
            _step(eng, sched, imgs[r].to(_dev()), txts[r].to(_dev()), tp, b)
            n_plain = eng.launch_count - n0
            if not arm:
                continue
            m = _bufs(B)
            n0 = eng.launch_count
            _step(eng, sched, imgs[r].to(_dev()), txts[r].to(_dev()), tp, b, m)
            assert eng.launch_count - n0 == n_plain + 2
            torch.cuda.synchronize()
            _check_indices(m[1], ref["i2t_index"], ref["i2t_margin"], f"{sched} i2t")
            if W == 1:
                _check_indices(m[2], ref["t2i_index"], ref["t2i_margin"], f"{sched} t2i")
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. a captured single-rank metrics step follows new inputs on replay
# ---------------------------------------------------------------------------------------------------------------------
def test_cuda_graph_replay_follows_inputs():
    B, D = 256, 128
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    eng = _engine(B, D)
    (img0,), (txt0,) = _planted([B], D, 41)
    img = img0.to(_dev()).clone()
    txt = txt0.to(_dev()).clone()
    m = _bufs(B)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _step(eng, "fused", img, txt, tp, b, m)   # warm-up: allocations happen outside the capture
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            eng.request_metrics(*m)
            eng.fwd_bwd(img, txt, tp, b, torch.float32)
    torch.cuda.synchronize()
    for seed in (42, 43):
        (i1,), (t1,) = _planted([B], D, seed)
        img.copy_(i1.to(_dev()))
        txt.copy_(t1.to(_dev()))
        graph.replay()
        torch.cuda.synchronize()
        ref = _oracle([i1], [t1])[0]
        _check_indices(m[1], ref["i2t_index"], ref["i2t_margin"], f"replay {seed} i2t")
        _check_indices(m[2], ref["t2i_index"], ref["t2i_margin"], f"replay {seed} t2i")
    eng.close()


def test_first_request_inside_a_capture_allocates_the_keys():
    """A single-rank context holds no key buffers until metrics are first asked for (its workspace is what it was
    without the feature); that first request may come inside a CUDA-graph capture."""
    B, D = 256, 128
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    eng = _engine(B, D)
    (img0,), (txt0,) = _planted([B], D, 44)
    img, txt = img0.to(_dev()).clone(), txt0.to(_dev()).clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eng.fwd_bwd(img, txt, tp, b, torch.float32)   # warm-up without metrics
        torch.cuda.synchronize()
        ws = eng.workspace_bytes
        m = _bufs(B)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            eng.request_metrics(*m)
            eng.fwd_bwd(img, txt, tp, b, torch.float32)
    assert eng.workspace_bytes == ws + 4 * B * 8
    graph.replay()
    torch.cuda.synchronize()
    ref = _oracle([img0], [txt0])[0]
    _check_indices(m[1], ref["i2t_index"], ref["i2t_margin"], "captured first request i2t")
    _check_indices(m[2], ref["t2i_index"], ref["t2i_margin"], "captured first request t2i")
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# 7. error statuses
# ---------------------------------------------------------------------------------------------------------------------
def test_error_statuses():
    from distributed_sigmoid_loss_b200 import _capi

    B, D = 64, 64
    eng = _engine(B, D)
    L = _capi.lib()
    assert L.siglip_request_metrics(eng._h, None, None, None) == _capi.SIGLIP_ERR_INVALID
    assert L.siglip_request_metrics(None, None, None, None) == _capi.SIGLIP_ERR_INVALID
    m = _bufs(B)
    assert L.siglip_request_metrics(eng._h, m[0].data_ptr(), None, None) == _capi.SIGLIP_OK
    h = torch.zeros(B, D, dtype=torch.bfloat16)
    ticket = ctypes.c_ulonglong(0)
    rc = L.siglip_host_submit(eng._h, h.data_ptr(), h.data_ptr(), 0.0, 0.0, ctypes.byref(ticket),
                              torch.cuda.current_stream().cuda_stream)
    assert rc == _capi.SIGLIP_ERR_STATE and b"metrics" in L.siglip_last_error()
    # the armed request still applies to the next device step, with the index outputs left out
    (img,), (txt,) = _planted([B], D, 51)
    _step(eng, "fwd", img.to(_dev()), txt.to(_dev()), _scal(1.0), _scal(0.0))
    torch.cuda.synchronize()
    assert float(m[0][0]) >= 0.0 and int(m[1][0]) == -7
    # only a loopback context has stand-in peer partials
    keys = torch.zeros(B, dtype=torch.int64, device=_dev())
    assert L.siglip_debug_set_peer_metric_keys(eng._h, 0, keys.data_ptr(), None) == _capi.SIGLIP_ERR_INVALID
    lb = _engine(B, D, rank_world=(1, 2), loopback=True)
    assert L.siglip_debug_set_peer_metric_keys(lb._h, 1, keys.data_ptr(), None) == _capi.SIGLIP_ERR_INVALID
    assert L.siglip_debug_set_peer_metric_keys(lb._h, 0, keys.data_ptr(), None) == _capi.SIGLIP_OK
    lb.close()
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# 8. modules
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,normalize,grad", [(torch.bfloat16, False, True), (torch.float32, False, True),
                                                  (torch.float32, True, True), (torch.bfloat16, False, False)])
def test_ddp_module_returns_metrics(dtype, normalize, grad):
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss

    B, D = 300, 130
    (img,), (txt,) = _planted([B], D, 61)
    mod = DDPSigmoidLoss(B, normalize_inputs=normalize).to(_dev())
    x = img.to(_dev(), dtype).requires_grad_(grad)
    y = txt.to(_dev(), dtype).requires_grad_(grad)
    with torch.set_grad_enabled(grad):
        plain = mod(x, y)
        loss, met = mod(x, y, return_metrics=True)
    assert torch.equal(plain, loss)
    assert set(met) == {"i2t_top1", "t2i_top1", "i2t_index", "t2i_index"}
    assert met["i2t_top1"].shape == () and met["i2t_index"].dtype == torch.int64
    assert not any(v.requires_grad for v in met.values())
    if grad:
        loss.backward()
    ref = _oracle([img], [txt])[0]
    _check_indices(met["i2t_index"], ref["i2t_index"], ref["i2t_margin"], "module i2t")
    _check_indices(met["t2i_index"], ref["t2i_index"], ref["t2i_margin"], "module t2i")


def test_ddp_module_multi_positive_and_siglip_output_dict():
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    B, D = 128, 64
    (img,), (txt,) = _planted([B], D, 71)
    ids32 = (torch.arange(B) // 2).to(torch.int32)
    mod = DDPSigmoidLoss(B, multi_positive=True).to(_dev())
    loss, met = mod(img.to(_dev()), txt.to(_dev()), sample_ids=ids32.to(_dev()), return_metrics=True)
    ref = _oracle([img], [txt], [ids32.to(torch.int64)])[0]
    _check_top1(torch.stack([met["i2t_top1"], met["t2i_top1"]]), met["i2t_index"], met["t2i_index"], ref["gid"], 0)
    sig = SigLipLoss()
    out, met2 = sig(img.to(_dev()), txt.to(_dev()), torch.tensor(math.log(10.0), device=_dev()),
                    torch.tensor(-10.0, device=_dev()), output_dict=True, return_metrics=True)
    assert set(out) == {"contrastive_loss"}
    ref = _oracle([img], [txt])[0]
    _check_indices(met2["i2t_index"], ref["i2t_index"], ref["i2t_margin"], "SigLipLoss i2t")
