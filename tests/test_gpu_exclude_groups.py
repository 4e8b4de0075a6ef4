"""Excluded same-group pairs (SIGLIP_OPT_EXCLUDE_GROUPS, DDPSigmoidLoss / SigLipLoss(exclude_groups=True)) on the H100.
Random groups are checked against the float64 oracle with labels in {+1, -1, 0} at logits where the excluded pairs carry
real weight (clustered embeddings, bias -5: a same-cluster negative has sigma(z) ~ 0.2), so a kernel that drops an
excluded pair from the loss but keeps its sigma in the gradient operand fails the gradient checks. Unique groups and
all-negative groups are checked against the step without the option: bit for bit for loss, gradients, dt', dbias,
metrics and top-K lists, to within 1e-6 relative for the per-sample losses."""
import math

import numpy as np
import pytest
import torch

from exclude_groups_oracle import closed_form_groups, clustered, group_labels, pad_rows, torch_loss
from sample_weights_oracle import label_blocks

pytestmark = pytest.mark.gpu

TOL = 1e-3
TP, BIAS = math.log(10.0), -5.0
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


def _engine(B, D, W=1, r=0, cg=2, mcast=1, stages=0, Ts=None, Rs=None, ids=False, extra_ids=False, weights=False,
            groups=True, budget=None):
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi

    eng = SigmoidLossEngine(B, D, _dev(), cta_group=cg, rank_world=(r, W), loopback=W > 1, texts_per_rank=Ts,
                            images_per_rank=Rs)
    if mcast != 1:
        eng.set_option(_capi.SIGLIP_OPT_MCAST, mcast)
    if stages:
        eng.set_option(_capi.SIGLIP_OPT_STAGES_LOSS, stages)
    if ids:
        eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 1)
    if extra_ids:
        eng.set_option(_capi.SIGLIP_OPT_EXTRA_TEXT_IDS, 1)
    if weights:
        eng.set_option(_capi.SIGLIP_OPT_SAMPLE_WEIGHTS, 1)
    if groups:
        eng.set_option(_capi.SIGLIP_OPT_EXCLUDE_GROUPS, 1)
    if budget:
        eng.set_sigma_budget(budget)
    eng.grouped, eng.weighted = groups, weights
    return eng


class Problem:
    """Rank r of a W-rank job: W text chunks (B paired texts + K extras each), this rank's B + E images, groups drawn
    from n_groups classes (a fraction of them -1), clustered embeddings around the group centres. mode: pos, ids
    (duplicated sample ids), extra (extra texts with ids)."""

    def __init__(self, B, D, W=1, r=0, K=0, E=0, mode="pos", weights=False, n_groups=7, seed=0, neg_frac=0.2):
        rng = np.random.default_rng(seed)
        self.B, self.D, self.W, self.r, self.K, self.E, self.mode = B, D, W, r, K, E, mode
        self.Bs, self.Ts, self.Rs = [B] * W, [B + K] * W, [B + E] * W
        # groups of the paired samples (image i and text i of a rank share one), then of the extras
        pg = [rng.integers(0, n_groups, B) for _ in range(W)]
        self.tg = [np.concatenate([pg[c], rng.integers(0, n_groups, K)]) for c in range(W)]
        self.ig = np.concatenate([pg[r], rng.integers(0, n_groups, E)])
        emb = lambda g, s: torch.from_numpy(clustered(g, D, n_groups, seed, s)).float().to(torch.bfloat16)  # noqa: E731
        self.texts = [emb(self.tg[c], 1000 * seed + c + 1) for c in range(W)]
        self.img = emb(self.ig, 1000 * seed + 999)
        for g in self.tg + [self.ig]:   # some samples have no group
            g[rng.random(len(g)) < neg_frac] = -1
        self.ids = self.eids = None
        if mode != "pos":
            self.ids = [torch.from_numpy(rng.integers(0, B, B)) for _ in range(W)]
            self.eids = [torch.from_numpy(rng.integers(0, 2 * B, K)) for _ in range(W)]
        self.iw = self.tws = None
        if weights:
            self.iw = torch.from_numpy(rng.random(B + E)).float()
            self.tws = [torch.from_numpy(rng.random(B + K)).float() for _ in range(W)]

    def labels(self, groups=True):
        f = (lambda xs: None if xs is None else [x.numpy() for x in xs])  # noqa: E731
        lab = label_blocks(self.Bs, self.Ts, f(self.ids), f(self.eids) if self.mode == "extra" else None)
        lab = pad_rows([lab[self.r]], [self.Rs[self.r]])
        return group_labels(lab, [self.ig], self.tg) if groups else lab

    def oracle(self, groups=True):
        imgs = [self.img.double().numpy()]
        txts = [t.double().numpy() for t in self.texts]
        iws = None if self.iw is None else [self.iw.double().numpy()]
        tws = None if self.tws is None else [t.double().numpy() for t in self.tws]
        return closed_form_groups(imgs, txts, TP, BIAS, self.labels(groups), [self.B], iws, tws)[0]

    def seed_peers(self, eng):
        for k in range(self.W):
            eng.debug_set_text_chunk(k, self.texts[k].to(_dev()))
            if k == self.r:
                continue
            if self.ids is not None:
                eng.debug_set_chunk_ids(k, (torch.cat([self.ids[k], self.eids[k]]) if eng.extra_text_ids
                                            else self.ids[k]).to(_dev()))
            if eng.weighted:
                eng.debug_set_chunk_weights(k, self.tws[k].to(_dev()))
            if eng.grouped:
                eng.debug_set_chunk_groups(k, torch.from_numpy(self.tg[k]).to(_dev()))

    def step(self, eng, sched="fused", groups=None, losses=False, metrics_k=0):
        """One step; returns its outputs by name (the contributions to the peers' chunks as slot<k>)."""
        r = self.r
        if self.ids is not None:
            eng.set_sample_ids(self.ids[r].to(_dev()))
            if eng.extra_text_ids:
                eng.set_extra_text_ids(self.eids[r].to(_dev()))
        if eng.weighted:
            eng.set_sample_weights(self.iw.to(_dev()), self.tws[r].to(_dev()))
        if eng.grouped:
            ig, tg = groups if groups is not None else (self.ig, self.tg[r])
            eng.set_groups(torch.as_tensor(ig).to(_dev()), torch.as_tensor(tg).to(_dev()))
        out = {}
        if losses:
            out["image_loss"] = torch.full((eng.images,), -1.0, device=_dev())
            out["text_loss"] = torch.full((eng.texts,), -1.0, device=_dev())
            eng.request_sample_losses(out["image_loss"], out["text_loss"])
        if metrics_k:
            out["top1"] = torch.zeros(2, device=_dev())
            out["i2t"] = torch.zeros(eng.metric_images, dtype=torch.int64, device=_dev())
            out["t2i"] = torch.zeros(eng.metric_texts, dtype=torch.int64, device=_dev())
            eng.request_metrics(out["top1"], out["i2t"], out["t2i"])
            if metrics_k > 1:
                out["recall"] = torch.zeros(2 * metrics_k, device=_dev())
                out["i2t_k"] = torch.zeros(eng.metric_images, metrics_k, dtype=torch.int64, device=_dev())
                out["t2i_k"] = torch.zeros(eng.metric_texts, metrics_k, dtype=torch.int64, device=_dev())
                eng.request_topk(metrics_k, out["recall"], out["i2t_k"], out["t2i_k"])
        img, txt = self.img.to(_dev()), self.texts[r].to(_dev())
        tp, b = _scal(TP), _scal(BIAS)
        if sched == "fused":
            out["loss"], out["dimg"], out["dtxt"], out["dtp"], out["db"] = eng.fwd_bwd(img, txt, tp, b)
        elif sched == "split":
            out["loss"] = eng.forward(img, txt, tp, b, True)
            out["dimg"], out["dtxt"], out["dtp"], out["db"] = eng.backward(img, txt, tp, None)
        else:
            out["loss"] = eng.fwd(img, txt, tp, b)
        for k in range(eng.world):
            if k != r and sched != "fwd":
                out[f"slot{k}"] = eng.debug_get_slot(k)
        torch.cuda.synchronize()
        return {k: v.clone() for k, v in out.items()}

    def check(self, tag, out, ref, tol=TOL):
        _check(f"{tag} loss", out["loss"], ref["loss"], tol)
        if "dimg" not in out:
            return
        _check(f"{tag} dimg", out["dimg"], ref["dimg"], tol)
        _check(f"{tag} dt_prime", out["dtp"], ref["dt_prime"], tol)
        _check(f"{tag} dbias", out["db"], ref["dbias"], tol)
        for k in range(self.W):
            got = out["dtxt"] if k == self.r else out[f"slot{k}"]
            _check(f"{tag} contribution to chunk {k}", got, ref["contrib"][k], tol)
        if "image_loss" in out:
            _check(f"{tag} image_loss", out["image_loss"], ref["image_loss"], tol)
            if self.W == 1:
                _check(f"{tag} text_loss", out["text_loss"], ref["text_part"][0], tol)


def _excluded(p):
    return sum(int((y == 0).sum()) for y in p.labels()[0])


# ---------------------------------------------------------------------------------------------------------------------
# 1. against the float64 oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sched", ["fused", "split"])
@pytest.mark.parametrize("stages", [4, 6])
@pytest.mark.parametrize("cg,mcast", CLUSTERS)
@pytest.mark.parametrize("B,D", [(300, 136), (40, 1152)])
def test_random_groups_match_the_oracle(B, D, cg, mcast, stages, sched):
    p = Problem(B, D, seed=B + D)
    assert _excluded(p) > B   # the test has excluded pairs to get wrong
    eng = _engine(B, D, cg=cg, mcast=mcast, stages=stages)
    ref = p.oracle()
    p.check(f"B={B} D={D} cg={cg} mc={mcast} st={stages} {sched}", p.step(eng, sched), ref)
    # the excluded pairs matter at these logits: without the exclusion the results differ far beyond the tolerance
    base = p.oracle(groups=False)
    assert _rel(ref["dimg"], base["dimg"]) > 20 * TOL and abs(ref["dbias"] - base["dbias"]) > 20 * TOL * abs(base["dbias"])


@pytest.mark.parametrize("mode,K,E,weights", [("pos", 0, 0, True), ("ids", 0, 0, False), ("ids", 0, 0, True),
                                              ("pos", 37, 0, False), ("extra", 29, 0, True), ("pos", 0, 23, False),
                                              ("ids", 13, 19, True)])
def test_options_compose_with_groups(mode, K, E, weights):
    B, D = 300, 136
    p = Problem(B, D, K=K, E=E, mode=mode, weights=weights, seed=K + 3 * E + (mode == "ids"))
    eng = _engine(B, D, Ts=[B + K] if K else None, Rs=[B + E] if E else None, ids=mode != "pos",
                  extra_ids=mode == "extra", weights=weights)
    p.check(f"{mode} K={K} E={E} w={weights}", p.step(eng, losses=True), p.oracle())
    p.check(f"{mode} K={K} E={E} w={weights} fwd", p.step(eng, "fwd"), p.oracle())


@pytest.mark.parametrize("W,mode,K", [(2, "pos", 0), (3, "ids", 0), (3, "extra", 17), (2, "pos", 11)])
@pytest.mark.parametrize("cg,mcast", [(2, 1), (1, 1)])
def test_loopback_peer_groups(W, mode, K, cg, mcast):
    B, D = 136, 264
    r = W - 1
    p = Problem(B, D, W=W, r=r, K=K, mode=mode, weights=(W == 3), seed=10 * W + K)
    eng = _engine(B, D, W=W, r=r, cg=cg, mcast=mcast, Ts=[B + K] * W if K else None, ids=mode != "pos",
                  extra_ids=mode == "extra", weights=(W == 3))
    p.seed_peers(eng)
    ref = p.oracle()
    for sched in ("fused", "split"):
        p.check(f"W={W} {mode} K={K} {sched}", p.step(eng, sched, losses=(sched == "fused")), ref)


def test_row_panels_under_a_sigma_budget():
    B, D = 1000, 136
    p = Problem(B, D, seed=5)
    eng = _engine(B, D, budget=1 << 20)
    assert eng.sigma_panels()[1] > 1
    p.check("panels", p.step(eng, losses=True), p.oracle())
    W = 2
    p2 = Problem(B, D, W=W, r=1, mode="ids", seed=6)
    eng2 = _engine(B, D, W=W, r=1, ids=True, budget=2 << 20)
    assert eng2.sigma_panels()[1] > 1
    p2.seed_peers(eng2)
    p2.check("panels W=2", p2.step(eng2, losses=True), p2.oracle())


# ---------------------------------------------------------------------------------------------------------------------
# 2. bit for bit the step without the option
# ---------------------------------------------------------------------------------------------------------------------
# The per-sample sums of the groups kernel round their fp32 partials differently from the per-sample-loss kernel's
# (a few ulps: the compiler contracts the term additions differently in the two instantiations); every other output
# is bit-identical.
ULP_KEYS = ("image_loss", "text_loss")


def _same(tag, a, b):
    assert a.keys() == b.keys()
    bad = {k: float((a[k].double() - b[k].double()).abs().max()) for k in a if not torch.equal(a[k], b[k])}
    near = {k: v for k, v in bad.items() if k in ULP_KEYS and torch.allclose(a[k], b[k], rtol=1e-6, atol=0)}
    bad = {k: v for k, v in bad.items() if k not in near}
    assert not bad, f"{tag}: differs (max abs difference) {bad}"


@pytest.mark.parametrize("kind", ["unique", "none"])
@pytest.mark.parametrize("mode,K,E", [("pos", 0, 0), ("ids", 0, 0), ("pos", 37, 23), ("extra", 29, 0)])
@pytest.mark.parametrize("cg,mcast", [(2, 1), (1, 1)])
def test_unique_or_no_groups_are_bitwise_the_plain_step(kind, mode, K, E, cg, mcast):
    """Unique groups (each image shares its group with its positives only) and negative groups (no group at all) give
    the plain step's loss, gradients, dt', dbias, metrics, top-K lists and per-sample losses bit for bit."""
    B, D = 300, 136
    p = Problem(B, D, K=K, E=E, mode=mode, weights=True, seed=7)
    if kind == "unique":
        # paired sample i: group i (ids mode: its sample id, so that every id-positive shares it); extras: none or fresh
        ig = p.ids[0].numpy() if mode != "pos" else np.arange(B)
        tg = np.concatenate([ig, p.eids[0].numpy() if mode == "extra" else -np.ones(K, np.int64)])
        ig = np.concatenate([ig, -np.ones(E, np.int64)])
    else:
        ig, tg = -np.ones(B + E, np.int64), -np.arange(1, B + K + 1)
    kw = dict(cg=cg, mcast=mcast, Ts=[B + K] if K else None, Rs=[B + E] if E else None, ids=mode != "pos",
              extra_ids=mode == "extra", weights=True)
    on, off = _engine(B, D, **kw), _engine(B, D, groups=False, **kw)
    for sched in ("fused", "split", "fwd"):
        for k in (0, 1, 5):
            a = p.step(on, sched, groups=(ig, tg), losses=(sched == "fused"), metrics_k=k)
            b = p.step(off, sched, losses=(sched == "fused"), metrics_k=k)
            _same(f"{kind} {mode} {sched} k={k}", a, b)


def test_loopback_unique_groups_are_bitwise_the_plain_step():
    B, D, W, r = 136, 264, 3, 1
    p = Problem(B, D, W=W, r=r, mode="ids", seed=8)
    kw = dict(W=W, r=r, ids=True)
    on, off = _engine(B, D, **kw), _engine(B, D, groups=False, **kw)
    p.tg = [x.numpy().copy() for x in p.ids]   # unique: the sample ids themselves
    p.ig = p.tg[r].copy()
    p.seed_peers(on)
    p.seed_peers(off)
    _same("loopback", p.step(on, losses=True, metrics_k=5), p.step(off, losses=True, metrics_k=5))


# ---------------------------------------------------------------------------------------------------------------------
# 3. capture, modules, errors
# ---------------------------------------------------------------------------------------------------------------------
def test_single_rank_step_captures_into_a_cuda_graph():
    B, D = 300, 136
    p = Problem(B, D, seed=9)
    eng = _engine(B, D)
    img, txt, tp, b = p.img.to(_dev()), p.texts[0].to(_dev()), _scal(TP), _scal(BIAS)
    gi = torch.from_numpy(p.ig).to(_dev())
    gt = torch.from_numpy(p.tg[0]).to(_dev())
    eager = p.step(eng)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):   # warm-up outside the capture
        eng.set_groups(gi, gt)
        eng.fwd_bwd(img, txt, tp, b)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        eng.set_groups(gi, gt)
        loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, tp, b)
    gi.fill_(-1)   # the replay reads the groups at replay time: first none, then the problem's again
    gt.fill_(-1)
    g.replay()
    torch.cuda.synchronize()
    assert not torch.equal(dimg, eager["dimg"])
    gi.copy_(torch.from_numpy(p.ig))
    gt.copy_(torch.from_numpy(p.tg[0]))
    g.replay()
    torch.cuda.synchronize()
    for k, v in (("loss", loss), ("dimg", dimg), ("dtxt", dtxt), ("dtp", dtp), ("db", db)):
        assert torch.equal(v, eager[k]), k


@pytest.mark.parametrize("dtype,normalize", [(torch.bfloat16, False), (torch.float32, False), (torch.float32, True)])
def test_module_against_autograd_restatement(dtype, normalize):
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss

    B, D, K = 300, 136, 20
    p = Problem(B, D, K=K, seed=11)
    mod = DDPSigmoidLoss(B, normalize_inputs=normalize, hard_negatives=K, exclude_groups=True).to(_dev())
    with torch.no_grad():
        mod.bias.fill_(BIAS)
    scale = 3.0 if normalize else 1.0
    img = (p.img.float() * scale).to(dtype).to(_dev()).requires_grad_(True)
    txt = (p.texts[0].float() * scale).to(dtype).to(_dev())
    pos, neg = txt[:B].clone().requires_grad_(True), txt[B:].clone().requires_grad_(True)
    gi, gt = torch.from_numpy(p.ig).to(_dev()), torch.from_numpy(p.tg[0]).to(_dev())
    loss, sl = mod(img, pos, negative_text=neg, image_groups=gi, text_groups=gt, return_sample_losses=True)
    loss.backward()
    # float64 autograd of the torch restatement with the same labels
    y = torch.from_numpy(p.labels()[0][0])
    xi = img.detach().double().cpu().requires_grad_(True)
    xt = torch.cat([pos, neg]).detach().double().cpu().requires_grad_(True)
    tp = torch.tensor(TP, dtype=torch.float64, requires_grad=True)
    bb = torch.tensor(BIAS, dtype=torch.float64, requires_grad=True)
    ref = torch_loss(xi, xt, tp, bb, y, normalize=normalize, batch=B)
    ref.backward()
    tol = 4e-3 if dtype == torch.bfloat16 else TOL   # bf16 gradients: 2^-9 rounding
    _check("module loss", loss.detach(), ref.detach(), tol)
    _check("module dimg", img.grad, xi.grad, tol)
    _check("module dtxt", torch.cat([pos.grad, neg.grad]), xt.grad, tol)
    _check("module dt'", mod.t_prime.grad, tp.grad, tol)
    _check("module dbias", mod.bias.grad, bb.grad, tol)
    assert float(sl["image_loss"].sum()) == pytest.approx(float(loss) * B, rel=1e-4)


def test_siglip_loss_matches_ddp_module():
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    B, D = 300, 136
    p = Problem(B, D, seed=12)
    gi, gt = torch.from_numpy(p.ig).to(_dev()), torch.from_numpy(p.tg[0]).to(_dev())
    img, txt = p.img.to(_dev()), p.texts[0].to(_dev())
    ddp = DDPSigmoidLoss(B, exclude_groups=True).to(_dev())
    with torch.no_grad():
        ddp.bias.fill_(BIAS)
    a = ddp(img, txt, image_groups=gi, text_groups=gt)
    b = SigLipLoss(exclude_groups=True)(img, txt, torch.tensor(TP, device=_dev()), torch.tensor(BIAS, device=_dev()),
                                        image_groups=gi, text_groups=gt)
    assert float(a) == pytest.approx(float(b), rel=1e-5)
    _check("siglip vs oracle", b, p.oracle()["loss"])


def test_error_statuses():
    from distributed_sigmoid_loss_b200 import _capi

    B, D = 300, 136
    p = Problem(B, D, seed=13)
    eng = _engine(B, D)
    img, txt = p.img.to(_dev()), p.texts[0].to(_dev())
    with pytest.raises(_capi.SiglipError) as e:   # the mode without siglip_set_groups since the previous step
        eng.fwd_bwd(img, txt, _scal(TP), _scal(BIAS))
    assert e.value.code == _capi.SIGLIP_ERR_STATE
    p.step(eng)   # the refused step consumed nothing: the next one runs
    off = _engine(B, D, groups=False)
    g = torch.zeros(B, dtype=torch.int64, device=_dev())
    with pytest.raises(_capi.SiglipError) as e:
        off.set_groups(g, g)
    assert e.value.code == _capi.SIGLIP_ERR_STATE
    L = _capi.lib()
    assert L.siglip_ctx_set_option(eng._h, _capi.SIGLIP_OPT_DISTILL, 1) == _capi.SIGLIP_ERR_STATE
    eng.set_groups(g, g)
    with pytest.raises(_capi.SiglipError) as e:
        eng.fwd_bwd_host(p.img, p.texts[0], TP, BIAS)
    assert e.value.code == _capi.SIGLIP_ERR_STATE
