"""Multi-label positives (SIGLIP_OPT_LABEL_SETS, DDPSigmoidLoss / SigLipLoss(multi_label=M)) on the H100. Random label
sets (hierarchies and tags) are checked against the float64 oracle of tests/label_sets_oracle.py at logits where the
set positives carry real weight (clustered embeddings, bias -5), for the loss, the gradients, dt', dbias, the per-sample
losses and the retrieval outputs. M = 1 sets are checked bit for bit against multi_positive with the same ids, padded
sets against the unpadded ones, and a captured CUDA graph against the eager step."""
import math

import numpy as np
import pytest
import torch

from exclude_groups_oracle import closed_form_groups, clustered, group_labels, torch_loss
from label_sets_oracle import dense_labels, hierarchy_sets, meet, topk_retrieval_sets
from retrieval_metrics_oracle import key_as_int64, metric_key

pytestmark = pytest.mark.gpu

TOL = 1e-3
TP, BIAS = math.log(10.0), -5.0
CLUSTERS = [(1, 1), (2, 1), (2, 2)]
# a 4-level hierarchy over 24 leaves: leaf 100 + i, parent 50 + i // 3, grandparent 20 + i // 6, root i // 12
PARENTS = {**{100 + i: 50 + i // 3 for i in range(24)}, **{50 + i: 20 + i // 2 for i in range(8)},
           **{20 + i: i // 2 for i in range(4)}}


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


def _engine(B, D, M=2, W=1, r=0, cg=2, mcast=1, stages=0, Ts=None, Rs=None, weights=False, groups=False, budget=None,
            labels=True, ids=False, input_f16=False, bidir=False, Bs=None):
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi

    eng = SigmoidLossEngine(B, D, _dev(), cta_group=cg, rank_world=(r, W), loopback=W > 1, texts_per_rank=Ts,
                            images_per_rank=Rs, labels=M if labels else 0, batch_per_rank=Bs)
    if mcast != 1:
        eng.set_option(_capi.SIGLIP_OPT_MCAST, mcast)
    if stages:
        eng.set_option(_capi.SIGLIP_OPT_STAGES_LOSS, stages)
    if labels:
        eng.set_option(_capi.SIGLIP_OPT_LABEL_SETS, 1)
    if ids:
        eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 1)
        if Ts is not None:
            eng.set_option(_capi.SIGLIP_OPT_EXTRA_TEXT_IDS, 1)
        if Rs is not None:
            eng.set_option(_capi.SIGLIP_OPT_EXTRA_IMAGE_IDS, 1)
    if weights:
        eng.set_option(_capi.SIGLIP_OPT_SAMPLE_WEIGHTS, 1)
    if groups:
        eng.set_option(_capi.SIGLIP_OPT_EXCLUDE_GROUPS, 1)
    if input_f16:
        eng.set_option(_capi.SIGLIP_OPT_INPUT_F16, 1)
    if bidir:
        eng.set_option(_capi.SIGLIP_OPT_BIDIR, 1)
    if budget:
        eng.set_sigma_budget(budget)
    eng.weighted, eng.grouped, eng.labelled, eng.with_ids = weights, groups, labels, ids
    return eng


def _sets(rng, n, M, kind):
    """[n, M] sets: 'tree' = the hierarchy's chain from a random leaf (M levels), 'tags' = M random tags of 40 with
    empty slots, 'one' = one label of 12 then empty slots."""
    if kind == "tree":
        return hierarchy_sets(rng.integers(100, 124, n), PARENTS, M)
    if kind == "tags":
        s = rng.integers(0, 40, (n, M))
        s[rng.random((n, M)) < 0.3] = -1
        return s
    s = np.full((n, M), -1, np.int64)
    s[:, 0] = rng.integers(0, 12, n)
    return s


class Problem:
    """Rank r of a W-rank job: W text chunks (B_c paired texts + K extras each), this rank's B + E images, label sets of
    the given kind (extras carry their own), embeddings clustered around each sample's first label."""

    def __init__(self, Bs, D, M, W=1, r=0, K=0, E=0, kind="tree", weights=False, groups=False, seed=0):
        rng = np.random.default_rng(seed)
        self.Bs, self.D, self.M, self.W, self.r, self.K, self.E = list(Bs), D, M, W, r, K, E
        self.B = Bs[r]
        self.Ts, self.Rs = [b + K for b in Bs], [b + E for b in Bs]
        ps = [_sets(rng, b, M, kind) for b in Bs]
        self.tsets = [np.concatenate([ps[c], _sets(rng, K, M, kind)]) for c in range(W)]
        self.isets = np.concatenate([ps[r], _sets(rng, E, M, kind)])
        # every rank's image sets (the peers' extra images are ranked in the retrieval outputs)
        self.all_isets = [np.concatenate([ps[q], _sets(np.random.default_rng(seed + 77 + q), E, M, kind)])
                          for q in range(W)]
        self.all_isets[r] = self.isets
        key = lambda s: np.where(s[:, 0] >= 0, s[:, 0], np.arange(len(s)) + 1000)  # noqa: E731
        emb = lambda s, q: torch.from_numpy(clustered(key(s), D, 16, seed, q)).float().to(torch.bfloat16)  # noqa: E731
        self.texts = [emb(self.tsets[c], 1000 * seed + c + 1) for c in range(W)]
        self.img = emb(self.isets, 1000 * seed + 999)
        # every rank's images (the peers' only enter the float64 retrieval oracle)
        self.all_imgs = [self.img if q == r else emb(self.all_isets[q], 1000 * seed + 900 + q) for q in range(W)]
        self.iw = self.tws = None
        if weights:
            self.iw = torch.from_numpy(rng.random(self.Rs[r])).float()
            self.tws = [torch.from_numpy(rng.random(t)).float() for t in self.Ts]
        self.ig = self.tg = None
        if groups:
            self.ig = rng.integers(-1, 5, self.Rs[r])
            self.tg = [rng.integers(-1, 5, t) for t in self.Ts]

    def oracle(self, sets=True):
        imgs = [self.img.double().numpy()]
        txts = [t.double().numpy() for t in self.texts]
        iws = None if self.iw is None else [self.iw.double().numpy()]
        tws = None if self.tws is None else [t.double().numpy() for t in self.tws]
        if sets:
            isets, tsets = [self.isets], self.tsets
        else:
            isets, tsets = [np.full_like(self.isets, -1)], [np.full_like(t, -1) for t in self.tsets]
        # one rank's rows: the own chunk of rank r is chunk r, so the oracle's rank 0 is given batch B_r on chunk r
        lab = _one_rank_labels(isets[0], tsets, self.r, self.B)
        if self.ig is not None:
            lab = group_labels(lab, [self.ig], self.tg)
        return closed_form_groups(imgs, txts, TP, BIAS, lab, [self.B], iws, tws)[0]

    def n_set_positives(self):
        lab = _one_rank_labels(self.isets, self.tsets, self.r, self.B)
        return sum(int((y > 0).sum()) for y in lab[0]) - self.B

    def seed_peers(self, eng):
        for k in range(self.W):
            eng.debug_set_text_chunk(k, self.texts[k].to(_dev()))
            if k == self.r:
                continue
            eng.debug_set_chunk_label_sets(k, torch.from_numpy(self.tsets[k]).to(_dev()))
            if eng.weighted:
                eng.debug_set_chunk_weights(k, self.tws[k].to(_dev()))
            if eng.grouped:
                eng.debug_set_chunk_groups(k, torch.from_numpy(self.tg[k]).to(_dev()))
            if self.E:
                xs = torch.from_numpy(self.all_isets[k][self.Bs[k]:]).to(_dev())
                eng.debug_set_peer_extra_image_label_sets(k, xs)

    def step(self, eng, sched="fused", losses=False, metrics_k=0, sets=None):
        """One step; returns its outputs by name (the contributions to the peers' chunks as slot<k>)."""
        r, B = self.r, self.B
        isets, tset = sets if sets is not None else (self.isets, self.tsets[r])
        if eng.labelled:
            xt = torch.from_numpy(np.ascontiguousarray(tset[B:])).to(_dev()) if self.K else None
            xi = torch.from_numpy(np.ascontiguousarray(isets[B:])).to(_dev()) if self.E else None
            eng.set_label_sets(torch.from_numpy(np.ascontiguousarray(isets[:B])).to(_dev()), xt, xi)
        if eng.with_ids:   # M = 1 sets as sample ids
            eng.set_sample_ids(torch.from_numpy(isets[:B, 0].copy()).to(_dev()))
            if self.K:
                eng.set_extra_text_ids(torch.from_numpy(tset[B:, 0].copy()).to(_dev()))
            if self.E:
                eng.set_extra_image_ids(torch.from_numpy(isets[B:, 0].copy()).to(_dev()))
        if eng.weighted:
            eng.set_sample_weights(self.iw.to(_dev()), self.tws[r].to(_dev()))
        if eng.grouped:
            eng.set_groups(torch.from_numpy(self.ig).to(_dev()), torch.from_numpy(self.tg[r]).to(_dev()))
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
        if eng.images_f32:
            img, txt = eng.convert_f32(img.float(), True), eng.convert_f32(txt.float(), True)
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

    def check_retrieval(self, tag, out, k, t2i_want=None):
        """Retrieval outputs of a step against the float64 oracle with the set-intersection hit rule
        (``topk_retrieval_sets``): the i2t lists of all R images of the rank exactly, on the rows whose float64
        similarities separate the K + 1 best candidates by more than 1e-4; the t2i lists of all T texts the same way, or
        exactly t2i_want ([T, k] global indices) where the peers' candidates are seeded in loopback. The recall the
        kernel reports must be, bit for bit, the one the set rule gives its own lists."""
        r, K = self.r, k
        exp = topk_retrieval_sets([x.double().numpy() for x in self.all_imgs], [t.double().numpy() for t in self.texts],
                                  self.Bs, K, self.all_isets, self.tsets)[r]
        S, off, toff = exp["S"], exp["off"], exp["toff"]
        Y = dense_labels(self.all_isets, self.tsets, self.Bs) > 0
        i2t = out["i2t_k"].cpu().numpy() if K > 1 else out["i2t"].cpu().numpy()[:, None]
        t2i = out["t2i_k"].cpu().numpy() if K > 1 else out["t2i"].cpu().numpy()[:, None]
        assert i2t.shape == (self.Rs[r], K) and t2i.shape == (self.Ts[r], K), (tag, i2t.shape, t2i.shape)

        def clear(v):
            top = np.sort(v)[::-1][:K + 1]
            return len(top) <= 1 or float(np.min(top[:-1] - top[1:])) > 1e-4

        ci = np.array([clear(S[off[r] + i]) for i in range(self.Rs[r])])
        assert ci.mean() > 0.8, (tag, ci.mean())
        np.testing.assert_array_equal(i2t[ci], exp["i2t_topk"][ci], err_msg=f"{tag} i2t lists")
        if t2i_want is None:
            ct = np.array([clear(S[:, toff[r] + i]) for i in range(self.Ts[r])])
            assert ct.mean() > 0.8, (tag, ct.mean())
            np.testing.assert_array_equal(t2i[ct], exp["t2i_topk"][ct], err_msg=f"{tag} t2i lists")
        else:
            np.testing.assert_array_equal(t2i, t2i_want, err_msg=f"{tag} t2i lists")
        fi = np.array([next((s for s, j in enumerate(row) if j >= 0 and Y[off[r] + i, j]), K)
                       for i, row in enumerate(i2t)])
        ft = np.array([next((s for s, g in enumerate(row) if g >= 0 and Y[g, toff[r] + i]), K)
                       for i, row in enumerate(t2i)])
        np.testing.assert_array_equal(fi[ci], exp["i2t_first"][ci], err_msg=f"{tag} i2t first hits")
        rec = out["recall"].cpu().numpy() if K > 1 else out["top1"].cpu().numpy()
        want_i = [np.float32(np.count_nonzero(fi < q)) / np.float32(len(fi)) for q in range(1, K + 1)]
        want_t = [np.float32(np.count_nonzero(ft < q)) / np.float32(len(ft)) for q in range(1, K + 1)]
        assert rec[:K].tolist() == want_i, (tag, rec[:K], want_i)
        assert rec[K:2 * K].tolist() == want_t, (tag, rec[K:], want_t)
        assert (fi < K).mean() > 0.2   # the set hits are exercised
        return ft


def _one_rank_labels(isets, tsets, r, B):
    out = []
    for c, st in enumerate(tsets):
        pos = meet(isets, st)
        if c == r:
            pos[np.arange(B), np.arange(B)] = True
        out.append(np.where(pos, 1.0, -1.0))
    return [out]


def _fresh(eng):
    eng.images_f32 = False
    return eng


# ---------------------------------------------------------------------------------------------------------------------
# 1. against the float64 oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sched", ["fused", "split"])
@pytest.mark.parametrize("stages", [4, 6])
@pytest.mark.parametrize("cg,mcast", CLUSTERS)
@pytest.mark.parametrize("B,D,M,kind", [(300, 136, 4, "tree"), (40, 1152, 2, "tags"), (257, 264, 1, "one")])
def test_random_sets_match_the_oracle(B, D, M, kind, cg, mcast, stages, sched):
    p = Problem([B], D, M, kind=kind, seed=B + D + M)
    assert p.n_set_positives() > B   # the test has set positives to get wrong
    eng = _fresh(_engine(B, D, M, cg=cg, mcast=mcast, stages=stages))
    ref = p.oracle()
    p.check(f"B={B} M={M} {kind} cg={cg} mc={mcast} st={stages} {sched}", p.step(eng, sched, losses=True), ref)
    # the set positives matter at these logits
    base = p.oracle(sets=False)
    assert _rel(ref["dimg"], base["dimg"]) > 20 * TOL and abs(ref["dbias"] - base["dbias"]) > 20 * TOL * abs(base["dbias"])


@pytest.mark.parametrize("K,E,weights,groups,M", [(37, 0, False, False, 2), (0, 23, True, False, 4),
                                                  (29, 19, True, True, 4), (0, 0, False, True, 1),
                                                  (13, 7, False, False, 1)])
def test_options_compose_with_label_sets(K, E, weights, groups, M):
    B, D = 300, 136
    p = Problem([B], D, M, K=K, E=E, kind="tags" if M > 1 else "one", weights=weights, groups=groups,
                seed=K + 3 * E + M)
    eng = _fresh(_engine(B, D, M, Ts=[B + K] if K else None, Rs=[B + E] if E else None, weights=weights,
                         groups=groups))
    ref = p.oracle()
    tag = f"K={K} E={E} w={weights} g={groups} M={M}"
    p.check(tag, p.step(eng, losses=True), ref)
    p.check(f"{tag} fwd", p.step(eng, "fwd"), ref)
    for k in (1, 5):
        p.check_retrieval(f"{tag} k={k}", p.step(eng, metrics_k=k), k)


@pytest.mark.parametrize("W,K,E,bidir,uneven", [(2, 0, 0, False, False), (3, 17, 0, True, False),
                                                (3, 0, 11, False, True), (2, 9, 5, True, True)])
@pytest.mark.parametrize("cg,mcast", [(2, 1), (1, 1)])
def test_loopback_peer_sets(W, K, E, bidir, uneven, cg, mcast):
    D, M = 264, 2
    Bs = [136, 200, 96][:W] if uneven else [136] * W
    r = W - 1
    p = Problem(Bs, D, M, W=W, r=r, K=K, E=E, kind="tags", weights=(W == 3), groups=(W == 2), seed=10 * W + K + E)
    eng = _fresh(_engine(Bs[r], D, M, W=W, r=r, cg=cg, mcast=mcast, Ts=p.Ts if K else None, Rs=p.Rs if E else None,
                         weights=(W == 3), groups=(W == 2), bidir=bidir, Bs=Bs))
    if uneven:
        assert eng.batch_per_rank == Bs
    p.seed_peers(eng)
    ref = p.oracle()
    for sched in ("fused", "split"):
        p.check(f"W={W} K={K} E={E} {sched}", p.step(eng, sched, losses=(sched == "fused")), ref)
    out = p.step(eng, metrics_k=1)
    assert out["i2t"].shape[0] == p.Rs[r] and out["t2i"].shape[0] == p.Ts[r]


def _peer_candidates(p, i, q, n, want_hit):
    """n local image indices of peer q for my text i, alternating paired and extra images (paired only without
    extras), the first one chosen to meet (want_hit) or miss the text's set where such an image exists."""
    R, B = p.Rs[q], p.Bs[q]
    tset = p.tsets[p.r][i:i + 1]
    order = np.random.default_rng(1000 * q + i).permutation(R).tolist()
    kinds = [l for l in order if (l >= B) == (i % 2 == 1 and R > B)] or order
    hits = meet(p.all_isets[q][kinds], tset)[:, 0]
    first = next((l for l, h in zip(kinds, hits) if h == want_hit), kinds[0])
    rest = [l for l in order if l != first]
    out = [first]
    for l in rest:   # then paired and extra images alternately
        if len(out) == n:
            break
        if R > B and (l >= B) != (out[-1] >= B) or R == B:
            out.append(l)
    for l in rest:
        if len(out) == n:
            break
        if l not in out:
            out.append(l)
    return out


@pytest.mark.parametrize("W,r,K,E,M", [(2, 0, 0, 23, 2), (3, 2, 17, 11, 4), (3, 1, 0, 19, 2)])
@pytest.mark.parametrize("k", [1, 4])
def test_loopback_retrieval_across_ranks(W, r, K, E, M, k):
    """Loopback at W = 2 and 3: the peers' column partials (K = 1) or top-K lists (K > 1) of my texts are seeded so
    that every t2i list is made of the peers' paired and extra images (scores beyond any real logit), and the peers'
    extra-image sets are seeded as they would publish them. Some winners meet my text's set and some miss it, among
    the paired images (judged by the gathered text sets) and among the extra images (judged by the published sets).
    The t2i lists must be the seeded ones exactly, the recall the set rule's; the i2t side is checked against the
    oracle over every chunk's texts."""
    from distributed_sigmoid_loss_b200.loss import TOPK_MAX

    D = 136
    Bs = [96, 128, 80][:W]
    p = Problem(Bs, D, M, W=W, r=r, K=K, E=E, kind="tags", seed=40 + 10 * W + r + k)
    eng = _fresh(_engine(Bs[r], D, M, W=W, r=r, Ts=p.Ts, Rs=p.Rs, Bs=Bs))
    p.seed_peers(eng)
    off = np.cumsum([0] + p.Rs)
    peers = [q for q in range(W) if q != r]
    T = p.Ts[r]
    lists = {q: np.zeros((T, TOPK_MAX), np.int64) for q in peers}
    cand = []   # per text: (score, global image index) of every seeded candidate
    for i in range(T):
        c = []
        for n, q in enumerate(peers):
            loc = _peer_candidates(p, i, q, k, want_hit=(i // 2) % 2 == 0)
            for s, l in enumerate(loc):
                sc = 20.0 - s - 0.5 * ((n + i) % len(peers))   # distinct across the peers' lists
                lists[q][i, s] = key_as_int64(metric_key(sc, off[q] + l))
                c.append((sc, off[q] + l))
        cand.append(sorted(c, key=lambda x: (-x[0], x[1]))[:k])
    want = np.array([[g for _, g in c] for c in cand], np.int64)
    for q in peers:
        if k == 1:
            eng.debug_set_peer_metric_keys(q, torch.from_numpy(lists[q][:, 0].copy()).to(_dev()))
        else:
            eng.debug_set_peer_topk_keys(q, torch.from_numpy(lists[q]).to(_dev()))
    out = p.step(eng, metrics_k=k)
    ft = p.check_retrieval(f"W={W} r={r} K={K} E={E} M={M} k={k}", out, k, t2i_want=want)
    # the winners cover peers' paired and extra images, hits and misses of both
    Y = dense_labels(p.all_isets, p.tsets, p.Bs) > 0
    toff = np.cumsum([0] + p.Ts)
    top = want[:, 0]
    owner = np.searchsorted(off, top, side="right") - 1
    extra = top - off[owner] >= np.array(p.Bs)[owner]
    hit = Y[top, toff[r] + np.arange(T)]
    for kind in (False, True):
        sel = extra == kind
        assert sel.sum() > 4 and 0 < hit[sel].sum() < sel.sum(), (kind, int(sel.sum()), int(hit[sel].sum()))
    assert (ft == 0).sum() == hit.sum()


def test_row_panels_under_a_sigma_budget():
    B, D, M = 1000, 136, 4
    p = Problem([B], D, M, E=40, kind="tree", weights=True, groups=True, seed=5)
    eng = _fresh(_engine(B, D, M, Rs=[B + 40], weights=True, groups=True, budget=1 << 20))
    assert eng.sigma_panels()[1] > 1
    ref = p.oracle()
    p.check("panels", p.step(eng, losses=True), ref)
    whole = _fresh(_engine(B, D, M, Rs=[B + 40], weights=True, groups=True))
    for k in (1, 4):
        a, b = p.step(eng, metrics_k=k, losses=True), p.step(whole, metrics_k=k, losses=True)
        for key in ("top1", "i2t", "t2i", "recall", "i2t_k", "t2i_k", "image_loss", "text_loss"):
            if key in a:
                assert torch.equal(a[key], b[key]), key
    W = 2
    p2 = Problem([B] * W, D, 2, W=W, r=1, kind="tags", seed=6)
    eng2 = _fresh(_engine(B, D, 2, W=W, r=1, budget=2 << 20))
    assert eng2.sigma_panels()[1] > 1
    p2.seed_peers(eng2)
    p2.check("panels W=2", p2.step(eng2, losses=True), p2.oracle())


def test_input_f16_engine():
    B, D, M = 300, 136, 2
    p = Problem([B], D, M, kind="tags", seed=14)
    eng = _fresh(_engine(B, D, M, input_f16=True))
    eng.images_f32 = True
    p.check("INPUT_F16", p.step(eng, losses=True), p.oracle())


# ---------------------------------------------------------------------------------------------------------------------
# 2. bit for bit
# ---------------------------------------------------------------------------------------------------------------------
ULP_KEYS = ("image_loss", "text_loss")


def _same(tag, a, b, ulp_ok=True):
    assert a.keys() == b.keys()
    bad = {k: float((a[k].double() - b[k].double()).abs().max()) for k in a if not torch.equal(a[k], b[k])}
    if ulp_ok:
        near = {k: v for k, v in bad.items() if k in ULP_KEYS and torch.allclose(a[k], b[k], rtol=1e-6, atol=0)}
        bad = {k: v for k, v in bad.items() if k not in near}
    assert not bad, f"{tag}: differs (max abs difference) {bad}"


@pytest.mark.parametrize("K,E", [(0, 0), (29, 0), (0, 23), (13, 19)])
@pytest.mark.parametrize("cg,mcast", [(2, 1), (1, 1)])
def test_m1_sets_are_bitwise_multi_positive(K, E, cg, mcast):
    """M = 1 sets with labels >= 0 give multi_positive's loss, gradients, dt', dbias, metrics and top-K lists bit for
    bit, and its per-sample losses to within a few ulps (the sums of the two instantiations round differently)."""
    B, D = 300, 136
    p = Problem([B], D, 1, K=K, E=E, kind="one", seed=7)
    kw = dict(cg=cg, mcast=mcast, Ts=[B + K] if K else None, Rs=[B + E] if E else None)
    on = _fresh(_engine(B, D, 1, **kw))
    ids = _fresh(_engine(B, D, 1, labels=False, ids=True, **kw))
    for sched in ("fused", "split", "fwd"):
        for k in (0, 1, 5):
            a = p.step(on, sched, losses=(sched == "fused"), metrics_k=k)
            b = p.step(ids, sched, losses=(sched == "fused"), metrics_k=k)
            _same(f"M=1 K={K} E={E} {sched} k={k}", a, b)


def test_loopback_m1_sets_are_bitwise_multi_positive():
    B, D, W, r, K = 136, 264, 3, 1, 11
    p = Problem([B] * W, D, 1, W=W, r=r, K=K, kind="one", seed=8)
    on = _fresh(_engine(B, D, 1, W=W, r=r, Ts=p.Ts))
    ids = _fresh(_engine(B, D, 1, W=W, r=r, Ts=p.Ts, labels=False, ids=True))
    p.seed_peers(on)
    for k in range(W):
        ids.debug_set_text_chunk(k, p.texts[k].to(_dev()))
        if k != r:
            ids.debug_set_chunk_ids(k, torch.from_numpy(p.tsets[k][:, 0].copy()).to(_dev()))
    _same("loopback", p.step(on, losses=True, metrics_k=5), p.step(ids, losses=True, metrics_k=5))


def test_padded_sets_are_bitwise_the_unpadded_ones():
    """A set with its labels is the same set padded with -1 slots and duplicates, at M = 1 and M = 4: every output bit
    for bit."""
    B, D, K, E = 300, 136, 21, 17
    p = Problem([B], D, 1, K=K, E=E, kind="one", weights=True, seed=15)
    rng = np.random.default_rng(3)

    def pad(s):
        out = np.full((len(s), 4), -1, np.int64)
        for i, x in enumerate(s[:, 0]):
            slots = rng.permutation(4)[:rng.integers(1, 4)]
            out[i, slots] = x
            out[i, out[i] < 0] = -rng.integers(1, 9, int((out[i] < 0).sum()))
        return out

    one = _fresh(_engine(B, D, 1, Ts=[B + K], Rs=[B + E], weights=True))
    four = _fresh(_engine(B, D, 4, Ts=[B + K], Rs=[B + E], weights=True))
    ps, ts = pad(p.isets), pad(p.tsets[0])
    ts[:B] = ps[:B]   # a sample's text shares its image's set
    p4 = Problem([B], D, 4, K=K, E=E, kind="one", weights=True, seed=15)
    p4.isets, p4.tsets = ps, [ts]
    p4.img, p4.texts, p4.iw, p4.tws = p.img, p.texts, p.iw, p.tws
    for sched in ("fused", "split"):
        for k in (0, 1, 5):
            a = p.step(one, sched, losses=(sched == "fused"), metrics_k=k)
            b = p4.step(four, sched, losses=(sched == "fused"), metrics_k=k)
            _same(f"padded {sched} k={k}", a, b, ulp_ok=False)


# ---------------------------------------------------------------------------------------------------------------------
# 3. capture, modules, errors
# ---------------------------------------------------------------------------------------------------------------------
def test_single_rank_step_captures_into_a_cuda_graph():
    B, D, M = 300, 136, 4
    p = Problem([B], D, M, kind="tree", seed=9)
    eng = _fresh(_engine(B, D, M))
    img, txt, tp, b = p.img.to(_dev()), p.texts[0].to(_dev()), _scal(TP), _scal(BIAS)
    sl = torch.from_numpy(p.isets).to(_dev())
    eager = p.step(eng)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):   # warm-up outside the capture
        eng.set_label_sets(sl)
        eng.fwd_bwd(img, txt, tp, b)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        eng.set_label_sets(sl)
        loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, tp, b)
    sl.fill_(-1)   # the replay reads the sets at replay time: first none, then the problem's again
    g.replay()
    torch.cuda.synchronize()
    assert not torch.equal(dimg, eager["dimg"])
    sl.copy_(torch.from_numpy(p.isets))
    g.replay()
    torch.cuda.synchronize()
    for k, v in (("loss", loss), ("dimg", dimg), ("dtxt", dtxt), ("dtp", dtp), ("db", db)):
        assert torch.equal(v, eager[k]), k


@pytest.mark.parametrize("dtype,normalize,M", [(torch.bfloat16, False, 2), (torch.float32, False, 4),
                                               (torch.float32, True, 1)])
def test_module_against_autograd_restatement(dtype, normalize, M):
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss

    B, D, K, E = 300, 136, 20, 12
    p = Problem([B], D, M, K=K, E=E, kind="tags" if M > 1 else "one", seed=11 + M)
    mod = DDPSigmoidLoss(B, normalize_inputs=normalize, extra_texts=K, extra_images=E, multi_label=M).to(_dev())
    with torch.no_grad():
        mod.bias.fill_(BIAS)
    scale = 3.0 if normalize else 1.0
    imgs = (p.img.float() * scale).to(dtype).to(_dev())
    txt = (p.texts[0].float() * scale).to(dtype).to(_dev())
    img, ximg = imgs[:B].clone().requires_grad_(True), imgs[B:].clone().requires_grad_(True)
    pos, xt = txt[:B].clone().requires_grad_(True), txt[B:].clone().requires_grad_(True)
    sets = torch.from_numpy(p.isets).to(_dev())
    tsets = torch.from_numpy(p.tsets[0]).to(_dev())
    loss, met, out = mod(img, pos, extra_text=xt, extra_image=ximg, sample_labels=sets[:B],
                         extra_text_labels=tsets[B:], extra_image_labels=sets[B:], return_sample_losses=True,
                         return_metrics=True, metrics_topk=3)
    loss.backward()
    y = torch.from_numpy(_one_rank_labels(p.isets, p.tsets, 0, B)[0][0])
    xi = torch.cat([img, ximg]).detach().double().cpu().requires_grad_(True)
    xtt = torch.cat([pos, xt]).detach().double().cpu().requires_grad_(True)
    tp = torch.tensor(TP, dtype=torch.float64, requires_grad=True)
    bb = torch.tensor(BIAS, dtype=torch.float64, requires_grad=True)
    ref = torch_loss(xi, xtt, tp, bb, y, normalize=normalize, batch=B)
    ref.backward()
    tol = 4e-3 if dtype == torch.bfloat16 else TOL
    _check("module loss", loss.detach(), ref.detach(), tol)
    _check("module dimg", torch.cat([img.grad, ximg.grad]), xi.grad, tol)
    _check("module dtxt", torch.cat([pos.grad, xt.grad]), xtt.grad, tol)
    _check("module dt'", mod.t_prime.grad, tp.grad, tol)
    _check("module dbias", mod.bias.grad, bb.grad, tol)
    assert float(out["image_loss"].sum()) == pytest.approx(float(loss) * B, rel=1e-4)
    assert out["image_loss"].shape[0] == B + E and out["text_loss"].shape[0] == B + K
    # the metrics rank every image and every text of the rank, extras included
    assert met["i2t_index"].shape[0] == met["i2t_topk"].shape[0] == B + E
    assert met["t2i_index"].shape[0] == met["t2i_topk"].shape[0] == B + K


def test_siglip_loss_matches_ddp_module():
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    B, D, M = 300, 136, 4
    p = Problem([B], D, M, kind="tree", seed=12)
    sets = torch.from_numpy(p.isets).to(_dev())
    img, txt = p.img.to(_dev()), p.texts[0].to(_dev())
    ddp = DDPSigmoidLoss(B, multi_label=M).to(_dev())
    with torch.no_grad():
        ddp.bias.fill_(BIAS)
    a = ddp(img, txt, sample_labels=sets)
    b = SigLipLoss(multi_label=M)(img, txt, torch.tensor(TP, device=_dev()), torch.tensor(BIAS, device=_dev()),
                                  sample_labels=sets)
    assert float(a) == pytest.approx(float(b), rel=1e-5)
    _check("siglip vs oracle", b, p.oracle()["loss"])


def test_error_statuses():
    from distributed_sigmoid_loss_b200 import _capi

    B, D, M = 300, 136, 2
    p = Problem([B], D, M, kind="tags", seed=13)
    eng = _fresh(_engine(B, D, M))
    img, txt = p.img.to(_dev()), p.texts[0].to(_dev())
    with pytest.raises(_capi.SiglipError) as e:   # the mode without siglip_set_label_sets since the previous step
        eng.fwd_bwd(img, txt, _scal(TP), _scal(BIAS))
    assert e.value.code == _capi.SIGLIP_ERR_STATE
    p.step(eng)   # the refused step consumed nothing: the next one runs
    L = _capi.lib()
    for opt in (_capi.SIGLIP_OPT_SAMPLE_IDS, _capi.SIGLIP_OPT_EXTRA_TEXT_IDS, _capi.SIGLIP_OPT_EXTRA_IMAGE_IDS,
                _capi.SIGLIP_OPT_DISTILL):
        assert L.siglip_ctx_set_option(eng._h, opt, 1) == _capi.SIGLIP_ERR_STATE
    s = torch.from_numpy(p.isets).to(_dev())
    eng.set_label_sets(s)
    with pytest.raises(_capi.SiglipError) as e:
        eng.fwd_bwd_host(p.img, p.texts[0], TP, BIAS)
    assert e.value.code == _capi.SIGLIP_ERR_STATE
    # a context created without label sets refuses the option, and its setter
    off = _fresh(_engine(B, D, M, labels=False))
    assert L.siglip_ctx_set_option(off._h, _capi.SIGLIP_OPT_LABEL_SETS, 1) == _capi.SIGLIP_ERR_STATE
    assert L.siglip_set_label_sets(off._h, s.data_ptr(), None, None, None) == _capi.SIGLIP_ERR_STATE
    # a labels context with sample ids on refuses the option until they are off
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine

    both = SigmoidLossEngine(B, D, _dev(), labels=M)
    both.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 1)
    assert L.siglip_ctx_set_option(both._h, _capi.SIGLIP_OPT_LABEL_SETS, 1) == _capi.SIGLIP_ERR_STATE
    both.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 0)
    both.set_option(_capi.SIGLIP_OPT_LABEL_SETS, 1)
