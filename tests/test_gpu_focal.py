"""The focal pair loss (SIGLIP_OPT_FOCAL, DDPSigmoidLoss / SigLipLoss(focal_gamma=, focal_alpha=)) on the H100, against
the float64 oracle of tests/focal_oracle.py: gamma in {0, 0.5, 2, 5} x alpha in {None, 0.25}, every kModeFocal
instantiation, both schedules, bidir, row panels, fp32 and bf16 inputs, both gradient tile widths, every option it
composes with, loopback ranks, trained-model logits, non-finite inputs, weight-0 samples, bitwise repeatability and
the refusals. Problems, engines and loopback seeding are those of tests/test_gpu_label_sets.py; only the loss changes.
`pytest -s` prints the largest relative error of each group and the difference between the focal kernel at gamma = 0
(no alpha) and the plain step.

Observed on one H100 80GB HBM3 (700 W), largest relative error per group (the file runs in about 20 s there):
  against the oracle (every case but those below)       2.0e-4   TOL 1e-3
  trained-model logits, trained / t300                  3.9e-5 / 4.4e-5
  modules against autograd (bf16 inputs: 4e-3)          3.6e-3
  gamma = 0 without alpha against the plain step        0 (identical outputs at biases -5 and -10)"""
import math

import numpy as np
import pytest
import torch

from exclude_groups_oracle import group_labels, operand_values
from focal_oracle import closed_form_focal, torch_focal_loss
from test_gpu_label_sets import BIAS, CLUSTERS, TP, Problem, _dev, _engine, _fresh, _one_rank_labels, _rel, _scal
from trained_regime import REGIMES, make_batch

pytestmark = pytest.mark.gpu

TOL = 1e-3
GAMMAS = (0.0, 0.5, 2.0, 5.0)
ALPHAS = (None, 0.25)
INSTANCES = [(cg, mc, st) for cg, mc in CLUSTERS for st in (4, 6)]
_OBSERVED = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(_OBSERVED):
        print(f"focal: {k}: {_OBSERVED[k]:.3e}")


def _note(key, err):
    _OBSERVED[key] = max(_OBSERVED.get(key, 0.0), err)


def _check(group, name, got, ref, tol=TOL):
    err = _rel(got, ref)
    _note(f"{group} max error", err)
    assert err <= tol, f"{group} {name}: relative error {err:.3e}"


def _focal(eng, gamma, alpha):
    from distributed_sigmoid_loss_b200 import _capi

    eng.set_option(_capi.SIGLIP_OPT_FOCAL, 1)
    eng.set_focal(gamma, alpha)
    return eng


class FocalProblem(Problem):
    """The label-set Problem with the focal oracle: labels as the engine's options give them (label sets, the sets'
    first labels as sample ids, or positional with hard negatives), excluded groups after them."""

    def focal_oracle(self, gamma, alpha, sets=True):
        imgs = [self.img.double().numpy()]
        txts = [t.double().numpy() for t in self.texts]
        iws = None if self.iw is None else [self.iw.double().numpy()]
        tws = None if self.tws is None else [t.double().numpy() for t in self.tws]
        if sets:
            lab = _one_rank_labels(self.isets, self.tsets, self.r, self.B)
        else:
            lab = _one_rank_labels(np.full_like(self.isets, -1), [np.full_like(t, -1) for t in self.tsets], self.r,
                                   self.B)
        if self.ig is not None:
            lab = group_labels(lab, [self.ig], self.tg)
        return closed_form_focal(imgs, txts, TP, BIAS, lab, gamma, alpha, [self.B], iws, tws)[0]

    def seed_peers(self, eng):
        """The peers' text chunks, and their label sets, weights, groups and extra-image sets where the engine takes
        them."""
        for k in range(self.W):
            eng.debug_set_text_chunk(k, self.texts[k].to(_dev()))
            if k == self.r:
                continue
            if eng.labelled:
                eng.debug_set_chunk_label_sets(k, torch.from_numpy(self.tsets[k]).to(_dev()))
                if self.E:
                    xs = torch.from_numpy(self.all_isets[k][self.Bs[k]:]).to(_dev())
                    eng.debug_set_peer_extra_image_label_sets(k, xs)
            if eng.weighted:
                eng.debug_set_chunk_weights(k, self.tws[k].to(_dev()))
            if eng.grouped:
                eng.debug_set_chunk_groups(k, torch.from_numpy(self.tg[k]).to(_dev()))

    def check(self, tag, out, ref, tol=TOL, group="oracle"):
        _check(group, f"{tag} loss", out["loss"], ref["loss"], tol)
        if "dimg" in out:
            _check(group, f"{tag} dimg", out["dimg"], ref["dimg"], tol)
            _check(group, f"{tag} dt_prime", out["dtp"], ref["dt_prime"], tol)
            _check(group, f"{tag} dbias", out["db"], ref["dbias"], tol)
            for k in range(self.W):
                got = out["dtxt"] if k == self.r else out[f"slot{k}"]
                _check(group, f"{tag} contribution to chunk {k}", got, ref["contrib"][k], tol)
        if "image_loss" in out:
            _check(group, f"{tag} image_loss", out["image_loss"], ref["image_loss"], tol)
            if self.W == 1:
                _check(group, f"{tag} text_loss", out["text_loss"], ref["text_part"][0], tol)


# ---------------------------------------------------------------------------------------------------------------------
# 1. against the float64 oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alpha", ALPHAS)
@pytest.mark.parametrize("gamma", GAMMAS)
def test_gamma_alpha_grid(gamma, alpha):
    """Positional labels, every instantiation in turn, fused and split steps with per-sample losses."""
    B, D = 300, 136
    n = GAMMAS.index(gamma) * len(ALPHAS) + ALPHAS.index(alpha)
    cg, mc, st = INSTANCES[n % len(INSTANCES)]
    p = FocalProblem([B], D, 2, kind="tags", seed=n + 1)
    eng = _focal(_fresh(_engine(B, D, cg=cg, mcast=mc, stages=st, labels=False)), gamma, alpha)
    ref = p.focal_oracle(gamma, alpha, sets=False)
    for sched in ("fused", "split"):
        p.check(f"gamma={gamma} alpha={alpha} cg={cg} mc={mc} st={st} {sched}", p.step(eng, sched, losses=True), ref)
    if gamma > 0:   # the focal terms matter at these logits
        plain = p.focal_oracle(0.0, None, sets=False)
        assert _rel(ref["dimg"], plain["dimg"]) > 20 * TOL


@pytest.mark.parametrize("cg,mc,st", INSTANCES)
def test_every_instantiation_with_label_sets_groups_and_weights(cg, mc, st):
    B, D, M, K, E = 300, 136, 2, 29, 19
    p = FocalProblem([B], D, M, K=K, E=E, kind="tags", weights=True, groups=True, seed=20 + cg + 3 * mc + st)
    eng = _focal(_fresh(_engine(B, D, M, cg=cg, mcast=mc, stages=st, Ts=[B + K], Rs=[B + E], weights=True,
                                groups=True)), 2.0, 0.25)
    ref = p.focal_oracle(2.0, 0.25)
    for sched in ("fused", "split", "fwd"):
        p.check(f"cg={cg} mc={mc} st={st} {sched}", p.step(eng, sched, losses=(sched != "fwd")), ref)


@pytest.mark.parametrize("K,E,weights,groups,M,ids,sets", [
    (37, 0, False, False, 2, False, False),    # hard negatives
    (0, 23, True, False, 4, False, False),     # hard-negative images, weights
    (29, 19, True, True, 4, False, True),      # label sets with extras, weights, groups
    (0, 0, False, True, 1, False, False),      # groups alone
    (13, 7, True, False, 1, True, True),       # multi_positive with extra texts and images (ids = the M = 1 sets)
])
def test_options_compose_with_focal(K, E, weights, groups, M, ids, sets):
    B, D, gamma, alpha = 300, 136, 2.0, 0.25
    p = FocalProblem([B], D, M, K=K, E=E, kind="tags" if M > 1 else "one", weights=weights, groups=groups,
                     seed=K + 3 * E + M)
    eng = _focal(_fresh(_engine(B, D, M, Ts=[B + K] if K else None, Rs=[B + E] if E else None, weights=weights,
                                groups=groups, labels=sets and not ids, ids=ids)), gamma, alpha)
    ref = p.focal_oracle(gamma, alpha, sets=sets)
    tag = f"K={K} E={E} w={weights} g={groups} M={M} ids={ids} sets={sets}"
    p.check(tag, p.step(eng, losses=True), ref)
    p.check(f"{tag} fwd", p.step(eng, "fwd"), ref)
    # metrics and top-K lists ignore the loss: the same bits as the step without focal
    plain = _fresh(_engine(B, D, M, Ts=[B + K] if K else None, Rs=[B + E] if E else None, weights=weights,
                           groups=groups, labels=sets and not ids, ids=ids))
    for k in (1, 5):
        a, b = p.step(eng, metrics_k=k), p.step(plain, metrics_k=k)
        for key in ("top1", "i2t", "t2i", "recall", "i2t_k", "t2i_k"):
            if key in a:
                assert torch.equal(a[key], b[key]), (tag, k, key)


@pytest.mark.parametrize("W,K,E,bidir,uneven", [(2, 0, 0, False, False), (3, 17, 0, True, False),
                                                (3, 0, 11, False, True), (2, 9, 5, True, True)])
@pytest.mark.parametrize("cg,mcast", [(2, 1), (1, 1)])
def test_loopback_ranks(W, K, E, bidir, uneven, cg, mcast):
    D, M = 264, 2
    Bs = [136, 200, 96][:W] if uneven else [136] * W
    r = W - 1
    sets = (W == 3)
    p = FocalProblem(Bs, D, M, W=W, r=r, K=K, E=E, kind="tags", weights=(W == 3), groups=(W == 2),
                     seed=10 * W + K + E)
    eng = _focal(_fresh(_engine(Bs[r], D, M, W=W, r=r, cg=cg, mcast=mcast, Ts=p.Ts if K else None,
                                Rs=p.Rs if E else None, weights=(W == 3), groups=(W == 2), bidir=bidir, Bs=Bs,
                                labels=sets)), 5.0 if bidir else 0.5, None if uneven else 0.25)
    p.seed_peers(eng)
    ref = p.focal_oracle(5.0 if bidir else 0.5, None if uneven else 0.25, sets=sets)
    for sched in ("fused", "split"):
        p.check(f"W={W} K={K} E={E} bidir={bidir} {sched}", p.step(eng, sched, losses=(sched == "fused")), ref)


def test_row_panels_under_a_sigma_budget():
    B, D, M = 1000, 136, 4
    p = FocalProblem([B], D, M, E=40, kind="tree", weights=True, groups=True, seed=5)
    eng = _focal(_fresh(_engine(B, D, M, Rs=[B + 40], weights=True, groups=True, budget=1 << 20)), 2.0, 0.25)
    assert eng.sigma_panels()[1] > 1
    p.check("panels", p.step(eng, losses=True), p.focal_oracle(2.0, 0.25))
    whole = _focal(_fresh(_engine(B, D, M, Rs=[B + 40], weights=True, groups=True)), 2.0, 0.25)
    a, b = p.step(eng, losses=True), p.step(whole, losses=True)
    for key in ("image_loss", "text_loss"):
        assert torch.equal(a[key], b[key]), key
    W = 2
    p2 = FocalProblem([B] * W, D, 2, W=W, r=1, kind="tags", seed=6)
    eng2 = _focal(_fresh(_engine(B, D, 2, W=W, r=1, budget=2 << 20, labels=False)), 0.5, None)
    assert eng2.sigma_panels()[1] > 1
    p2.seed_peers(eng2)
    p2.check("panels W=2", p2.step(eng2, losses=True), p2.focal_oracle(0.5, None, sets=False))


def test_input_f16_engine():
    B, D, M = 300, 136, 2
    p = FocalProblem([B], D, M, kind="tags", seed=14)
    eng = _focal(_fresh(_engine(B, D, M, input_f16=True)), 2.0, None)
    eng.images_f32 = True
    p.check("INPUT_F16", p.step(eng, losses=True), p.focal_oracle(2.0, None))


@pytest.mark.parametrize("tile_n", [128, 256])
def test_gradient_tile_widths(tile_n):
    from distributed_sigmoid_loss_b200 import _capi

    B, D = 1024, 264
    p = FocalProblem([B], D, 2, kind="tags", seed=30)
    eng = _focal(_fresh(_engine(B, D, labels=False)), 2.0, 0.25)
    eng.set_option(_capi.SIGLIP_OPT_GRAD_TILE_N, tile_n)
    p.check(f"grad tiles {tile_n}", p.step(eng), p.focal_oracle(2.0, 0.25, sets=False))


@pytest.mark.parametrize("gamma,alpha", [(2.0, 0.25), (5.0, None), (0.5, None)])
@pytest.mark.parametrize("regime", ["trained", "t300"])
def test_trained_model_logits(regime, gamma, alpha):
    """Logits of a trained model (tests/trained_regime.py): the negatives carry the gradient, and the series and
    general paths share every tile. Under focal the easy negatives' g * 2^14 lies deep in fp16's subnormals or
    flushes to 0 (DESIGN.md, "Focal pair loss"); the result must stay within the tolerance all the same."""
    reg = REGIMES[regime]
    B, D = 1024, 264
    imgs, texts, _, _ = make_batch(reg, [B], [0], D, seed=3)
    eng = _focal(_fresh(_engine(B, D, labels=False)), gamma, alpha)
    tp = math.log(reg.t)
    img, txt = imgs[0].to(_dev()), texts[0].to(_dev())
    loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, _scal(tp), _scal(reg.bias))
    torch.cuda.synchronize()
    lab = [[np.where(np.eye(B) > 0, 1.0, -1.0)]]
    ref = closed_form_focal([imgs[0].double().numpy()], [texts[0].double().numpy()], tp, reg.bias, lab, gamma,
                            alpha)[0]
    g = f"trained-model logits ({regime})"
    _check(g, "loss", loss, ref["loss"])
    _check(g, "dimg", dimg, ref["dimg"])
    _check(g, "dtxt", dtxt, ref["contrib"][0])
    # dt' and dbias cancel between the positives and the negatives: against their scale
    t = reg.t
    S = imgs[0].double().numpy() @ texts[0].double().numpy().T
    from focal_oracle import focal_terms

    _, gz = focal_terms(t * S + reg.bias, lab[0][0], gamma, alpha)
    assert abs(float(db) - ref["dbias"]) <= TOL * np.abs(gz).sum() / B
    assert abs(float(dtp) - ref["dt_prime"]) <= TOL * t * np.abs(gz * S).sum() / B


# ---------------------------------------------------------------------------------------------------------------------
# 2. semantics: gamma = 0, weight 0, non-finite inputs
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bias", [BIAS, -10.0])
def test_gamma_zero_without_alpha_is_the_plain_step(bias):
    """The focal kernel at gamma = 0 without alpha, through the C ABI, against the plain step: the same loss within
    float rounding (the focal epilogue forms sigma and softplus in another order)."""
    B, D = 1024, 264
    p = FocalProblem([B], D, 2, kind="tags", seed=41)
    img, txt = p.img.to(_dev()), p.texts[0].to(_dev())
    foc = _focal(_fresh(_engine(B, D, labels=False)), 0.0, None)
    plain = _fresh(_engine(B, D, labels=False))
    a = foc.fwd_bwd(img, txt, _scal(TP), _scal(bias))
    b = plain.fwd_bwd(img, txt, _scal(TP), _scal(bias))
    torch.cuda.synchronize()
    for name, x, y in zip(("loss", "dimg", "dtxt", "dt_prime", "dbias"), a, b):
        err = _rel(x, y)
        _note(f"gamma=0 vs plain step (bias {bias}) {name}", err)
        assert err <= 1e-4, (name, err)


def test_weight_zero_samples_drop_out_exactly():
    from distributed_sigmoid_loss_b200 import _capi

    B, D, K = 300, 136, 13
    p = FocalProblem([B], D, 2, K=K, kind="tags", weights=True, seed=17)
    drop = np.arange(0, B, 7)
    p.iw[drop] = 0.0
    p.tws[0][drop] = 0.0
    eng = _focal(_fresh(_engine(B, D, 2, Ts=[B + K], weights=True)), 2.0, 0.25)
    out = p.step(eng, losses=True)
    assert (out["dimg"][drop] == 0).all() and (out["dtxt"][drop] == 0).all()
    assert (out["image_loss"][drop] == 0).all() and (out["text_loss"][drop] == 0).all()
    p.check("weight 0", out, p.focal_oracle(2.0, 0.25))
    # the same loss as the batch without those samples, rescaled by B / (B - m)
    keep = np.setdiff1d(np.arange(B), drop)
    q = FocalProblem([len(keep)], D, 2, K=K, kind="tags", weights=True, seed=17)
    q.isets = np.concatenate([p.isets[keep], p.isets[B:]])
    q.tsets = [np.concatenate([p.tsets[0][keep], p.tsets[0][B:]])]
    q.img = p.img[keep]
    q.texts = [torch.cat([p.texts[0][keep], p.texts[0][B:]])]
    q.iw = p.iw[keep]
    q.tws = [torch.cat([p.tws[0][keep], p.tws[0][B:]])]
    small = _focal(_fresh(_engine(len(keep), D, 2, Ts=[len(keep) + K], weights=True)), 2.0, 0.25)
    ls = q.step(small)
    assert float(out["loss"]) * B == pytest.approx(float(ls["loss"]) * len(keep), rel=1e-5)
    assert _capi.SIGLIP_OPT_FOCAL == 29


@pytest.mark.parametrize("where", ["image_nan", "text_inf", "neg_inf"])
def test_non_finite_inputs(where):
    """DESIGN.md "Non-finite inputs": every output is non-finite exactly where float64 autograd of the loss on the
    operand values is (the focal terms in the form of ``torch_focal_terms``), and within the tolerance elsewhere. An
    infinite text entry makes z = +inf (g NaN, as autograd) and z = -inf (term and g 0, the limit) in one column."""
    B, D, gamma, alpha = 256, 136, 2.0, 0.25
    p = FocalProblem([B], D, 2, kind="tags", seed=23)
    img, txt = p.img.clone(), p.texts[0].clone()
    if where == "image_nan":
        img[5, 3] = float("nan")
    elif where == "text_inf":
        txt[9, 0] = float("inf")
    else:
        img[2, 1] = float("-inf")
    eng = _focal(_fresh(_engine(B, D, labels=False)), gamma, alpha)
    loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img.to(_dev()), txt.to(_dev()), _scal(TP), _scal(BIAS))
    torch.cuda.synchronize()
    xi = operand_values(img).requires_grad_(True)
    xt = operand_values(txt).requires_grad_(True)
    tp = torch.tensor(TP, dtype=torch.float64, requires_grad=True)
    bb = torch.tensor(BIAS, dtype=torch.float64, requires_grad=True)
    y = torch.where(torch.eye(B, dtype=torch.bool), 1.0, -1.0).double()
    ref = torch_focal_loss(xi, xt, tp, bb, y, gamma, alpha)
    ref.backward()
    for name, got, want in (("loss", loss, ref.detach()), ("dimg", dimg, xi.grad), ("dtxt", dtxt, xt.grad),
                            ("dt_prime", dtp, tp.grad), ("dbias", db, bb.grad)):
        got, want = got.double().cpu().reshape(want.shape), want.double()
        bad = ~torch.isfinite(want)
        assert torch.equal(~torch.isfinite(got), bad), (where, name, int(bad.sum()), int((~torch.isfinite(got)).sum()))
        if (~bad).any() and bad.any():
            assert _rel(got[~bad], want[~bad]) <= TOL, (where, name)


# ---------------------------------------------------------------------------------------------------------------------
# 3. bit for bit
# ---------------------------------------------------------------------------------------------------------------------
def test_repeated_steps_are_bitwise_identical_and_sample_losses_across_schedules():
    B, D, M, K, E = 300, 136, 2, 21, 9
    p = FocalProblem([B], D, M, K=K, E=E, kind="tags", weights=True, groups=True, seed=19)
    eng = _focal(_fresh(_engine(B, D, M, Ts=[B + K], Rs=[B + E], weights=True, groups=True)), 5.0, 0.25)
    first = p.step(eng, losses=True, metrics_k=3)
    again = p.step(eng, losses=True, metrics_k=3)
    for k in first:
        assert torch.equal(first[k], again[k]), k
    losses = [p.step(eng, s, losses=True) for s in ("fused", "split", "fwd")]
    for o in losses[1:]:
        assert torch.equal(o["image_loss"], losses[0]["image_loss"])
        assert torch.equal(o["text_loss"], losses[0]["text_loss"])
    # and under the other instantiations
    for cg, mc, st in INSTANCES[1:]:
        other = _focal(_fresh(_engine(B, D, M, cg=cg, mcast=mc, stages=st, Ts=[B + K], Rs=[B + E], weights=True,
                                      groups=True)), 5.0, 0.25)
        o = p.step(other, losses=True)
        assert torch.equal(o["image_loss"], losses[0]["image_loss"]), (cg, mc, st)
        assert torch.equal(o["text_loss"], losses[0]["text_loss"]), (cg, mc, st)


# ---------------------------------------------------------------------------------------------------------------------
# 4. modules and refusals
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,normalize,sync,bpr", [(torch.bfloat16, False, False, False),
                                                      (torch.float32, False, True, True),
                                                      (torch.float32, True, False, False)])
def test_module_against_autograd_restatement(dtype, normalize, sync, bpr):
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss

    B, D, K, E, M = 300, 136, 20, 12, 2
    gamma, alpha = 2.0, 0.25
    p = FocalProblem([B], D, M, K=K, E=E, kind="tags", seed=31)
    mod = DDPSigmoidLoss(B, normalize_inputs=normalize, extra_texts=K, extra_images=E, multi_label=M,
                         sync_scalar_grads=sync, batch_per_rank=[B] if bpr else None, focal_gamma=gamma,
                         focal_alpha=alpha).to(_dev())
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
    ref = torch_focal_loss(xi, xtt, tp, bb, y, gamma, alpha, normalize=normalize, batch=B)
    ref.backward()
    tol = 4e-3 if dtype == torch.bfloat16 else TOL
    g = "module"
    _check(g, "loss", loss.detach(), ref.detach(), tol)
    _check(g, "dimg", torch.cat([img.grad, ximg.grad]), xi.grad, tol)
    _check(g, "dtxt", torch.cat([pos.grad, xt.grad]), xtt.grad, tol)
    _check(g, "dt'", mod.t_prime.grad, tp.grad, tol)
    _check(g, "dbias", mod.bias.grad, bb.grad, tol)
    assert float(out["image_loss"].sum()) == pytest.approx(float(loss) * B, rel=1e-4)
    assert met["i2t_topk"].shape == (B + E, 3)


def test_siglip_loss_matches_ddp_module_and_none_is_unchanged():
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    B, D = 300, 136
    p = FocalProblem([B], D, 2, kind="tags", seed=12)
    img, txt = p.img.to(_dev()), p.texts[0].to(_dev())
    ddp = DDPSigmoidLoss(B, focal_gamma=0.5).to(_dev())
    with torch.no_grad():
        ddp.bias.fill_(BIAS)
    a = ddp(img, txt)
    b = SigLipLoss(focal_gamma=0.5)(img, txt, torch.tensor(TP, device=_dev()), torch.tensor(BIAS, device=_dev()))
    assert float(a) == pytest.approx(float(b), rel=1e-5)
    _check("module", "siglip vs oracle", b, p.focal_oracle(0.5, None, sets=False)["loss"])
    # focal_gamma=None: the module without the option, bit for bit
    c = SigLipLoss(focal_gamma=None)(img, txt, torch.tensor(TP, device=_dev()), torch.tensor(BIAS, device=_dev()))
    d = SigLipLoss()(img, txt, torch.tensor(TP, device=_dev()), torch.tensor(BIAS, device=_dev()))
    assert torch.equal(c, d)


def test_error_statuses():
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi

    B, D = 256, 136
    p = FocalProblem([B], D, 2, kind="tags", seed=13)
    img, txt = p.img.to(_dev()), p.texts[0].to(_dev())
    L = _capi.lib()
    eng = _fresh(_engine(B, D, labels=False))
    # the setter outside the mode, then the mode without a setter call: refused before any launch
    assert L.siglip_set_focal(eng._h, 2.0, 0.25) == _capi.SIGLIP_ERR_STATE
    eng.set_option(_capi.SIGLIP_OPT_FOCAL, 1)
    with pytest.raises(_capi.SiglipError) as e:
        eng.fwd_bwd(img, txt, _scal(TP), _scal(BIAS))
    assert e.value.code == _capi.SIGLIP_ERR_STATE
    for gamma, alpha in ((-0.1, 0.25), (8.5, -1.0), (float("nan"), -1.0), (float("inf"), -1.0), (2.0, 1.5),
                         (2.0, float("nan"))):
        assert L.siglip_set_focal(eng._h, gamma, alpha) == _capi.SIGLIP_ERR_INVALID, (gamma, alpha)
    with pytest.raises(_capi.SiglipError):
        eng.fwd_bwd(img, txt, _scal(TP), _scal(BIAS))   # refused values are not recorded
    assert L.siglip_set_focal(eng._h, 2.0, -1.0) == 0
    a = eng.fwd_bwd(img, txt, _scal(TP), _scal(BIAS))
    b = eng.fwd_bwd(img, txt, _scal(TP), _scal(BIAS))   # the values persist across steps
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    _check("refusals", "persisted values", a[0], p.focal_oracle(2.0, None, sets=False)["loss"])
    with pytest.raises(_capi.SiglipError) as e:
        eng.fwd_bwd_host(p.img, p.texts[0], TP, BIAS)
    assert e.value.code == _capi.SIGLIP_ERR_STATE
    # with distillation, in both orders
    dist = SigmoidLossEngine(B, D, _dev(), teacher_dim=64)
    dist.set_option(_capi.SIGLIP_OPT_DISTILL, 1)
    assert L.siglip_ctx_set_option(dist._h, _capi.SIGLIP_OPT_FOCAL, 1) == _capi.SIGLIP_ERR_STATE
    dist.set_option(_capi.SIGLIP_OPT_DISTILL, 0)
    dist.set_option(_capi.SIGLIP_OPT_FOCAL, 1)
    assert L.siglip_ctx_set_option(dist._h, _capi.SIGLIP_OPT_DISTILL, 1) == _capi.SIGLIP_ERR_STATE
    # turning the option off gives the plain step back
    eng.set_option(_capi.SIGLIP_OPT_FOCAL, 0)
    plain = _fresh(_engine(B, D, labels=False))
    c = eng.fwd_bwd(img, txt, _scal(TP), _scal(BIAS))
    d = plain.fwd_bwd(img, txt, _scal(TP), _scal(BIAS))
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(c, d))
