"""The loss and gradient kernels at the logits of a trained model (tests/trained_regime.py), against the float64 oracle.

At t = 10, b = -10 (the rest of the suite) the negatives are under 1 % of the own chunk's gradient norm, so a 1e-3
check of the whole tensor cannot see them. Here t is 100 or 300, the negatives carry most of the gradient, the series
and general paths share every tile, and sigma * 2^14 spans fp16 from 16384 down to its subnormals. Besides the whole
tensors, every gradient check also compares the part that passes through the 16-bit sigma operand G — the kernel's
output minus the oracle's own-diagonal term, which the kernel adds in fp32 — with the oracle's remaining part, so the
sigma-operand path is measured on its own, and the cold regime (t = 10) runs that check once per label mode.
dbias and dt' are checked against tol * sum |G| and tol * t sum |G s|: at the stationary bias their values cancel.

Observed errors on one H100 80GB HBM3 (largest over the cases of each group; tensors: max of relative Frobenius and
max-abs / max over dimg, every contribution and their parts through G; scalars: dbias, dt' relative to their scale).
`pytest -s` prints them at the end of the module. The file runs in about 60 s there.
  group                                tensors   loss      scalars   tolerance
  cold (t 10, b -10), part through G   2.2e-4    1.0e-7    9.3e-8    TOL 1e-3
  trained (t 100, b -13)               1.4e-4    3.1e-6    2.7e-6    TOL
  stationary (t 100, sum G = 0)        2.8e-4    1.0e-6    3.1e-6    TOL
  t300 (t 300, b -30)                  1.1e-4    6.5e-6    5.5e-6    TOL
  separated (t 100, b -10)             2.5e-4    9.5e-7    7.1e-7    TOL
  trained, B 16384, D 1024             4.6e-5    3.7e-6    2.5e-6    TOL
  module, fp32 inputs, t 100 / 300     2.9e-4 / 4.6e-4   2.3e-5   1.7e-5   TOL
  module, normalize_inputs, t 100 / 300  2.6e-4 / 5.5e-4  2.3e-5   1.7e-5   TOL
  bf16 gradient outputs                3.1e-3    -         -         BF16_TOL 4.9e-3
The fp16(16 x) operands of fp32 inputs cost more as t grows (2e-4 at t = 10), but stay within 1e-3 at t = 300.
"""
import math

import numpy as np
import pytest
import torch

from sample_weights_oracle import closed_form_weighted, label_blocks
from trained_regime import (REGIMES, cold_batch, make_batch, random_weights, scalar_scales, split_own_diagonal,
                            stationary_bias)

pytestmark = pytest.mark.gpu

TOL = 1e-3
# bf16 gradient outputs: the oracle tolerance plus their own rounding, up to half an ulp of the largest binade = 2^-8 of
# the largest element in the max-abs / max measure
BF16_TOL = TOL + 2.0 ** -8
MODES = ["pos", "ids", "hn", "extra"]
_OBSERVED = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(_OBSERVED):
        print(f"trained-regime max error {k}: {_OBSERVED[k]:.3e}")


def _dev():
    return torch.device("cuda", 0)


def _scal(x):
    return torch.tensor([x], device=_dev(), dtype=torch.float32)


def _f32(x):
    return float(np.float32(x))


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return max(float((a - b).norm() / (b.norm() + 1e-300)), float((a - b).abs().max() / (b.abs().max() + 1e-300)))


def _note(group, what, err):
    key = f"{group} {what}"
    _OBSERVED[key] = max(_OBSERVED.get(key, 0.0), err)


def _check(group, name, got, ref, tol):
    err = _rel(got, ref)
    _note(group, name.split()[-1], err)
    assert err <= tol, f"{group} {name}: relative error {err:.3e} (tolerance {tol:.1e})"


def _check_scalar(group, name, got, ref, scale, tol):
    err = abs(float(got) - float(ref)) / scale
    _note(group, name.split()[-1], err)
    assert err <= tol, f"{group} {name}: {float(got)} vs {float(ref)}, error {err:.3e} of the scale {scale:.3e}"


def _engine(B, D, cg=2, mcast=1, ids=False, extra_ids=False, weighted=False, **kw):
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi

    eng = SigmoidLossEngine(B, D, _dev(), cta_group=cg, **kw)
    if mcast != 1:
        eng.set_option(_capi.SIGLIP_OPT_MCAST, mcast)
    if ids:
        eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 1)
    if extra_ids:
        eng.set_option(_capi.SIGLIP_OPT_EXTRA_TEXT_IDS, 1)
    if weighted:
        eng.set_option(_capi.SIGLIP_OPT_SAMPLE_WEIGHTS, 1)
    eng.weighted = weighted
    return eng


def _dv(x):
    return None if x is None else x.to(_dev())


def _step(eng, sched, img, txt, tp, b, ids=None, eids=None, iw=None, tw=None, grad_dtype=torch.float32):
    """One step: [loss] (fwd) or [loss, dimg, dtxt, dt', dbias] plus, at W > 1, this rank's contribution slots."""
    if ids is not None:
        eng.set_sample_ids(_dv(ids))
    if eids is not None and eng.extra_text_ids:
        eng.set_extra_text_ids(_dv(eids))
    if eng.weighted:
        eng.set_sample_weights(_dv(iw), _dv(tw))
    img, txt, tp, b = img.to(_dev()), txt.to(_dev()), _scal(tp), _scal(b)
    if sched == "fused":
        loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, tp, b, grad_dtype)
    elif sched == "split":
        loss = eng.forward(img, txt, tp, b, True)
        dimg, dtxt, dtp, db = eng.backward(img, txt, tp, None, grad_dtype)
    else:
        return [eng.fwd(img, txt, tp, b).clone()]
    outs = [loss, dimg, dtxt, dtp, db]
    if eng.world > 1:
        outs += [eng.debug_get_slot(k) for k in range(eng.world) if k != eng.rank]
    torch.cuda.synchronize()
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


class Problem:
    """Inputs, labels, bias and the float64 oracle (with its own-diagonal split and scalar scales) of one batch."""

    def __init__(self, Bs, Ks, D, seed, mode, regime=None, weighted=False):
        self.Bs, self.Ks, self.mode = list(Bs), list(Ks), mode
        self.Ts = [b + k for b, k in zip(Bs, Ks)]
        if regime is None:       # the cold regime of the rest of the suite
            self.imgs, self.texts, self.ids, self.eids = cold_batch(Bs, Ks, D, seed, mode)
            tp, bias = math.log(10.0), -10.0
        else:
            self.imgs, self.texts, self.ids, self.eids = make_batch(regime, Bs, Ks, D, seed, mode)
            tp, bias = regime.t_prime, regime.bias
        g = torch.Generator().manual_seed(seed + 1)
        self.iws = [random_weights(g, b) for b in Bs] if weighted else None
        self.tws = [random_weights(g, t) for t in self.Ts] if weighted else None
        f = (lambda xs: None if xs is None else [x.numpy() for x in xs])  # noqa: E731
        self.labels = label_blocks(self.Bs, self.Ts, f(self.ids), f(self.eids) if mode == "extra" else None)
        self.tp = _f32(tp)
        self.bias = _f32(stationary_bias(self.imgs, self.texts, self.tp, self.iws, self.tws, self.labels)
                         if bias is None else bias)
        args = (self.imgs, self.texts, self.tp, self.bias, self.iws, self.tws, self.labels)
        d = (lambda xs: None if xs is None else [x.double().numpy() for x in xs])  # noqa: E731
        self.ref = closed_form_weighted(d(self.imgs), d(self.texts), self.tp, self.bias, d(self.iws), d(self.tws),
                                        self.labels)
        self.parts = split_own_diagonal(*args)
        self.scales = scalar_scales(*args)

    def engine(self, r, cg=2, mcast=1, **kw):
        W = len(self.Bs)
        lb = dict(rank_world=(r, W), loopback=True) if W > 1 else {}
        eng = _engine(self.Bs[r], self.imgs[0].shape[1], cg, mcast, ids=self.mode != "pos",
                      extra_ids=self.mode == "extra", weighted=self.iws is not None, batch_per_rank=self.Bs,
                      texts_per_rank=self.Ts, **lb, **kw)
        if W > 1:
            _loopback(eng, r, self.texts, self.ids, self.eids, self.tws)
        return eng

    def step(self, eng, r, sched, grad_dtype=torch.float32):
        pick = (lambda xs: None if xs is None else xs[r])  # noqa: E731
        return _step(eng, sched, self.imgs[r], self.texts[r], self.tp, self.bias, pick(self.ids), pick(self.eids),
                     pick(self.iws), pick(self.tws), grad_dtype)

    def check(self, group, tag, out, r, tol=TOL):
        """loss; dimg, dt', dbias and every chunk contribution; and the parts of dimg and of the own contribution that
        pass through G (the output minus the oracle's own-diagonal term) against the oracle's remaining parts."""
        ref, part, sc = self.ref[r], self.parts[r], self.scales[r]
        _check(group, f"{tag} loss", out[0], ref["loss"], tol)
        if len(out) == 1:
            return
        W = len(self.Bs)
        _check(group, f"{tag} dimg", out[1], ref["dimg"], tol)
        _check_scalar(group, f"{tag} dbias", out[4], ref["dbias"], sc["dbias"], tol)
        _check_scalar(group, f"{tag} dt_prime", out[3], ref["dt_prime"], sc["dt_prime"], tol)
        slots = iter(out[5:])
        for k in range(W):
            got = out[2].float() if k == r else next(slots)
            _check(group, f"{tag} contribution to chunk {k}: contrib", got, ref["contrib"][k], tol)
            if k == r:
                own = got
        dimg = out[1].double().cpu() - torch.from_numpy(part["diag_dimg"])
        _check(group, f"{tag} dimg through G: rest_dimg", dimg, part["rest_dimg"], tol)
        contrib = own.double().cpu() - torch.from_numpy(part["diag_contrib"])
        _check(group, f"{tag} own contribution through G: rest_contrib", contrib, part["rest_contrib"], tol)


def _problem_shape(mode, B=1000, K=136, D=264):
    return (B,), (K if mode in ("hn", "extra") else 0,), D


# ---------------------------------------------------------------------------------------------------------------------
# 1. one rank at a ragged shape: every regime, label mode and weighting; cluster shapes, tile widths, split-K, bf16
# ---------------------------------------------------------------------------------------------------------------------
# (cta_group, mcast, SIGLIP_OPT_GRAD_TILE_N, SIGLIP_OPT_SPLIT_K)
CONFIGS = [(1, 1, 256, 0), (2, 1, 128, 0), (2, 2, 256, 0), (2, 1, 0, -1)]


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("regime", list(REGIMES))
def test_single_rank_trained_regime(regime, mode, weighted):
    from distributed_sigmoid_loss_b200 import _capi

    Bs, Ks, D = _problem_shape(mode)
    pb = Problem(Bs, Ks, D, 11 + MODES.index(mode), mode, REGIMES[regime], weighted)
    for cg, mcast, tn, sk in CONFIGS:
        eng = pb.engine(0, cg, mcast)
        eng.set_option(_capi.SIGLIP_OPT_GRAD_TILE_N, tn)
        eng.set_option(_capi.SIGLIP_OPT_SPLIT_K, sk)
        for sched in ("fused", "split", "fwd"):
            out = pb.step(eng, 0, sched)
            pb.check(regime, f"{sched} {mode} w={weighted} cg={cg} mcast={mcast} tn={tn} sk={sk}", out, 0)
        if (cg, mcast) == (2, 1) and tn == 128:
            out = pb.step(eng, 0, "fused", torch.bfloat16)
            pb.check(f"{regime} bf16-out", f"fused bf16 {mode} w={weighted}", out, 0, BF16_TOL)
        eng.close()


@pytest.mark.parametrize("mode", MODES)
def test_cold_regime_sigma_operand_part(mode):
    """t = 10, b = -10 and independent random embeddings, as the rest of the suite: the whole-tensor checks cannot see
    the negatives there, the check of the part through G can."""
    Bs, Ks, D = _problem_shape(mode)
    pb = Problem(Bs, Ks, D, 21 + MODES.index(mode), mode, None, weighted=mode in ("hn", "extra"))
    eng = pb.engine(0)
    for sched in ("fused", "split"):
        pb.check("cold", f"{sched} {mode}", pb.step(eng, 0, sched), 0)
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. loopback multi-chunk schedules: W = 3 with uneven batches, W = 4 bidirectional
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Bs,Ks,mode,bidir,weighted", [((160, 96, 130), (0, 0, 0), "pos", False, False),
                                                       ((160, 96, 130), (40, 0, 200), "extra", False, True),
                                                       ((128, 128, 128, 128), (0, 0, 0, 0), "ids", True, True),
                                                       ((128, 128, 128, 128), (16, 300, 5, 64), "hn", True, False)])
@pytest.mark.parametrize("regime", list(REGIMES))
def test_loopback_trained_regime(regime, Bs, Ks, mode, bidir, weighted):
    from distributed_sigmoid_loss_b200 import _capi

    pb = Problem(Bs, Ks, 264, sum(Bs) + sum(Ks), mode, REGIMES[regime], weighted)
    for r in range(len(Bs)):
        eng = pb.engine(r)
        if bidir:
            eng.set_option(_capi.SIGLIP_OPT_BIDIR, 1)
        for sched in ("fused", "split"):
            pb.check(regime, f"W={len(Bs)} r={r} {sched} {mode} w={weighted}", pb.step(eng, r, sched), r)
        eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. a large single-rank shape (float64 oracle on the CPU) and the benchmark's shape (float64 on the GPU)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("regime", ["trained", "t300"])
def test_large_batch_trained_regime(regime):
    from distributed_sigmoid_loss_b200 import _capi

    pb = Problem((4096,), (0,), 768, 4096, "pos", REGIMES[regime])
    eng = pb.engine(0)
    for tn, sk in ((128, 0), (256, 0), (0, -1)):
        eng.set_option(_capi.SIGLIP_OPT_GRAD_TILE_N, tn)
        eng.set_option(_capi.SIGLIP_OPT_SPLIT_K, sk)
        for sched in ("fused", "split"):
            pb.check(regime, f"B=4096 {sched} tn={tn} sk={sk}", pb.step(eng, 0, sched), 0)
    pb.check(f"{regime} bf16-out", "B=4096 fused bf16", pb.step(eng, 0, "fused", torch.bfloat16), 0, BF16_TOL)
    eng.close()


def test_headline_shape_against_float64_on_the_gpu():
    """B = 16384, D = 1024 at t = 100, b = -13: the oracle in float64 on the device (too large for the CPU here)."""
    R = REGIMES["trained"]
    B, D = 16384, 1024
    (img,), (txt,), _, _ = make_batch(R, (B,), (0,), D, 16384, "pos")
    tp, bias = _f32(R.t_prime), R.bias
    t = math.exp(tp)
    x, y = img.to(_dev()).double(), txt.to(_dev()).double()
    s = x @ y.T
    z = t * s + bias
    diag = torch.arange(B, device=_dev())
    zp = z[diag, diag].clone()
    # the regime: slabs of both paths (16-row bands x 32 columns, the own-diagonal band left out), negatives above 0
    smax = z.view(B // 16, 16, B // 32, 32).amax(dim=(1, 3))
    band = torch.arange(B // 16, device=_dev())[:, None] // 2 == torch.arange(B // 32, device=_dev())[None, :]
    fast = float((smax[~band] < -4.2).double().mean())
    z[diag, diag] = -math.inf
    assert 0.2 <= fast <= 0.8 and float((z > 0).double().mean()) > 1e-4, (fast, float((z > 0).double().mean()))
    neg = torch.sigmoid(z)
    G = neg / B
    G[diag, diag] = -torch.sigmoid(-zp) / B
    loss = float((torch.nn.functional.softplus(z).sum() + torch.nn.functional.softplus(-zp).sum()) / B)
    ref = dict(loss=loss, dimg=(t * (G @ y)).cpu(), dtxt=(t * (G.T @ x)).cpu(), dbias=float(G.sum()),
               dt_prime=float(t * (G * s).sum()))
    sc = dict(dbias=float(G.abs().sum()), dt_prime=float(t * (G * s).abs().sum()))
    gd = G[diag, diag].clone()
    G[diag, diag] = 0.0
    rest_dimg, rest_dtxt = (t * (G @ y)).cpu(), (t * (G.T @ x)).cpu()
    diag_dimg, diag_dtxt = (t * gd[:, None] * y).cpu(), (t * gd[:, None] * x).cpu()
    del s, z, neg, G, x, y
    torch.cuda.empty_cache()
    eng = _engine(B, D)
    out = _step(eng, "fused", img, txt, tp, bias)
    eng.close()
    group = "trained headline"
    _check(group, "loss", out[0], ref["loss"], TOL)
    _check(group, "dimg", out[1], ref["dimg"], TOL)
    _check(group, "dtxt: contrib", out[2], ref["dtxt"], TOL)
    _check_scalar(group, "dbias", out[4], ref["dbias"], sc["dbias"], TOL)
    _check_scalar(group, "dt_prime", out[3], ref["dt_prime"], sc["dt_prime"], TOL)
    _check(group, "dimg through G: rest_dimg", out[1].double().cpu() - diag_dimg, rest_dimg, TOL)
    _check(group, "dtxt through G: rest_contrib", out[2].double().cpu() - diag_dtxt, rest_dtxt, TOL)


# ---------------------------------------------------------------------------------------------------------------------
# 4. the module with fp32 inputs (fp16(16 x) operands) and with normalize_inputs=True
# ---------------------------------------------------------------------------------------------------------------------
def _normalize_bwd(x, dxhat):
    """Float64 backward of x -> x / |x| (rows)."""
    n = np.linalg.norm(x, axis=1, keepdims=True)
    xh = x / n
    return (dxhat - xh * (xh * dxhat).sum(1, keepdims=True)) / n


@pytest.mark.parametrize("inputs", ["fp32", "normalize"])
@pytest.mark.parametrize("regime", ["trained", "t300"])
def test_module_fp32_inputs_trained_regime(regime, inputs):
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss

    R = REGIMES[regime]
    B, D = 1000, 264
    (img,), (txt,), _, _ = make_batch(R, (B,), (0,), D, 31, "pos", dtype=torch.float32)
    xi, xt = img.double().numpy(), txt.double().numpy()
    if inputs == "normalize":   # rows of random norms: the module normalises them
        g = torch.Generator().manual_seed(32)
        img = img * (0.5 + 2 * torch.rand(B, 1, generator=g))
        txt = txt * (0.5 + 2 * torch.rand(B, 1, generator=g))
        xi = xi / np.linalg.norm(xi, axis=1, keepdims=True)
        xt = xt / np.linalg.norm(xt, axis=1, keepdims=True)
    ref = closed_form_weighted([xi], [xt], R.t_prime, R.bias)[0]
    part = split_own_diagonal([torch.from_numpy(xi)], [torch.from_numpy(xt)], R.t_prime, R.bias)[0]
    sc = scalar_scales([torch.from_numpy(xi)], [torch.from_numpy(xt)], R.t_prime, R.bias)[0]
    xi_raw, xt_raw = img.double().numpy(), txt.double().numpy()
    chain = ((lambda x, d: _normalize_bwd(x, d)) if inputs == "normalize" else (lambda x, d: d))  # noqa: E731
    group = f"{regime} module-{inputs}"
    for fused in (False, True):
        mod = DDPSigmoidLoss(B, normalize_inputs=inputs == "normalize", fused_step=fused).to(_dev())
        with torch.no_grad():
            mod.t_prime.fill_(R.t_prime)
            mod.bias.fill_(R.bias)
        a, b = img.to(_dev()).requires_grad_(True), txt.to(_dev()).requires_grad_(True)
        loss = mod(a, b)
        loss.backward()
        torch.cuda.synchronize()
        tag = f"fused={fused}"
        _check(group, f"{tag} loss", loss.detach(), ref["loss"], TOL)
        _check(group, f"{tag} dimg", a.grad, chain(xi_raw, ref["dimg"]), TOL)
        _check(group, f"{tag} dtxt: contrib", b.grad, chain(xt_raw, ref["contrib"][0]), TOL)
        _check_scalar(group, f"{tag} dbias", mod.bias.grad, ref["dbias"], sc["dbias"], TOL)
        _check_scalar(group, f"{tag} dt_prime", mod.t_prime.grad, ref["dt_prime"], sc["dt_prime"], TOL)
        _check(group, f"{tag} dimg through G: rest_dimg", a.grad.double().cpu().numpy() -
               chain(xi_raw, part["diag_dimg"]), chain(xi_raw, part["rest_dimg"]), TOL)
        _check(group, f"{tag} dtxt through G: rest_contrib", b.grad.double().cpu().numpy() -
               chain(xt_raw, part["diag_contrib"]), chain(xt_raw, part["rest_contrib"]), TOL)

