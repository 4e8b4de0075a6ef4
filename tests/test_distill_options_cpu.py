"""CPU checks of distillation with the other options: the composed float64 oracle against float64 autograd of a direct
restatement (extras, ids, label sets, excluded groups, weights; W = 1, 2, 3), its lambda -> 0 reductions to the
non-distillation oracles, the sign of every term and the per-sample sums, and the modules' argument handling (raised
before any GPU work)."""
import math

import numpy as np
import pytest
import torch

from distill_oracle import closed_form_distill
from distill_options_oracle import closed_form_distill_options
from exclude_groups_oracle import closed_form_groups, dtxt_of, group_labels, text_loss_of, torch_loss, torch_terms
from extra_images_oracle import label_blocks
from label_sets_oracle import set_labels

TP, BIAS, TTP, TBIAS = math.log(10.0), -6.0, math.log(14.0), -4.0


def _unit(g, n, D):
    x = g.standard_normal((n, D))
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def _close(a, b, tol=1e-10):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    assert np.abs(a - b).max() <= tol * max(1.0, np.abs(b).max()), np.abs(a - b).max()


def _problem(Bs, K_txt, K_img, D, DT, seed, labels="ids", groups=True, weights=True):
    """Rank r: B_r paired samples, K_img extra images, K_txt extra texts; labels from ids (every extra carries one),
    positions, or label sets (M = 2); optional groups (a few classes, so that exclusions happen) and weights."""
    g = np.random.default_rng(seed)
    Rs, Ts = [b + K_img for b in Bs], [b + K_txt for b in Bs]
    P = dict(Bs=Bs, Rs=Rs, Ts=Ts)
    P["imgs"] = [_unit(g, r, D) for r in Rs]
    P["txts"] = [_unit(g, t, D) for t in Ts]
    P["timgs"] = [_unit(g, r, DT) for r in Rs]
    P["ttxts"] = [_unit(g, t, DT) for t in Ts]
    if labels == "ids":
        ids = [g.integers(0, 4, b) for b in Bs]
        y = label_blocks(Bs, Rs, Ts, ids, [g.integers(0, 4, K_txt) for _ in Bs],
                         [g.integers(0, 4, K_img) for _ in Bs])
    elif labels == "sets":
        isets = [np.concatenate([g.integers(-1, 5, (b, 2)), g.integers(-1, 5, (K_img, 2))]) for b in Bs]
        tsets = [np.concatenate([isets[r][:b], g.integers(-1, 5, (K_txt, 2))]) for r, b in enumerate(Bs)]
        y = set_labels(isets, tsets, Bs)
    else:
        y = label_blocks(Bs, Rs, Ts)
    if groups:
        y = group_labels(y, [g.integers(-1, 3, r) for r in Rs], [g.integers(-1, 3, t) for t in Ts])
    P["labels"] = y
    P["iws"] = [g.random(r) for r in Rs] if weights else None
    P["tws"] = [g.random(t) for t in Ts] if weights else None
    return P


def _oracle(P, lam):
    return closed_form_distill_options(P["imgs"], P["txts"], TP, BIAS, P["timgs"], P["ttxts"], TTP, TBIAS, lam,
                                       P["labels"], P["Bs"], P["iws"], P["tws"])


CASES = [([7], 3, 2, "ids"), ([5, 9], 0, 3, "ids"), ([6, 4, 5], 2, 0, "sets"), ([6, 6], 0, 0, "positions"),
         ([4, 7, 3], 2, 2, "sets")]


@pytest.mark.parametrize("Bs,K_txt,K_img,labels", CASES)
def test_oracle_matches_autograd_of_the_restatement(Bs, K_txt, K_img, labels):
    P = _problem(Bs, K_txt, K_img, 12, 5, seed=len(Bs) + K_txt, labels=labels)
    lam = 0.35
    ref = _oracle(P, lam)
    assert any((np.concatenate(row, axis=1) == 0).any() for row in P["labels"])   # some pairs are excluded
    T = [torch.tensor(x, requires_grad=True) for x in P["txts"]]
    Tt = torch.cat([torch.tensor(x) for x in P["ttxts"]])
    tw = torch.cat([torch.tensor(x) for x in P["tws"]])
    for r, img in enumerate(P["imgs"]):
        I = torch.tensor(img, requires_grad=True)
        tpv = torch.tensor(TP, dtype=torch.float64, requires_grad=True)
        bv = torch.tensor(BIAS, dtype=torch.float64, requires_grad=True)
        y = torch.tensor(np.concatenate(P["labels"][r], axis=1))
        teacher = (torch.tensor(P["timgs"][r]), Tt, TTP, TBIAS, lam)
        for x in T:
            x.grad = None
        loss = torch_loss(I, torch.cat(T), tpv, bv, y, torch.tensor(P["iws"][r]), tw, batch=P["Bs"][r],
                          teacher=teacher)
        loss.backward()
        _close(ref[r]["loss"], float(loss.detach()))
        _close(ref[r]["dimg"], I.grad.numpy())
        _close(ref[r]["dt_prime"], float(tpv.grad))
        _close(ref[r]["dbias"], float(bv.grad))
        for c, x in enumerate(T):
            _close(ref[r]["contrib"][c], x.grad.numpy())
        terms = torch_terms(I.detach(), torch.cat(T).detach(), tpv.detach(), BIAS, y, torch.tensor(P["iws"][r]), tw,
                            teacher=teacher).numpy()
        _close(ref[r]["image_loss"], terms.sum(axis=1))
        _close(np.concatenate(ref[r]["text_part"]), terms.sum(axis=0))


@pytest.mark.parametrize("Bs,K_txt,K_img,labels", CASES)
def test_lambda_zero_is_the_hard_label_oracle(Bs, K_txt, K_img, labels):
    P = _problem(Bs, K_txt, K_img, 10, 7, seed=3, labels=labels)
    got = _oracle(P, 0.0)
    ref = closed_form_groups(P["imgs"], P["txts"], TP, BIAS, P["labels"], P["Bs"], P["iws"], P["tws"])
    for x, y in zip(got, ref):
        for k in ("loss", "dimg", "dt_prime", "dbias", "image_loss"):
            _close(x[k], y[k])
        for key in ("contrib", "text_part"):
            for a, b in zip(x[key], y[key]):
                _close(a, b)
    for c in range(len(Bs)):
        _close(dtxt_of(got, c), dtxt_of(ref, c))
        _close(text_loss_of(got, c), text_loss_of(ref, c))


def test_without_the_new_options_it_is_the_distillation_oracle():
    Bs = [6, 9, 5]
    P = _problem(Bs, 0, 0, 10, 7, seed=5, labels="ids", groups=False)
    got = _oracle(P, 0.6)
    ref = closed_form_distill(P["imgs"], P["txts"], TP, BIAS, P["timgs"], P["ttxts"], TTP, TBIAS, 0.6, P["iws"],
                              P["tws"], P["labels"])
    for x, y in zip(got, ref):
        for k in ("loss", "dimg", "dt_prime", "dbias"):
            _close(x[k], y[k])
        for a, b in zip(x["contrib"], y["contrib"]):
            _close(a, b)


@pytest.mark.parametrize("Bs,K_txt,K_img,labels", CASES)
@pytest.mark.parametrize("lam", [0.2, 1.0])
def test_terms_are_nonnegative_and_the_loss_divides_by_the_paired_batch(Bs, K_txt, K_img, labels, lam):
    P = _problem(Bs, K_txt, K_img, 10, 7, seed=11, labels=labels)
    for r, res in enumerate(_oracle(P, lam)):
        assert (res["image_loss"] >= 0).all() and all((x >= 0).all() for x in res["text_part"])
        _close(res["loss"], res["image_loss"].sum() / Bs[r])
        _close(res["loss"], sum(x.sum() for x in res["text_part"]) / Bs[r])


def test_teacher_equal_to_student_at_lambda_one_has_zero_gradient_on_the_extras_too():
    P = _problem([8, 5], 3, 2, 6, 6, seed=4, labels="sets")
    P["timgs"], P["ttxts"] = P["imgs"], P["txts"]
    res = closed_form_distill_options(P["imgs"], P["txts"], TP, BIAS, P["imgs"], P["txts"], TP, BIAS, 1.0,
                                      P["labels"], P["Bs"], P["iws"], P["tws"])
    for x in res:
        for k in ("dimg", "dt_prime", "dbias"):
            _close(x[k], np.zeros_like(np.asarray(x[k])), 1e-14)
        for a in x["contrib"]:
            _close(a, np.zeros_like(a), 1e-14)


# ---- the modules ----

def _mods():
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss, SigLipLoss

    return DDPSigmoidLoss, SigLipLoss


def test_distill_options_composes_with_every_option_but_focal():
    DDP, SL = _mods()
    for cls in (DDP, SL):
        args = (8,) if cls is DDP else ()
        for opt in (dict(multi_label=1), dict(exclude_groups=True), dict(hard_negatives=2),
                    dict(multi_positive=True, extra_texts=2), dict(extra_images=2)):
            # the refusals of distill without the flag are unchanged (they name the flag), and the flag lifts them
            with pytest.raises(RuntimeError, match="cannot be combined.*distill_options=True"):
                cls(*args, distill=0.5, **opt)
            cls(*args, distill=0.5, distill_options=True, **opt)
        cls(*args, distill=0.5, distill_options=True, hard_negatives=3, exclude_groups=True, sample_weights=True)
        cls(*args, distill=0.5, distill_options=True, multi_positive=True, extra_texts=2, extra_images=2)
        cls(*args, distill=0.5, distill_options=True, multi_label=2, extra_texts=3, extra_images=2, exclude_groups=True)
        with pytest.raises(RuntimeError, match="focal_gamma cannot be combined with distill"):
            cls(*args, distill=0.5, distill_options=True, focal_gamma=2.0)
        for bad in (1, "yes", None):
            with pytest.raises(RuntimeError, match="distill_options must be a bool"):
                cls(*args, distill=0.5, distill_options=bad)
        with pytest.raises(RuntimeError, match="distill_options=True needs distill=lambda"):
            cls(*args, distill_options=True)


def _call(mod, img, txt, **kw):
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss

    one = torch.tensor(1.0)
    scalars = ("teacher_t_prime", "teacher_bias") if isinstance(mod, DDPSigmoidLoss) else \
        ("teacher_logit_scale", "teacher_logit_bias")
    if "teacher_image" in kw:
        kw.update({n: one for n in scalars})
    if isinstance(mod, DDPSigmoidLoss):
        return mod(img, txt, **kw)
    return mod(img, txt, torch.tensor(2.3), torch.tensor(-10.0), **kw)


@pytest.mark.parametrize("which", ["ddp", "siglip"])
def test_teacher_extras_are_checked_before_any_gpu_work(which):
    DDP, SL = _mods()
    B, D, DT, K = 8, 16, 12, 3
    img, txt, neg = torch.randn(B, D), torch.randn(B, D), torch.randn(K, D)
    timg, ttxt, tneg = torch.randn(B, DT), torch.randn(B, DT), torch.randn(K, DT)
    opt = dict(distill=0.5, distill_options=True)
    mod = DDP(B, hard_negatives=K, **opt) if which == "ddp" else SL(hard_negatives=K, **opt)
    base = dict(negative_text=neg, teacher_image=timg, teacher_text=ttxt)
    with pytest.raises(RuntimeError, match=r"forward needs teacher_negative_text \(\[3, teacher_dim\]"):
        _call(mod, img, txt, **base)
    with pytest.raises(RuntimeError, match="teacher_extra_text given, but the loss has no such extras"):
        _call(mod, img, txt, **base, teacher_negative_text=tneg, teacher_extra_text=tneg)
    with pytest.raises(RuntimeError, match=r"teacher_negative_text must have shape \[3, 12\]"):
        _call(mod, img, txt, **base, teacher_negative_text=tneg[:, :5])
    with pytest.raises(RuntimeError, match="teacher_negative_text requires grad"):
        _call(mod, img, txt, **base, teacher_negative_text=tneg.clone().requires_grad_(True))
    with pytest.raises(RuntimeError, match="teacher_negative_text is torch.float64"):
        _call(mod, img, txt, **base, teacher_negative_text=tneg.double())
    with pytest.raises(RuntimeError, match="teacher_negative_text must be a floating-point tensor"):
        _call(mod, img, txt, **base, teacher_negative_text=tneg.long())
    # with valid arguments the call reaches the usual checks: CPU tensors are refused as before
    with pytest.raises(RuntimeError, match="CUDA|cuda|device"):
        _call(mod, img, txt, **base, teacher_negative_text=tneg)
    plain = DDP(B, hard_negatives=K) if which == "ddp" else SL(hard_negatives=K)
    with pytest.raises(RuntimeError, match="teacher_negative_text given, but the loss was built without distill"):
        _call(plain, img, txt, negative_text=neg, teacher_negative_text=tneg)
    xi = DDP(B, extra_images=2, **opt) if which == "ddp" else SL(extra_images=2, **opt)
    with pytest.raises(RuntimeError, match=r"forward needs teacher_extra_image"):
        _call(xi, img, txt, extra_image=torch.randn(2, D), teacher_image=timg, teacher_text=ttxt)


def test_c_abi_declares_the_new_entry():
    import os

    from distributed_sigmoid_loss_b200 import _capi

    hdr = open(os.path.join(os.path.dirname(__file__), "..", "include", "siglip_b200.h")).read()
    assert "int siglip_ctx_create_distill_extras(" in hdr
    assert "siglip_ctx_create_distill_extras" in _capi.EXPORTED_SYMBOLS


@pytest.mark.parametrize("metrics", [False, True])
def test_sample_losses_and_topk_under_distill_options_reach_the_tensor_checks(metrics):
    """Under distill without the flag the statistics are refused before any GPU work, as they always were; with it the
    call goes on to the usual checks, where CPU tensors are refused."""
    img, txt, one = torch.zeros(8, 16), torch.zeros(8, 16), torch.tensor(1.0)
    DDP, SL = _mods()
    t = dict(teacher_image=img, teacher_text=txt)
    for kw in (dict(return_sample_losses=True), dict(return_metrics=True, metrics_topk=5)):
        kw = dict(kw, return_metrics=metrics or "metrics_topk" in kw)
        with pytest.raises(RuntimeError, match="unavailable with distill.*distill_options=True"):
            DDP(8, distill=0.5)(img, txt, teacher_t_prime=one, teacher_bias=one, **t, **kw)
        with pytest.raises(RuntimeError, match="CUDA|cuda|device"):
            DDP(8, distill=0.5, distill_options=True)(img, txt, teacher_t_prime=one, teacher_bias=one, **t, **kw)
        with pytest.raises(RuntimeError, match="CUDA|cuda|device"):
            SL(distill=0.5, distill_options=True)(img, txt, one, one, teacher_logit_scale=one, teacher_logit_bias=one,
                                                  **t, **kw)
