"""Distillation with the other options on the H100 (kModeDistillOpts): hard negatives, extra texts with ids, extra
images with and without ids, per-sample losses, top-K, excluded groups, label sets and a cell with several at once,
through DDPSigmoidLoss against float64 autograd of the direct restatement (both schedules, a row-panel budget, fp32
inputs with normalize_inputs, a no-grad forward); the engine at loopback W = 2 / 3 (uneven, bidir) against the composed
oracle; and the exact properties: arming per-sample losses or top-K, or unique groups, changes no bit of the plain
distillation step; M = 1 label sets are the ids' step bit for bit; a teacher equal to the student at lambda = 1 leaves
no gradient, extras included."""
import math

import numpy as np
import pytest
import torch

from distill_options_oracle import closed_form_distill_options
from exclude_groups_oracle import group_labels, operand_values, torch_terms

pytestmark = pytest.mark.gpu

TOL = 1e-3
TTP, TBIAS = math.log(20.0), -8.0


def _dev():
    return torch.device("cuda", 0)


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return max(float((a - b).norm() / (b.norm() + 1e-300)), float((a - b).abs().max() / (b.abs().max() + 1e-300)))


def _check(name, got, ref, tol=TOL):
    err = _rel(got, ref)
    assert err <= tol, f"{name}: relative error {err:.3e}"


def _unit(g, n, D):
    return torch.nn.functional.normalize(torch.randn(n, D, generator=g))


K_NEG, K_TXT, K_IMG = 96, 40, 24

# (name, module kwargs): each newly allowed combination, then one with several at once
CELLS = [
    ("hard_negatives", dict(hard_negatives=K_NEG)),
    ("extra_texts_ids", dict(multi_positive=True, extra_texts=K_TXT)),
    ("extra_images", dict(extra_images=K_IMG)),
    ("extra_images_ids", dict(multi_positive=True, extra_images=K_IMG)),
    ("sample_losses", dict()),
    ("topk", dict()),
    ("groups", dict(exclude_groups=True)),
    ("label_sets", dict(multi_label=2)),
    ("several", dict(multi_label=2, extra_texts=K_TXT, extra_images=K_IMG, exclude_groups=True, sample_weights=True)),
]


def _inputs(B, D, DT, kw, seed, dtype=torch.bfloat16):
    """Student and teacher embeddings (the teacher a noisy copy of the student, so its probabilities are informative)
    and every per-sample argument a module built with kw takes."""
    g = torch.Generator().manual_seed(seed)
    R = B + kw.get("extra_images", 0)
    T = B + kw.get("hard_negatives", 0) + kw.get("extra_texts", 0)
    img, txt = _unit(g, R, D), _unit(g, T, D)
    txt[:B] = torch.nn.functional.normalize(txt[:B] + 2.0 * img[:B])   # positives score above the negatives
    proj = torch.randn(D, DT, generator=g) / math.sqrt(D)
    timg = torch.nn.functional.normalize(img @ proj + 0.3 * torch.randn(R, DT, generator=g))
    ttxt = torch.nn.functional.normalize(txt @ proj + 0.3 * torch.randn(T, DT, generator=g))
    a = dict(img=img.to(dtype), txt=txt.to(dtype), timg=timg.to(dtype), ttxt=ttxt.to(dtype), kw={}, B=B, R=R, T=T)
    ids = torch.randint(0, B // 3, (B,), generator=g)
    if kw.get("multi_positive"):
        a["kw"]["sample_ids"] = ids
        if kw.get("extra_texts"):
            a["kw"]["extra_text_ids"] = torch.randint(0, B // 3, (T - B,), generator=g)
        if kw.get("extra_images"):
            a["kw"]["extra_image_ids"] = torch.randint(0, B // 3, (R - B,), generator=g)
    if kw.get("multi_label"):
        M = kw["multi_label"]
        a["kw"]["sample_labels"] = torch.randint(-1, 12, (B, M), generator=g)
        if kw.get("extra_texts"):
            a["kw"]["extra_text_labels"] = torch.randint(-1, 12, (T - B, M), generator=g)
        if kw.get("extra_images"):
            a["kw"]["extra_image_labels"] = torch.randint(-1, 12, (R - B, M), generator=g)
    if kw.get("exclude_groups"):
        a["kw"]["image_groups"] = torch.randint(-1, 40, (R,), generator=g)
        a["kw"]["text_groups"] = torch.randint(-1, 40, (T,), generator=g)
    if kw.get("sample_weights"):
        a["kw"]["image_weights"] = torch.rand(R, generator=g)
        a["kw"]["text_weights"] = torch.rand(T, generator=g)
    return a


def _labels(a, kw):
    """[R, T] labels in {+1, -1, 0} of a W = 1 step, from the oracles' label rules."""
    from extra_images_oracle import label_blocks
    from label_sets_oracle import set_labels

    B, R, T, k = a["B"], a["R"], a["T"], a["kw"]
    if kw.get("multi_label"):
        isets = k["sample_labels"].numpy()
        if "extra_image_labels" in k:
            isets = np.concatenate([isets, k["extra_image_labels"].numpy()])
        tsets = k["sample_labels"].numpy()
        if "extra_text_labels" in k:
            tsets = np.concatenate([tsets, k["extra_text_labels"].numpy()])
        tsets = np.concatenate([tsets, -np.ones((T - tsets.shape[0], tsets.shape[1]), np.int64)])
        y = set_labels([isets], [tsets], [B])
    elif kw.get("multi_positive"):
        y = label_blocks([B], [R], [T], [k["sample_ids"].numpy()],
                         [k["extra_text_ids"].numpy()] if "extra_text_ids" in k else None,
                         [k["extra_image_ids"].numpy()] if "extra_image_ids" in k else None)
    else:
        y = label_blocks([B], [R], [T])
    if kw.get("exclude_groups"):
        y = group_labels(y, [k["image_groups"].numpy()], [k["text_groups"].numpy()])
    return torch.from_numpy(y[0][0])


def _module_call(kw, a, lam, fused, normalize=False, budget=None, losses=False, topk=None, grad=True, teacher=True,
                 tscalars=(TTP, TBIAS), options=True):
    """One forward (and backward) of DDPSigmoidLoss(distill=lam, distill_options=options, **kw) on the inputs a; returns
    the loss, the gradients of the paired and extra tensors, t_prime.grad / bias.grad and the per-sample losses /
    metrics when asked. options=False: a module without distill_options, which takes none of the new options."""
    from distributed_sigmoid_loss_b200 import DDPSigmoidLoss

    d = _dev()
    B = a["B"]
    mod = DDPSigmoidLoss(B, fused_step=fused, normalize_inputs=normalize, sigma_budget_bytes=budget,
                         distill=lam if teacher else None, distill_options=teacher and options, **kw).to(d)
    K_n, K_t = kw.get("hard_negatives", 0), kw.get("extra_texts", 0)
    leaf = dict(img=a["img"][:B], txt=a["txt"][:B], neg=a["txt"][B:B + K_n], xt=a["txt"][B + K_n:],
                xi=a["img"][B:])
    leaf = {n: x.to(d).requires_grad_(grad) for n, x in leaf.items()}
    args = {n: v.to(d) for n, v in a["kw"].items()}
    if K_n:
        args["negative_text"] = leaf["neg"]
    if K_t:
        args["extra_text"] = leaf["xt"]
    if kw.get("extra_images"):
        args["extra_image"] = leaf["xi"]
    if teacher:
        args.update(teacher_image=a["timg"][:B].to(d), teacher_text=a["ttxt"][:B].to(d),
                    teacher_t_prime=torch.tensor(tscalars[0], device=d),
                    teacher_bias=torch.tensor(tscalars[1], device=d))
        if K_n:
            args["teacher_negative_text"] = a["ttxt"][B:B + K_n].to(d)
        if K_t:
            args["teacher_extra_text"] = a["ttxt"][B + K_n:].to(d)
        if kw.get("extra_images"):
            args["teacher_extra_image"] = a["timg"][B:].to(d)
    if topk is not None:   # K = 1: the top-1 metrics alone, which a module without distill_options takes too
        args.update(return_metrics=True, **({} if topk == 1 else dict(metrics_topk=topk)))
    out = mod(leaf["img"], leaf["txt"], return_sample_losses=losses, **args)
    res = {}
    if isinstance(out, tuple):
        loss = out[0]
        for x in out[1:]:
            res.update(x)
    else:
        loss = out
    res["loss"] = loss.detach().clone()
    if grad:
        loss.backward()
        res["dimg"] = torch.cat([leaf["img"].grad] + ([leaf["xi"].grad] if kw.get("extra_images") else []))
        res["dtxt"] = torch.cat([leaf["txt"].grad] + ([leaf["neg"].grad] if K_n else []) +
                                ([leaf["xt"].grad] if K_t else []))
        res["dtp"], res["db"] = mod.t_prime.grad.clone(), mod.bias.grad.clone()
    torch.cuda.synchronize()
    return {k: (v.clone() if isinstance(v, torch.Tensor) else v) for k, v in res.items()}


def _reference(kw, a, lam, normalize=False):
    """float64 autograd of exclude_groups_oracle.torch_loss with the teacher, on the values the kernels consume."""
    img = operand_values(a["img"]).requires_grad_(True)
    txt = operand_values(a["txt"]).requires_grad_(True)
    tp = torch.tensor(math.log(10.0), dtype=torch.float64, requires_grad=True)
    b = torch.tensor(-10.0, dtype=torch.float64, requires_grad=True)
    y = _labels(a, kw).double()
    k = a["kw"]
    iw = k["image_weights"].double() if "image_weights" in k else None
    tw = k["text_weights"].double() if "text_weights" in k else None
    teacher = (operand_values(a["timg"]), operand_values(a["ttxt"]), TTP, TBIAS, lam)
    terms = torch_terms(img, txt, tp, b, y, iw, tw, normalize, teacher)
    loss = terms.sum() / a["B"]
    loss.backward()
    return dict(loss=loss.detach(), dimg=img.grad, dtxt=txt.grad, dtp=tp.grad, db=b.grad,
                image_loss=terms.detach().sum(1), text_loss=terms.detach().sum(0))


def _check_against(tag, got, ref, losses=False):
    for k in ("loss", "dimg", "dtxt", "dtp", "db"):
        _check(f"{tag} {k}", got[k], ref[k])
    if losses:
        _check(f"{tag} image_loss", got["image_loss"], ref["image_loss"])
        _check(f"{tag} text_loss", got["text_loss"], ref["text_loss"])


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("name,kw", CELLS, ids=[c[0] for c in CELLS])
def test_module_matches_the_oracle(name, kw, fused):
    # fp32 inputs: fp16(16 x) operands and fp32 gradients (bf16 inputs would get bf16 gradients, rounded by 2^-9)
    B, D, DT = 300, 136, 72
    a = _inputs(B, D, DT, kw, seed=len(name), dtype=torch.float32)
    losses = name in ("sample_losses", "several")
    topk = 5 if name in ("topk", "several") else None
    got = _module_call(kw, a, 0.5, fused, losses=losses, topk=topk)
    _check_against(f"{name} fused={fused}", got, _reference(kw, a, 0.5), losses)
    if topk is not None:
        # the lists rank the student's logits: those of the same step without a teacher, bit for bit
        plain = _module_call(kw, a, 0.5, fused, topk=topk, teacher=False)
        for k in ("i2t_topk", "t2i_topk", "i2t_recall", "t2i_recall", "i2t_top1", "t2i_top1"):
            assert torch.equal(got[k], plain[k]), k


@pytest.mark.parametrize("name,kw", [CELLS[0], CELLS[-1]], ids=["hard_negatives", "several"])
def test_fp32_inputs_with_normalize_inputs_and_a_row_panel_budget(name, kw):
    B, D, DT = 600, 136, 72
    a = _inputs(B, D, DT, kw, seed=5, dtype=torch.float32)
    a["img"], a["txt"] = a["img"] * 3.0, a["txt"] * 0.5   # not unit: normalize_inputs does that
    a["timg"], a["ttxt"] = a["timg"] * 2.0, a["ttxt"] * 0.7
    for budget in (None, 1 << 20):
        got = _module_call(kw, a, 0.6, True, normalize=True, budget=budget, losses=True)
        _check_against(f"{name} fp32 normalize budget={budget}", got, _reference(kw, a, 0.6, normalize=True), True)


def test_no_grad_forward_gives_the_per_sample_losses():
    kw = dict(hard_negatives=K_NEG, exclude_groups=True)
    a = _inputs(300, 136, 72, kw, seed=9)
    with torch.no_grad():
        got = _module_call(kw, a, 0.8, True, losses=True, grad=False)
    ref = _reference(kw, a, 0.8)
    _check("no-grad loss", got["loss"], ref["loss"])
    _check("no-grad image_loss", got["image_loss"], ref["image_loss"])
    _check("no-grad text_loss", got["text_loss"], ref["text_loss"])
    assert (got["image_loss"] >= 0).all() and (got["text_loss"] >= 0).all()


def _same_bits(tag, x, y, keys=("loss", "dimg", "dtxt", "dtp", "db")):
    for k in keys:
        assert torch.equal(x[k], y[k]), f"{tag}: {k} differs"


@pytest.mark.parametrize("fused", [True, False])
def test_statistics_change_no_bit_of_the_distillation_step(fused):
    """kModeDistill (no statistics) against kModeDistillOpts (per-sample losses, top-K): loss, gradients, dt', dbias and
    the top-1 metrics are the same bits."""
    kw = dict(multi_positive=True)
    a = _inputs(700, 136, 72, kw, seed=3)
    plain = _module_call(kw, a, 0.5, fused, topk=1, options=False)
    for losses, topk in ((True, 1), (False, 5), (True, 5)):
        got = _module_call(kw, a, 0.5, fused, losses=losses, topk=topk)
        _same_bits(f"losses={losses} topk={topk}", got, plain,
                   ("loss", "dimg", "dtxt", "dtp", "db", "i2t_top1", "t2i_top1", "i2t_index", "t2i_index"))


def test_unique_groups_change_no_bit():
    kw = dict(sample_weights=True)
    a = _inputs(700, 136, 72, kw, seed=4)
    plain = _module_call(kw, a, 0.5, True, options=False)
    a["kw"]["image_groups"] = torch.arange(700)
    a["kw"]["text_groups"] = torch.arange(700) + 700
    _same_bits("unique groups", _module_call(dict(kw, exclude_groups=True), a, 0.5, True), plain)


def test_one_label_per_set_is_the_ids_step():
    a = _inputs(700, 136, 72, dict(multi_positive=True), seed=6)
    ids = _module_call(dict(multi_positive=True), a, 0.5, True, options=False)
    a["kw"] = dict(sample_labels=a["kw"]["sample_ids"][:, None])
    _same_bits("M = 1 sets vs ids", _module_call(dict(multi_label=1), a, 0.5, True), ids)


@pytest.mark.parametrize("name,kw", [CELLS[0], CELLS[2], CELLS[-1]], ids=["hard_negatives", "extra_images", "several"])
def test_teacher_equal_to_the_student_at_lambda_one_leaves_no_gradient(name, kw):
    a = _inputs(300, 136, 136, kw, seed=8)
    a["timg"], a["ttxt"] = a["img"], a["txt"]
    # the teacher's scalars are the module's own (t' = log 10, b = -10)
    got = _module_call(kw, a, 1.0, True, losses=True, tscalars=(math.log(10.0), -10.0))
    for k in ("dimg", "dtxt"):
        assert not got[k].any(), f"{name}: {k} is not exactly zero"


# ---- the engine, other ranks through the loopback hooks ----

def _engine(B, W, r, Bs, Ts, D, DT, bidir):
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi

    eng = SigmoidLossEngine(B, D, _dev(), rank_world=(r, W), loopback=W > 1, batch_per_rank=Bs, texts_per_rank=Ts,
                            teacher_dim=DT, distill_options=True)
    if bidir:
        eng.set_option(_capi.SIGLIP_OPT_BIDIR, 1)
    eng.set_option(_capi.SIGLIP_OPT_DISTILL, 1)
    eng.set_option(_capi.SIGLIP_OPT_EXCLUDE_GROUPS, 1)
    return eng


@pytest.mark.parametrize("sched", ["fused", "split"])
@pytest.mark.parametrize("Bs,K,bidir", [([256, 190], 64, False), ([200, 130, 257], 40, True)])
def test_loopback_hard_negatives_and_groups_match_the_oracle(Bs, K, bidir, sched):
    W, D, DT, lam = len(Bs), 136, 72, 0.7
    Ts = [b + K for b in Bs]
    g = torch.Generator().manual_seed(W * 17 + K)
    imgs = [_unit(g, b, D).to(torch.bfloat16) for b in Bs]
    txts = [_unit(g, t, D).to(torch.bfloat16) for t in Ts]
    timgs = [_unit(g, b, DT).to(torch.bfloat16) for b in Bs]
    ttxts = [_unit(g, t, DT).to(torch.bfloat16) for t in Ts]
    igs = [torch.randint(-1, 30, (b,), generator=g) for b in Bs]
    tgs = [torch.randint(-1, 30, (t,), generator=g) for t in Ts]
    f = (lambda xs: [x.double().numpy() for x in xs])  # noqa: E731
    from extra_images_oracle import label_blocks

    labels = group_labels(label_blocks(Bs, Bs, Ts), [x.numpy() for x in igs], [x.numpy() for x in tgs])
    ref = closed_form_distill_options(f(imgs), f(txts), math.log(10.0), -10.0, f(timgs), f(ttxts), TTP, TBIAS, lam,
                                      labels, Bs)
    d = _dev()
    sc = lambda x: torch.tensor([x], device=d, dtype=torch.float32)  # noqa: E731
    for r in range(W):
        eng = _engine(Bs[r], W, r, Bs, Ts, D, DT, bidir)
        for k in range(W):
            eng.debug_set_text_chunk(k, txts[k].to(d))
            eng.debug_set_teacher_text_chunk(k, ttxts[k].to(d))
            if k != r:
                eng.debug_set_chunk_groups(k, tgs[k].to(d))
        eng.set_groups(igs[r].to(d), tgs[r].to(d))
        # set_teacher records pointers: the tensors stay referenced until the step has run
        teacher = (timgs[r].to(d), ttxts[r].to(d), sc(TTP), sc(TBIAS))
        eng.set_teacher(*teacher, lam)
        il, tl = torch.empty(Bs[r], device=d), torch.empty(Ts[r], device=d)
        eng.request_sample_losses(il, tl)
        img, txt = imgs[r].to(d), txts[r].to(d)
        if sched == "fused":
            loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, sc(math.log(10.0)), sc(-10.0))
        else:
            loss = eng.forward(img, txt, sc(math.log(10.0)), sc(-10.0), True)
            dimg, dtxt, dtp, db = eng.backward(img, txt, sc(math.log(10.0)), None)
        slots = {k: eng.debug_get_slot(k).clone() for k in range(W) if k != r}
        torch.cuda.synchronize()
        tag = f"W={W} rank {r} {sched}"
        _check(f"{tag} loss", loss, ref[r]["loss"])
        _check(f"{tag} dimg", dimg, ref[r]["dimg"])
        _check(f"{tag} dt_prime", dtp, ref[r]["dt_prime"])
        _check(f"{tag} dbias", db, ref[r]["dbias"])
        for k in range(W):
            _check(f"{tag} contribution to chunk {k}", dtxt.float() if k == r else slots[k], ref[r]["contrib"][k])
        _check(f"{tag} image_loss", il, ref[r]["image_loss"])
        eng.close()


# ---- the C-ABI statuses: a siglip_ctx_create_distill_extras context takes what a siglip_ctx_create_distill one refuses

def test_requests_under_distillation_depend_on_the_context():
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi

    B, D = 64, 64
    L = _capi.lib()
    sc = lambda x: torch.tensor([x], device=_dev(), dtype=torch.float32)  # noqa: E731
    recall = torch.empty(10, device=_dev())
    il, tl = torch.empty(B, device=_dev()), torch.empty(B, device=_dev())
    old = SigmoidLossEngine(B, D, _dev(), teacher_dim=D)   # siglip_ctx_create_distill: refusals unchanged
    old.set_option(_capi.SIGLIP_OPT_DISTILL, 1)
    assert L.siglip_request_topk(old._h, 5, recall.data_ptr(), None, None) == _capi.SIGLIP_ERR_STATE
    assert L.siglip_request_sample_losses(old._h, il.data_ptr(), tl.data_ptr()) == _capi.SIGLIP_ERR_STATE
    assert L.siglip_ctx_set_option(old._h, _capi.SIGLIP_OPT_EXCLUDE_GROUPS, 1) == _capi.SIGLIP_ERR_STATE
    old.set_option(_capi.SIGLIP_OPT_DISTILL, 0)
    old.set_option(_capi.SIGLIP_OPT_EXCLUDE_GROUPS, 1)
    assert L.siglip_ctx_set_option(old._h, _capi.SIGLIP_OPT_DISTILL, 1) == _capi.SIGLIP_ERR_STATE
    old.close()
    for armed_first in (False, True):   # the requests before or after the option: both run
        dis = SigmoidLossEngine(B, D, _dev(), teacher_dim=D, distill_options=True)
        if armed_first:
            assert L.siglip_request_topk(dis._h, 5, recall.data_ptr(), None, None) == _capi.SIGLIP_OK
            assert L.siglip_request_sample_losses(dis._h, il.data_ptr(), tl.data_ptr()) == _capi.SIGLIP_OK
        dis.set_option(_capi.SIGLIP_OPT_DISTILL, 1)
        if not armed_first:
            assert L.siglip_request_topk(dis._h, 5, recall.data_ptr(), None, None) == _capi.SIGLIP_OK
            assert L.siglip_request_sample_losses(dis._h, il.data_ptr(), tl.data_ptr()) == _capi.SIGLIP_OK
        x = torch.nn.functional.normalize(torch.randn(B, D, device=_dev())).to(torch.bfloat16)
        tsc = (sc(math.log(10.0)), sc(-10.0))   # recorded as pointers: referenced until the step has run
        dis.set_teacher(x, x, *tsc, 0.5)
        loss = dis.fwd(x, x, sc(math.log(10.0)), sc(-10.0))
        torch.cuda.synchronize()
        assert float(recall[4]) == 1.0   # every image finds its own caption among its 5 best
        assert abs(float(il.sum()) / B - float(loss)) <= 1e-5 * abs(float(loss))
        dis.close()


def test_options_compose_with_distill_in_either_order():
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi

    L = _capi.lib()
    for opt in (_capi.SIGLIP_OPT_EXCLUDE_GROUPS, _capi.SIGLIP_OPT_LABEL_SETS):
        for distill_first in (False, True):
            eng = SigmoidLossEngine(64, 64, _dev(), teacher_dim=64, labels=2, distill_options=True)
            order = [_capi.SIGLIP_OPT_DISTILL, opt] if distill_first else [opt, _capi.SIGLIP_OPT_DISTILL]
            for o in order:
                assert L.siglip_ctx_set_option(eng._h, o, 1) == _capi.SIGLIP_OK, L.siglip_last_error()
            # focal stays refused under distillation
            assert L.siglip_ctx_set_option(eng._h, _capi.SIGLIP_OPT_FOCAL, 1) == _capi.SIGLIP_ERR_STATE
            eng.close()
