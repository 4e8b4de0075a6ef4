"""CPU checks of the non-finite oracle: float64 autograd of ``exclude_groups_oracle.torch_loss`` on the operand values
the kernels consume (``operand_values``), with NaN and +-inf in embeddings and scalars. Hand-made cases pin where the
non-finite values land (a NaN in text j: every dimg row and dtxt row j; an inf image entry at dimension k: column k of
dtxt), the per-sample-loss classes (``sample_loss_classes``: NaN and +inf partials, partials of 2^16 and more), the
distillation terms and the finite degenerate case of a zero row under normalize."""
import math

import numpy as np
import pytest
import torch

from distill_oracle import closed_form_distill
from exclude_groups_oracle import (COL_PARTIAL_ROWS, ROW_PARTIAL_COLS, operand_values, sample_loss_classes,
                                   torch_loss, torch_terms)

TP, BIAS = math.log(10.0), -10.0


def _unit(g, n, d):
    return torch.nn.functional.normalize(torch.randn(n, d, generator=g, dtype=torch.float64))


def _labels(R, B, T):
    y = -torch.ones(R, T, dtype=torch.float64)
    y[torch.arange(B), torch.arange(B)] = 1.0
    return y


def _grads(img, txt, y, tp=TP, bias=BIAS, **kw):
    """loss, dimg, dtxt, dt', dbias and the pair terms by float64 autograd."""
    xi, xt = img.clone().requires_grad_(True), txt.clone().requires_grad_(True)
    tpt = torch.tensor(tp, dtype=torch.float64, requires_grad=True)
    bt = torch.tensor(bias, dtype=torch.float64, requires_grad=True)
    loss = torch_loss(xi, xt, tpt, bt, y, batch=kw.pop("batch", None), **kw)
    loss.backward()
    terms = torch_terms(img, txt, torch.tensor(tp, dtype=torch.float64), torch.tensor(bias, dtype=torch.float64), y,
                        **kw)
    return dict(loss=loss.detach(), dimg=xi.grad, dtxt=xt.grad, dtp=tpt.grad, db=bt.grad, terms=terms)


def _bad(x):
    return ~torch.isfinite(torch.as_tensor(x))


def _problem(B=12, D=10, K=0, E=0, seed=0):
    g = torch.Generator().manual_seed(seed)
    return _unit(g, B + E, D) * 2, _unit(g, B + K, D) * 2, _labels(B + E, B, B + K)


def test_finite_inputs_give_finite_outputs():
    img, txt, y = _problem()
    r = _grads(img, txt, y)
    assert all(bool(torch.isfinite(v).all()) for v in r.values())


def test_nan_in_a_text_poisons_every_image_row_and_its_own_text_row():
    img, txt, y = _problem()
    j = 5
    txt[j, 3] = float("nan")
    r = _grads(img, txt, y)
    assert _bad(r["loss"]) and _bad(r["dtp"]) and _bad(r["db"])
    assert bool(_bad(r["dimg"]).all())                     # G[:, j] is NaN: every image row
    rows = _bad(r["dtxt"]).any(dim=1)
    assert rows.tolist() == [i == j for i in range(txt.shape[0])]   # G[:, j] reaches dtxt row j only
    assert bool(_bad(r["dtxt"][j]).all())


@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_inf_image_entry_makes_column_k_of_dtxt_non_finite(sign):
    img, txt, y = _problem(seed=1)
    i, k = 4, 7
    img[i, k] = sign * float("inf")
    r = _grads(img, txt, y)
    # z[i, :] = +-inf: the loss is +inf through the negatives at +inf, while the pair gradients sigma(.) stay finite
    assert float(r["loss"]) == float("inf")
    assert bool(torch.isfinite(r["dimg"]).all()) and bool(torch.isfinite(r["db"]))
    assert _bad(r["dtp"])                                   # t sum G s with s = +-inf
    bad = _bad(r["dtxt"])
    assert bool(bad[:, k].all()) and not bool(bad[:, [c for c in range(txt.shape[1]) if c != k]].any())


def test_nan_row_of_an_extra_image_and_of_a_hard_negative():
    B, K, E = 10, 3, 2
    img, txt, y = _problem(B, 8, K, E, seed=2)
    img[B + 1] = float("nan")
    r = _grads(img, txt, y, batch=B)
    assert _bad(r["dimg"]).any(dim=1).tolist() == [i == B + 1 for i in range(B + E)]
    assert bool(_bad(r["dtxt"]).all())
    img, txt, y = _problem(B, 8, K, E, seed=3)
    txt[B + 2, 0] = float("inf")
    r = _grads(img, txt, y, batch=B)
    # column B + 2 of the logits is +-inf: dimg column 0 is non-finite in every row, dtxt row B + 2 stays finite
    assert bool(_bad(r["dimg"][:, 0]).all()) and not bool(_bad(r["dimg"][:, 1:]).any())
    assert not bool(_bad(r["dtxt"]).any())


def test_non_finite_scalars():
    img, txt, y = _problem(seed=4)
    r = _grads(img, txt, y, tp=float("nan"))
    assert all(bool(_bad(r[k]).all()) for k in ("loss", "dimg", "dtxt", "dtp", "db"))
    r = _grads(img, txt, y, bias=float("nan"))
    assert all(bool(_bad(r[k]).all()) for k in ("loss", "dimg", "dtxt", "dtp", "db"))
    # t' = 1000: t = exp(t') is +inf in float64 as in fp32; every logit is +-inf, dbias = sum G stays finite
    r = _grads(img, txt, y, tp=1000.0)
    assert float(r["loss"]) == float("inf") and bool(torch.isfinite(r["db"]))
    assert all(bool(_bad(r[k]).all()) for k in ("dimg", "dtxt", "dtp"))


def test_operand_values():
    x = torch.tensor([[1.0 / 3.0, float("nan"), float("inf"), -float("inf"), 5000.0, -1e30, 0.0, 2.0 ** -20]])
    v = operand_values(x)
    assert math.isnan(float(v[0, 1])) and float(v[0, 2]) == float("inf") and float(v[0, 3]) == -float("inf")
    assert float(v[0, 0]) == float(torch.tensor(16.0 / 3.0).half()) / 16.0 != 1.0 / 3.0
    assert float(v[0, 4]) == 4094.0 and float(v[0, 5]) == -4094.0 and float(v[0, 6]) == 0.0
    assert float(v[0, 7]) == float(torch.tensor(2.0 ** -16).half()) / 16.0
    torch.testing.assert_close(operand_values(x.half()), operand_values(x.half().float()), rtol=0, atol=0,
                               equal_nan=True)
    b = x.to(torch.bfloat16)   # bf16 as it is (NaN != NaN: compared through its pattern)
    ob = operand_values(b)
    assert torch.equal(torch.isnan(ob), torch.isnan(b.double()))
    assert torch.equal(torch.nan_to_num(ob, nan=0.0), torch.nan_to_num(b.double(), nan=0.0))


def test_sample_loss_classes():
    B, D = 40, 16
    g = torch.Generator().manual_seed(5)
    img, txt = _unit(g, B, D), _unit(g, B, D)
    y = _labels(B, B, B)
    # finite: the row and column sums
    t = torch_terms(img, txt, torch.tensor(TP, dtype=torch.float64), torch.tensor(BIAS, dtype=torch.float64), y)
    c = sample_loss_classes(t, [B])
    np.testing.assert_allclose(c["image_loss"], t.sum(1).numpy(), rtol=1e-14)
    np.testing.assert_allclose(c["text_loss_part"], t.sum(0).numpy(), rtol=1e-14)
    # a NaN in text j: every image loss NaN (each row partial over j's tile), text j NaN, every other text finite
    txt2 = txt.clone()
    txt2[7, 2] = float("nan")
    c = sample_loss_classes(torch_terms(img, txt2, torch.tensor(TP, dtype=torch.float64),
                                        torch.tensor(BIAS, dtype=torch.float64), y), [B])
    assert bool(np.isnan(c["image_loss"]).all())
    assert np.isnan(c["text_loss_part"]).tolist() == [j == 7 for j in range(B)]
    # +inf terms (an image entry at +inf): +inf, not NaN, wherever no partial is NaN
    img2 = img.clone()
    img2[3, 0] = float("inf")
    t2 = torch_terms(img2, txt, torch.tensor(TP, dtype=torch.float64), torch.tensor(BIAS, dtype=torch.float64), y)
    c = sample_loss_classes(t2, [B])
    assert float(c["image_loss"][3]) == float("inf") and np.isfinite(np.delete(c["image_loss"], 3)).all()
    hot = np.isinf(t2[3].numpy())
    assert (np.isinf(c["text_loss_part"]) == hot).all() and hot.any() and not np.isnan(c["text_loss_part"]).any()


def test_sample_loss_overflow_is_per_partial():
    """A row whose terms sum past 2^16 within one 128-column partial is +inf; the same total spread over partials that
    each stay below 2^16 is finite."""
    R, T = 2 * COL_PARTIAL_ROWS, 3 * ROW_PARTIAL_COLS
    terms = np.zeros((R, T))
    terms[0, :ROW_PARTIAL_COLS] = 600.0            # one partial of 76800
    terms[1, :] = 400.0                             # three partials of 51200, total 153600
    terms[2, 5] = float("inf")
    c = sample_loss_classes(terms, [T])
    assert float(c["image_loss"][0]) == float("inf") and float(c["image_loss"][1]) == 400.0 * T
    assert float(c["image_loss"][2]) == float("inf") and float(c["image_loss"][3]) == 0.0
    assert np.isinf(c["text_loss_part"]).tolist() == [j == 5 for j in range(T)]
    # two chunks: the partials restart at each chunk's first column
    c = sample_loss_classes(np.full((1, 200), 600.0), [100, 100])   # 60000 + 60000
    assert float(c["image_loss"][0]) == 120000.0
    c = sample_loss_classes(np.full((1, 200), 600.0), [200])        # 76800 + 43200
    assert float(c["image_loss"][0]) == float("inf")


def test_distillation_terms_match_the_distillation_oracle_and_propagate_teacher_nan():
    B, D, DT, lam = 9, 8, 6, 0.6
    g = torch.Generator().manual_seed(6)
    img, txt, timg, ttxt = _unit(g, B, D), _unit(g, B, D), _unit(g, B, DT), _unit(g, B, DT)
    y = _labels(B, B, B)
    teacher = (timg, ttxt, math.log(20.0), -8.0, lam)
    r = _grads(img, txt, y, teacher=teacher)
    ref = closed_form_distill([img.numpy()], [txt.numpy()], TP, BIAS, [timg.numpy()], [ttxt.numpy()], math.log(20.0),
                              -8.0, lam)[0]
    assert float(r["loss"]) == pytest.approx(ref["loss"], rel=1e-12)
    np.testing.assert_allclose(r["dimg"].numpy(), ref["dimg"], rtol=1e-10, atol=1e-14)
    np.testing.assert_allclose(r["dtxt"].numpy(), ref["contrib"][0], rtol=1e-10, atol=1e-14)
    assert float(r["dtp"]) == pytest.approx(ref["dt_prime"], rel=1e-10)
    assert float(r["db"]) == pytest.approx(ref["dbias"], rel=1e-10)
    # a NaN teacher image row i: the targets of row i are NaN, so dimg row i and every dtxt row are NaN
    timg = timg.clone()
    timg[2, 1] = float("nan")
    r = _grads(img, txt, y, teacher=(timg, ttxt, math.log(20.0), -8.0, lam))
    assert _bad(r["loss"]) and _bad(r["dtp"]) and _bad(r["db"])
    assert _bad(r["dimg"]).any(dim=1).tolist() == [i == 2 for i in range(B)]
    assert bool(_bad(r["dtxt"]).all())


def test_zero_row_under_normalize_is_dxhat_over_eps():
    """F.normalize of a zero row is 0 and its gradient dxhat / 1e-12: what normalize_bwd computes with inv = 1e12."""
    img, txt, y = _problem(seed=7)
    img[3] = 0.0
    r = _grads(img, txt, y, normalize=True)
    xh = torch.nn.functional.normalize(img).requires_grad_(True)
    th = torch.nn.functional.normalize(txt)
    loss = torch_loss(xh, th, torch.tensor(TP, dtype=torch.float64), torch.tensor(BIAS, dtype=torch.float64), y)
    loss.backward()
    torch.testing.assert_close(r["dimg"][3], xh.grad[3] / 1e-12, rtol=1e-12, atol=0)
    assert bool(torch.isfinite(r["dimg"]).all()) and float(r["dimg"][3].abs().max()) > 1e9
