"""256-column tiles of the gradient kernel (wgmma m64n256, SIGLIP_OPT_GRAD_TILE_N = 256) against 128-column ones:
every schedule, output format, cluster shape and stage request that the gradient kernel runs must give the same bits,
because each output element is accumulated over k in the same order whatever the tile width. One comparison against
the float64 oracle at a shape that is not a multiple of any tile."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _dev():
    return torch.device("cuda", 0)


def _scal(x):
    return torch.tensor([x], device=_dev(), dtype=torch.float32)


def _emb(n, D, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.nn.functional.normalize(torch.randn(n, D, generator=g)).to(torch.bfloat16).to(_dev())


def _engine(B, D, cg=2, **kw):
    from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi

    eng = SigmoidLossEngine(B, D, _dev(), cta_group=cg, **kw)
    eng.set_option(_capi.SIGLIP_OPT_SPLIT_K, 0)   # split-K always runs 128-column tiles
    return eng


def _set_width(eng, tn):
    from distributed_sigmoid_loss_b200 import _capi

    eng.set_option(_capi.SIGLIP_OPT_GRAD_TILE_N, tn)


def _fused(eng, img, txt, grad_dtype=torch.float32):
    out = {}
    for tn in (128, 256):
        _set_width(eng, tn)
        _, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, _scal(math.log(10.0)), _scal(-10.0), grad_dtype)
        torch.cuda.synchronize()
        out[tn] = (dimg.clone(), dtxt.clone(), dtp.clone(), db.clone())
    return out


def _assert_same(out):
    for a, b, name in zip(out[128], out[256], ("dimg", "dtxt", "dt_prime", "dbias")):
        assert torch.equal(a, b), f"{name}: 256-column tiles differ from 128-column ones by {(a.float() - b.float()).abs().max():.3e}"


def test_split_schedule_bf16_outputs():
    """siglip_forward + siglip_backward with bf16 gradients written by the kernel epilogue."""
    B, D = 2048, 768
    img, txt = _emb(B, D, 1), _emb(B, D, 2)
    eng = _engine(B, D)
    tp, b = _scal(math.log(10.0)), _scal(-10.0)
    out = {}
    for tn in (128, 256):
        _set_width(eng, tn)
        eng.forward(img, txt, tp, b, True)
        dimg, dtxt, dtp, db = eng.backward(img, txt, tp, None, torch.bfloat16)
        torch.cuda.synchronize()
        assert dimg.dtype == torch.bfloat16
        out[tn] = (dimg.clone(), dtxt.clone(), dtp.clone(), db.clone())
    _assert_same(out)
    eng.close()


@pytest.mark.parametrize("cg", [1, 2])
def test_four_cta_clusters(cg):
    """SIGLIP_OPT_MCAST = 2: clusters of 2 (cta_group 1) or 4 CTAs; a 4-CTA cluster fetches one whole {64, 64} box of
    the 256-column B tile per CTA."""
    from distributed_sigmoid_loss_b200 import _capi

    B, D = 2048, 1024
    eng = _engine(B, D, cg)
    eng.set_option(_capi.SIGLIP_OPT_MCAST, 2)
    _assert_same(_fused(eng, _emb(B, D, 3), _emb(B, D, 4)))
    eng.close()


@pytest.mark.parametrize("stages", [4, 6])
def test_stage_requests(stages):
    """Both pipeline depths the option accepts; 256-column tiles run 4 stages either way."""
    from distributed_sigmoid_loss_b200 import _capi

    B, D = 1536, 512
    eng = _engine(B, D)
    eng.set_option(_capi.SIGLIP_OPT_STAGES_GRAD, stages)
    _assert_same(_fused(eng, _emb(B, D, 5), _emb(B, D, 6)))
    eng.close()


def test_hard_negatives_and_extra_texts():
    """T > B texts: the dimg contraction has K = T, the dtxt one M = T rows, of which the last T - B take no
    positive-pair term."""
    B, T, D = 1000, 1304, 256
    eng = _engine(B, D, texts_per_rank=[T])
    _assert_same(_fused(eng, _emb(B, D, 7), _emb(T, D, 8)))
    eng.close()


def test_two_rank_loopback_with_in_kernel_fold():
    """Rank 1 of a 2-rank step on one GPU: two gradient launches, the second adds the folded peer contribution
    (p1_wait_flag), seeded non-zero through the loopback stand-in, and the running dimg of the first."""
    B, D = 1024, 768
    out = {}
    peer = _emb(B, D, 22).float() * 1e-3
    for tn in (128, 256):
        eng = _engine(B, D, rank_world=(1, 2), loopback=True)
        _set_width(eng, tn)
        for k in range(2):
            eng.debug_set_text_chunk(k, _emb(B, D, 20 + k))
        eng.debug_set_peer_contribution(0, peer)
        _, dimg, dtxt, dtp, db = eng.fwd_bwd(_emb(B, D, 30), _emb(B, D, 21), _scal(math.log(10.0)), _scal(-10.0))
        torch.cuda.synchronize()
        out[tn] = (dimg.clone(), torch.cat([dtxt.float(), eng.debug_get_slot(0)]), dtp.clone(), db.clone())
        eng.close()
    _assert_same(out)


@pytest.mark.parametrize("D", [264, 1160])
def test_partial_last_column_tile(D):
    """D not a multiple of 256 (nor of 128): the last tile's columns past D are fetched as zeros and never written."""
    B = 1280
    eng = _engine(B, D)
    _assert_same(_fused(eng, _emb(B, D, 9), _emb(B, D, 10)))
    eng.close()


def test_headline_shape():
    """B = 16384, D = 1024: the shape the benchmark measures, and the default width there is 256."""
    B, D = 16384, 1024
    img, txt = _emb(B, D, 11), _emb(B, D, 12)
    eng = _engine(B, D)
    out = _fused(eng, img, txt)
    _assert_same(out)
    _set_width(eng, 0)
    _, dimg, dtxt, _, _ = eng.fwd_bwd(img, txt, _scal(math.log(10.0)), _scal(-10.0))
    torch.cuda.synchronize()
    assert torch.equal(dimg, out[256][0]) and torch.equal(dtxt, out[256][1])
    eng.close()


def test_against_float64_oracle_at_a_ragged_shape():
    """256-column tiles at B = 1000, D = 392 (two tiles, the second 136 columns of 256) within the 1e-3 budget of the
    float64 closed form."""
    from oracle.siglip_oracle import closed_form

    B, D = 1000, 392
    img, txt = _emb(B, D, 13), _emb(B, D, 14)
    eng = _engine(B, D)
    _set_width(eng, 256)
    tp, bias = math.log(10.0), -10.0
    loss, dimg, dtxt, dtp, db = eng.fwd_bwd(img, txt, _scal(tp), _scal(bias))
    torch.cuda.synchronize()
    ref = closed_form(img.double().cpu().numpy(), txt.double().cpu().numpy(), tp, bias, 1)[0]
    for name, got, want in (("dimg", dimg, ref["dimg"]), ("dtxt", dtxt, ref["dtxt"])):
        got = got.double().cpu().numpy()
        ef = np.linalg.norm(got - want) / np.linalg.norm(want)
        em = np.abs(got - want).max() / np.abs(want).max()
        assert ef <= 1e-3 and em <= 1e-3, f"{name}: rel-Frobenius {ef:.3e}, max-abs/max {em:.3e}"
    assert abs(float(dtp) - ref["dt_prime"]) <= 1e-3 * abs(ref["dt_prime"])
    assert abs(float(db) - ref["dbias"]) <= 1e-3 * abs(ref["dbias"])
    eng.close()
