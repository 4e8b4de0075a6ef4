"""The per-step inputs of a module step on a recording engine, on CPU: the split schedule's backward re-runs the forward
when another forward ran in between, and that re-run must set the same ids, extra-text and extra-image ids, weights,
groups, label sets and teacher as the forward did (otherwise its gradients would use the previous call's inputs). It
must not re-arm the forward's metric or per-sample-loss requests, and nothing is set again when the saved state is
still this call's, or on the fused schedule."""
import pytest
import torch

from distributed_sigmoid_loss_b200 import loss as loss_mod

B, D, K_TXT, K_IMG, M, DT = 4, 8, 2, 1, 3, 8
R, T = B + K_IMG, B + K_TXT


class RecordingEngine:
    """Stands in for SigmoidLossEngine: the conversions clone, the steps return zeros, every set_* / request_* call
    is logged with its arguments."""

    def __init__(self):
        self.calls = []
        self.saved_generation = 0

    def __getattr__(self, name):
        if name.startswith(("set_", "request_")):
            return lambda *args: self.calls.append((name, args))
        raise AttributeError(name)

    def convert_f32(self, x, f16):
        return x.clone()

    def teacher_operand(self, x, normalize):
        return x.clone()

    def forward(self, img, txt, t_prime, bias, save_for_backward):
        self.saved_generation += 1
        return torch.zeros(1)

    def backward(self, img, txt, t_prime, grad_out, grad_dtype):
        return (torch.zeros(img.shape, dtype=grad_dtype), torch.zeros(txt.shape, dtype=grad_dtype), torch.zeros(1),
                torch.zeros(1))

    def fwd_bwd(self, img, txt, t_prime, bias, grad_dtype):
        self.saved_generation += 1
        return (torch.zeros(1), torch.zeros(img.shape, dtype=grad_dtype), torch.zeros(txt.shape, dtype=grad_dtype),
                torch.zeros(1), torch.zeros(1))

    def scale(self, src, g):
        return src * g


def _step(fused: bool, other_forward_between: bool):
    """One forward + backward of _SigmoidLossFn with all seven per-step inputs; returns the engine's log of the
    forward and of the backward."""
    g = torch.Generator().manual_seed(0)
    ids = lambda n: torch.randint(0, 3, (n,), generator=g)  # noqa: E731
    inputs = loss_mod._StepInputs(
        ids=ids(B), extra_text_ids=ids(K_TXT), extra_image_ids=ids(K_IMG),
        weights=(torch.rand(R, generator=g), torch.rand(T, generator=g)),
        groups=(ids(R), ids(T)),
        label_sets=(torch.randint(-1, 5, (B, M), generator=g), torch.randint(-1, 5, (K_TXT, M), generator=g),
                    torch.randint(-1, 5, (K_IMG, M), generator=g)),
        teacher=(torch.randn(R, DT, generator=g), torch.randn(T, DT, generator=g), torch.tensor(2.0),
                 torch.tensor(-5.0), 0.5))
    img = torch.randn(R, D, generator=g, requires_grad=True)
    txt = torch.randn(T, D, generator=g, requires_grad=True)
    t_prime = torch.tensor(2.3, dtype=torch.float64, requires_grad=True)
    bias = torch.tensor(-10.0, requires_grad=True)
    metrics = (torch.empty(2), torch.empty(R, dtype=torch.int64), torch.empty(T, dtype=torch.int64))
    sample_losses = (torch.empty(R), torch.empty(T))
    eng = RecordingEngine()
    loss = loss_mod._SigmoidLossFn.apply(img, txt, t_prime, bias, eng, False, fused, inputs, metrics, sample_losses)
    fwd, eng.calls = eng.calls, []
    if other_forward_between:
        eng.saved_generation += 1
    loss.backward()
    assert img.grad is not None and txt.grad is not None and t_prime.grad is not None and bias.grad is not None
    return inputs, fwd, eng.calls


def _by_method(calls):
    out = {}
    for name, args in calls:
        out.setdefault(name, []).append(args)
    return out


def test_forward_sets_every_input_and_arms_the_requests():
    inputs, fwd, _ = _step(fused=False, other_forward_between=False)
    seen = _by_method(fwd)
    assert sorted(seen) == ["request_metrics", "request_sample_losses", "set_extra_image_ids", "set_extra_text_ids",
                            "set_groups", "set_label_sets", "set_sample_ids", "set_sample_weights", "set_teacher"]
    assert all(len(v) == 1 for v in seen.values())
    assert seen["set_sample_ids"][0][0] is inputs.ids
    assert seen["set_extra_text_ids"][0][0] is inputs.extra_text_ids
    assert seen["set_extra_image_ids"][0][0] is inputs.extra_image_ids
    assert seen["set_sample_weights"][0] == inputs.weights
    assert seen["set_groups"][0] == inputs.groups
    assert seen["set_label_sets"][0] == inputs.label_sets
    timg, ttxt, ttp, tbias, lam = seen["set_teacher"][0]
    # the teacher goes through teacher_operand (a clone here), the scalars to fp32 [1]
    assert torch.equal(timg, inputs.teacher[0]) and timg is not inputs.teacher[0]
    assert torch.equal(ttxt, inputs.teacher[1]) and ttxt is not inputs.teacher[1]
    assert ttp.dtype == tbias.dtype == torch.float32 and ttp.shape == tbias.shape == (1,) and lam == 0.5


def test_split_rerun_sets_what_the_forward_set():
    _, fwd, rerun = _step(fused=False, other_forward_between=True)
    want = {k: v for k, v in _by_method(fwd).items() if k.startswith("set_")}
    got = _by_method(rerun)
    # per method, not in sequence: the order of these host-side copies does not matter
    assert sorted(got) == sorted(want)
    for name, calls in want.items():
        assert len(got[name]) == len(calls) == 1, name
        assert len(got[name][0]) == len(calls[0]), name
        for a, b in zip(got[name][0], calls[0]):
            assert a is b, name


@pytest.mark.parametrize("fused,other_forward_between", [(False, False), (True, False), (True, True)])
def test_nothing_is_set_again_without_a_rerun(fused, other_forward_between):
    _, fwd, rest = _step(fused, other_forward_between)
    assert len(fwd) == 9 and rest == []
