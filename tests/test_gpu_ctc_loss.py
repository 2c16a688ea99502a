"""
CTC loss on the sm_90a kernels (csrc/ctc_loss.cu, bonito_b200.ctc.loss) against torch's CPU ctc_loss in float64 on the
same fp32 log-probs.  The non-finite pattern (which losses are inf, which gradient entries NaN) must match exactly; finite
losses must be within LOSS_ABS + LOSS_REL |ref| per sample (for 'mean' / 'sum', of the reduced value) and gradients
within GRAD_TOL per unit of upstream gradient (max |g|: 1 for 'none' and 'sum', 1 / (N min(target_lengths, 1)) for
'mean').  The fp32 log-sum-exp rounding adds up over the frames: measured on an H100, the gradient error per unit of g is
5.2e-5 at 200 frames of peaked log-probs, 1.05e-4 at the QuartzNet shape (1334 frames, ~430 labels; torch's own CUDA
kernel is 1.65e-3 off there) and 3.1e-2 with a 4096-label target in 4396 frames (MAX_TARGET_GRAD_TOL).  Also: bitwise-equal results over two runs, a second backward, the refusals, `Model.loss` of a seeded
QuartzNet v1 model against the reference's formula in float64, and torch's own CUDA ctc_loss.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import _oracle_ctc_loss as O
from bonito_b200 import native, synth
from bonito_b200.ctc.loss import ctc_loss
from bonito_b200.ctc.model import Model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LOSS_ABS, LOSS_REL = 1e-3, 1e-5
GRAD_TOL = 2e-4
MAX_TARGET_GRAD_TOL = 5e-2
TORCH_CUDA_GRAD_TOL = 5e-3


def _inputs(c, dtype=torch.float32):
    lp = torch.from_numpy(c["log_probs"]).to(dtype)
    return lp, torch.from_numpy(c["targets"]), torch.from_numpy(c["input_lengths"]), torch.from_numpy(c["target_lengths"])


def _reference(lp, targets, il, tl, blank, reduction, zero_infinity):
    x = lp.double().cpu().requires_grad_()
    loss = F.ctc_loss(x, targets.cpu(), il.cpu(), tl.cpu(), blank=blank, reduction=reduction, zero_infinity=zero_infinity)
    loss.sum().backward()
    return loss.detach(), x.grad


def _native(lp, targets, il, tl, blank, reduction, zero_infinity, retain_graph=False):
    x = lp.to(DEV).requires_grad_()
    loss = ctc_loss(x, targets.to(DEV), il, tl, blank=blank, reduction=reduction, zero_infinity=zero_infinity)
    loss.sum().backward(retain_graph=retain_graph)
    return loss, x


def _errors(loss, grad, ref_loss, ref_grad, g_max=1.0):
    """(worst loss error over its bound, worst gradient |d| / g_max), after checking the non-finite patterns are equal."""
    loss, grad = loss.detach().double().cpu().reshape(-1), grad.double().cpu()
    ref_loss = ref_loss.reshape(-1)
    assert torch.equal(torch.isinf(loss), torch.isinf(ref_loss)) and torch.equal(torch.isnan(loss), torch.isnan(ref_loss))
    assert torch.equal(torch.isnan(grad), torch.isnan(ref_grad)) and not torch.isinf(grad).any()
    fin = torch.isfinite(ref_loss)
    lerr = float(((loss[fin] - ref_loss[fin]).abs() / (LOSS_ABS + LOSS_REL * ref_loss[fin].abs())).max()) if fin.any() else 0.
    ok = ~torch.isnan(ref_grad)
    gerr = float((grad[ok] - ref_grad[ok]).abs().max()) / g_max if ok.any() else 0.
    return lerr, gerr


def _g_max(reduction, tl):
    return 1.0 / (len(tl) * max(int(tl.min()), 1)) if reduction == "mean" else 1.0


@pytest.mark.parametrize("zero_infinity", [False, True])
@pytest.mark.parametrize("reduction", ["none", "sum", "mean"])
@pytest.mark.parametrize("c", O.cases(), ids=lambda c: c["name"])
def test_cases_against_torch_cpu_float64(c, reduction, zero_infinity):
    args = _inputs(c) + (c["blank"], reduction, zero_infinity)
    loss, x = _native(*args)
    ref_loss, ref_grad = _reference(*args)
    lerr, gerr = _errors(loss, x.grad, ref_loss, ref_grad, _g_max(reduction, c["target_lengths"]))
    il = c["input_lengths"]
    for n in range(len(il)):
        assert not x.grad[il[n]:, n].any()                  # exactly 0 past the input length
    print(f"{c['name']} {reduction} zero_infinity={zero_infinity}: loss {lerr:.3f} of bound, grad max|d|/g {gerr:.2e}")
    assert lerr <= 1.0 and gerr <= GRAD_TOL


def _long_target(L, seed):
    rng = np.random.default_rng(seed)
    t = [int(rng.integers(1, 5))]
    while len(t) < L:                                       # no repeats: L frames suffice
        t.append(int(rng.choice([c for c in range(1, 5) if c != t[-1]])))
    return t


def test_target_at_the_limit_and_one_over():
    L = native.ctc_loss_max_target()
    assert L >= 4096
    c = O.case("max_target", L + 300, 2, 5, [L + 300, L + 37], [_long_target(L, 1), _long_target(L - 1, 2)], seed=11)
    args = _inputs(c) + (0, "none", False)
    loss, x = _native(*args)
    lerr, gerr = _errors(loss, x.grad, *_reference(*args))
    print(f"max target {L}: loss {lerr:.3f} of bound, grad max|d| {gerr:.2e}")
    assert lerr <= 1.0 and gerr <= MAX_TARGET_GRAD_TOL
    over = O.case("over", L + 2, 1, 5, [L + 2], [_long_target(L + 1, 3)], seed=12)
    lp, tg, il, tl = _inputs(over)
    with pytest.raises(ValueError, match="longer than"):
        ctc_loss(lp.to(DEV), tg, il, tl)


def test_batch_larger_than_one_grid_dimension():
    N = 70000
    rng = np.random.default_rng(5)
    targets = [list(rng.integers(1, 5, size=int(rng.integers(0, 3)))) for _ in range(N)]
    c = O.case("wide", 6, N, 5, rng.integers(4, 7, size=N), targets, seed=13)
    args = _inputs(c) + (0, "none", False)
    loss, x = _native(*args)
    lerr, gerr = _errors(loss, x.grad, *_reference(*args))
    assert lerr <= 1.0 and gerr <= GRAD_TOL


def test_fp16_and_permuted_view():
    c = O.cases()[-1]                                       # peaked, 200 frames
    lp, tg, il, tl = _inputs(c)
    half = lp.half()
    x = half.to(DEV).requires_grad_()
    loss = ctc_loss(x, tg, il, tl, reduction="sum")
    loss.backward()
    ref_loss, ref_grad = _reference(half.float(), tg, il, tl, 0, "sum", False)
    assert x.grad.dtype == torch.float16
    lerr, _ = _errors(loss, x.grad.float(), ref_loss, ref_grad)
    assert lerr <= 1.0 and float((x.grad.double().cpu() - ref_grad).abs().max()) <= 1e-3   # fp16 rounding of the gradient
    # the native engine's [N, T, C] layout, permuted to [T, N, C]: read in place, same loss and gradient bits
    base = lp.permute(1, 0, 2).contiguous().to(DEV).requires_grad_()
    view = base.permute(1, 0, 2)
    assert not view.is_contiguous()
    loss_v = ctc_loss(view, tg, il, tl, reduction="none")
    loss_v.sum().backward()
    loss_c, xc = _native(lp, tg, il, tl, 0, "none", False)
    assert torch.equal(loss_v, loss_c) and torch.equal(base.grad.permute(1, 0, 2), xc.grad)


def _quartznet_batch(N=16, T=1334, seed=21):
    rng = np.random.default_rng(seed)
    lengths = rng.integers(380, 480, size=N)
    tg = [list(rng.integers(1, 5, size=int(n))) for n in lengths]
    return O.case("quartznet", T, N, 5, np.full(N, T), tg, seed=seed)


def test_bitwise_reproducible_and_second_backward():
    c = _quartznet_batch()
    lp, tg, il, tl = _inputs(c)
    runs = []
    for _ in range(2):
        loss, x = _native(lp, tg, il, tl, 0, "none", False, retain_graph=True)
        first = x.grad.clone()
        loss.sum().backward()                               # the workspace survives: the second backward adds the same
        assert torch.equal(x.grad, 2 * first)
        runs.append((loss.detach(), first))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    lerr, gerr = _errors(runs[0][0], runs[0][1], *_reference(lp, tg, il, tl, 0, "none", False))
    print(f"quartznet shape: loss {lerr:.3f} of bound, grad max|d| {gerr:.2e}")
    assert lerr <= 1.0 and gerr <= GRAD_TOL


def test_torch_cuda_ctc_loss_agrees():
    c = _quartznet_batch(seed=22)
    lp, tg, il, tl = _inputs(c)
    for reduction in ("none", "mean"):
        loss, x = _native(lp, tg, il, tl, 0, reduction, False)
        y = lp.to(DEV).requires_grad_()
        ref = F.ctc_loss(y, tg.to(DEV), il.to(DEV), tl.to(DEV), reduction=reduction)
        ref.sum().backward()
        lerr, gerr = _errors(loss, x.grad, ref.detach().double().cpu(), y.grad.double().cpu(), _g_max(reduction, tl))
        print(f"torch CUDA {reduction}: loss {lerr:.3f} of bound, grad max|d|/g {gerr:.2e}")
        assert lerr <= 1.0 and gerr <= TORCH_CUDA_GRAD_TOL


def test_refusals():
    c = O.cases()[0]
    lp, tg, il, tl = _inputs(c)
    x = lp.to(DEV)
    with pytest.raises(native.NativeError, match="CUDA"):
        ctc_loss(lp, tg, il, tl)
    with pytest.raises(ValueError, match="reduction"):
        ctc_loss(x, tg, il, tl, reduction="max")
    with pytest.raises(ValueError, match=r"\[T, N, C\]"):
        ctc_loss(x[0], tg, il, tl)
    with pytest.raises(ValueError, match="entries"):
        ctc_loss(x, tg, il[:-1], tl)
    with pytest.raises(ValueError, match="input_lengths"):
        ctc_loss(x, tg, il + 1, tl)
    with pytest.raises(ValueError, match="input_lengths"):
        ctc_loss(x, tg, il * 0, tl)
    with pytest.raises(ValueError, match="negative"):
        ctc_loss(x, tg, il, tl - 1)
    with pytest.raises(ValueError, match="padded targets"):
        ctc_loss(x, tg[:, :1], il, tl)
    with pytest.raises(ValueError, match="blank"):
        ctc_loss(x, tg, il, tl, blank=5)
    n = int(tl.argmax())
    bad = tg.clone()
    bad[n, 0] = 0                                           # the blank as a label
    with pytest.raises(ValueError, match="label"):
        ctc_loss(x, bad, il, tl)
    bad[n, 0] = 5                                           # outside [0, C)
    with pytest.raises(ValueError, match="label"):
        ctc_loss(x, bad, il, tl)
    bad = tg.clone()
    assert int(tl[1]) == 1 < bad.shape[1]
    bad[1, 1] = 9                                           # padding past the target length is not read
    ctc_loss(x, bad, il, tl)


def test_model_loss_on_quartznet_v1_output():
    spec = synth.quartznet_spec("v1", max_repeat=1)
    m = Model(synth.quartznet_config(spec))
    m.load_state_dict(synth.make_quartznet_weights(spec, seed=51))
    m.use_koi(batchsize=8, chunksize=3999, quantize=False)
    m = m.half().eval().to(DEV)
    x = synth.squiggle(8, 3999, seed=4).half()
    with torch.inference_mode():
        out = m(x.to(DEV))                                  # [N, T, 5] fp16
    log_probs = out.clone().permute(1, 0, 2)                # the reference layout, read in place
    T, N, C = log_probs.shape
    rng = np.random.default_rng(6)
    lengths = torch.from_numpy(rng.integers(T // 4, T // 3, size=N))
    targets = torch.from_numpy(rng.integers(1, 5, size=(N, int(lengths.max()))))
    got = m.loss(log_probs, targets, lengths)
    # the reference's formula, evaluated with torch on the CPU in float64 (the smoothing term in the input's dtype)
    lp = log_probs.cpu()
    weights = torch.cat([torch.tensor([0.4]), (0.1 / (C - 1)) * torch.ones(C - 1)])
    ctc = F.ctc_loss(lp.double(), targets, torch.full((N,), T, dtype=torch.int64), lengths, reduction="mean")
    smooth = -((lp * weights).mean())
    assert got["loss"].dtype == torch.float32 and got["label_smooth_loss"].dtype == smooth.dtype
    print(f"Model.loss: ctc {float(got['loss']):.6f} against {float(ctc):.6f}, smoothing {float(got['label_smooth_loss']):.6f}")
    assert abs(float(got["loss"]) - float(ctc)) <= LOSS_ABS + LOSS_REL * abs(float(ctc))
    assert abs(float(got["label_smooth_loss"]) - float(smooth)) <= 1e-5 * abs(float(smooth))
    assert abs(float(got["total_loss"]) - float(ctc + smooth)) <= LOSS_ABS + LOSS_REL * abs(float(ctc + smooth))
    w = torch.tensor([0.2, 0.2, 0.2, 0.2, 0.2])             # a given tensor is used as it is (the reference raises)
    got_w = m.ctc_label_smoothing_loss(log_probs, targets, lengths, weights=w)
    assert abs(float(got_w["label_smooth_loss"]) + float((lp * w).mean())) <= 1e-5 * abs(float((lp * w).mean()))
