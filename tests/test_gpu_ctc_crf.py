"""CTC_CRF scoring API and CTC loss on the sm_90a kernels (csrc/ctc_crf.cu) against the float64 oracle
(tests/_oracle_ctc_crf.py).

Tolerances come from fp32 arithmetic: logZ (and every alpha / beta entry) |d| <= 1e-3 + 2e-6 |ref|; posteriors and score
gradients max |d| <= 1e-4; per-chunk loss relative 1e-5.  Max-semiring paths must match exactly."""
import pytest
import torch

import _oracle_ctc_crf as X
from bonito_b200.crf.lattice import target_logz, target_viterbi
from bonito_b200.crf.model import CTC_CRF, Max, SeqdistModel

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _scores(T, N, state_len, seed, quantise=False):
    g = torch.Generator().manual_seed(seed)
    x = 5 * torch.tanh(torch.randn(T, N, 5 * 4 ** state_len, generator=g))
    if quantise:
        x = torch.round(x * 2) / 2
    return x


def _logz_err(got, ref):
    """max of |d| / (1e-3 + 2e-6 |ref|): <= 1 passes."""
    got, ref = got.double().cpu(), ref.double()
    return float(((got - ref).abs() / (1e-3 + 2e-6 * ref.abs())).max())


SHAPES = [(k, N, T) for k in range(1, 6) for N in (1, 3, 37) for T in (1, 2, 7, 400)] + [(4, 3, 2000), (5, 3, 2000)]


@pytest.mark.parametrize("state_len,N,T", SHAPES)
def test_scores_logz_and_posteriors(state_len, N, T):
    x = _scores(T, N, state_len, seed=state_len * 1000 + N * 10 + T)
    xd = x.double()
    seqdist = CTC_CRF(state_len, "NACGT")
    xg = x.to(DEV)
    logz = seqdist.logZ(xg)
    logz_max = seqdist.logZ(xg, Max)
    alpha = seqdist.forward_scores(xg)
    beta = seqdist.backward_scores(xg)
    beta_max = seqdist.backward_scores(xg, Max)
    post = seqdist.posteriors(xg)
    errs = {
        "logZ": _logz_err(logz, X.sparse_logz(xd, state_len)),
        "logZ max": _logz_err(logz_max, X.sparse_logz(xd, state_len, "max")),
        "alpha": _logz_err(alpha, X.sparse_alpha(xd, state_len)),
        "beta": _logz_err(beta, X.sparse_beta(xd, state_len)),
        "beta max": _logz_err(beta_max, X.sparse_beta(xd, state_len, "max")),
    }
    post_err = float((post.double().cpu() - X.sparse_posteriors(xd, state_len)).abs().max())
    print(f"k={state_len} N={N} T={T}: relative to bound {errs}; posteriors max|d| {post_err:.2e}")
    assert alpha.shape == (T + 1, N, 4 ** state_len) and post.shape == x.shape
    assert all(e <= 1.0 for e in errs.values()), errs
    assert post_err <= 1e-4


@pytest.mark.parametrize("quantise", [False, True])
@pytest.mark.parametrize("state_len", [1, 2, 3, 4, 5])
def test_viterbi_equals_oracle(state_len, quantise):
    T, N = 400, 5
    x = _scores(T, N, state_len, seed=7 + state_len, quantise=quantise)
    seqdist = CTC_CRF(state_len, "NACGT")
    path = seqdist.viterbi(x.to(DEV)).cpu()
    ref = X.viterbi(x.double(), state_len)
    onehot = seqdist.posteriors(x.to(DEV), Max).cpu()
    ref_onehot = X.sparse_max_onehot(x.double(), state_len).float()
    print(f"k={state_len} quantised={quantise}: {(path != ref).sum().item()} path differences")
    assert torch.equal(path, ref)
    assert torch.equal(onehot, ref_onehot)


def _targets(N, T, state_len, seed):
    """Zero-padded targets of varying lengths (about 0.45 T), with infeasible chunks: one shorter than state_len and one
    with more moves than frames."""
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(int(0.3 * T) + state_len, int(0.6 * T) + state_len, (N,), generator=g)
    lengths[1] = state_len - 1
    lengths[3] = T + state_len + 2
    width = int(lengths.max()) + 3
    targets = torch.zeros(N, width, dtype=torch.long)
    for n in range(N):
        targets[n, :lengths[n]] = torch.randint(1, 5, (int(lengths[n]),), generator=g)
    return targets, lengths


def _infeasible(lengths, state_len, T):
    lt = lengths + 1 - state_len
    return (lt < 1) | (lt - 1 > T)


@pytest.mark.parametrize("state_len", [2, 3, 5])
@pytest.mark.parametrize("reduction", ["mean", "none"])
@pytest.mark.parametrize("loss_clip", [None, 10.0])
def test_ctc_loss_value_and_gradient(state_len, reduction, loss_clip):
    T, N = 120, 6
    x = _scores(T, N, state_len, seed=11 * state_len)
    targets, lengths = _targets(N, T, state_len, seed=state_len)
    bad = _infeasible(lengths, state_len, T)
    assert bad[1] and bad[3] and not bad[0]
    seqdist = CTC_CRF(state_len, "NACGT")

    xg = x.to(DEV).requires_grad_()
    loss = seqdist.ctc_loss(xg, targets.to(DEV), lengths.to(DEV), loss_clip=loss_clip, reduction=reduction)
    xd = x.double().requires_grad_()
    ref = X.ctc_loss(xd, targets, lengths, state_len, loss_clip=loss_clip, reduction=reduction)
    per = seqdist.ctc_loss(x.to(DEV), targets.to(DEV), lengths.to(DEV), loss_clip=loss_clip, reduction="none").cpu()
    per_ref = X.ctc_loss(x.double(), targets, lengths, state_len, loss_clip=loss_clip, reduction="none")
    fin = torch.isfinite(per_ref)
    rel = float(((per.double() - per_ref)[fin] / per_ref[fin].abs()).abs().max())
    if loss_clip:
        assert torch.isfinite(per).all() and torch.all(per[bad] == loss_clip)
    else:
        assert torch.isinf(per[bad]).all() and (per[bad] > 0).all()
    assert torch.equal(fin, torch.isfinite(per))

    # 'none': the sum of the finite per-chunk losses
    (loss if reduction == "mean" else loss[fin.to(DEV)].sum()).backward()
    (ref if reduction == "mean" else ref[fin].sum()).backward()
    grad = xg.grad.cpu()
    gerr = float((grad.double() - xd.grad).abs().max())
    print(f"k={state_len} {reduction} clip={loss_clip}: per-chunk loss rel {rel:.2e}; grad max|d| {gerr:.2e} "
          f"(max |grad| {float(xd.grad.abs().max()):.2e})")
    assert rel <= 1e-5
    assert not torch.isnan(grad).any()
    assert torch.all(grad[:, bad] == 0)
    assert gerr <= 1e-4


def test_infeasible_gradient_is_zero_even_for_an_infinite_loss():
    """Without loss_clip the mean loss is inf; the gradient of the feasible chunks is still finite and the infeasible ones
    get exactly 0."""
    state_len, T, N = 3, 60, 5
    x = _scores(T, N, state_len, seed=5)
    targets, lengths = _targets(N, T, state_len, seed=9)
    bad = _infeasible(lengths, state_len, T)
    xg = x.to(DEV).requires_grad_()
    loss = CTC_CRF(state_len, "NACGT").ctc_loss(xg, targets.to(DEV), lengths.to(DEV))
    loss.backward()
    assert torch.isinf(loss)
    grad = xg.grad.cpu()
    assert torch.isfinite(grad).all() and torch.all(grad[:, bad] == 0) and grad[:, ~bad].abs().sum() > 0


def test_seqdist_model_loss_applies_target_projection():
    state_len, T, N = 3, 80, 4
    seqdist = CTC_CRF(state_len, "NACGT")
    projection = [2, 1, 4, 3]
    model = SeqdistModel(torch.nn.Identity(), seqdist, target_projection=projection).to(DEV)
    x = _scores(T, N, state_len, seed=21)
    targets, lengths = _targets(N, T, state_len, seed=22)
    xg = x.half().to(DEV).requires_grad_()                       # fp16 scores are upcast to fp32
    loss = model.loss(xg, targets.to(DEV), lengths.to(DEV), loss_clip=10.0)
    loss.backward()
    projected = torch.tensor([0] + projection)[targets]
    xd = x.half().double().requires_grad_()
    ref = X.ctc_loss(xd, projected, lengths, state_len, loss_clip=10.0)
    ref.backward()
    gerr = float((xg.grad.double().cpu() - xd.grad).abs().max())
    print(f"model.loss: |d| {abs(float(loss) - float(ref)):.2e}; grad max|d| {gerr:.2e}")
    assert abs(float(loss) - float(ref)) <= 1e-5 * abs(float(ref))
    assert gerr <= 1e-4


@pytest.mark.parametrize("quantise", [False, True])
@pytest.mark.parametrize("state_len", [1, 3, 5])
def test_ctc_viterbi_alignments_equal_oracle(state_len, quantise):
    T, N = 150, 6
    x = _scores(T, N, state_len, seed=31 + state_len, quantise=quantise)
    targets, lengths = _targets(N, T, state_len, seed=32)
    got = CTC_CRF(state_len, "NACGT").ctc_viterbi_alignments(x.to(DEV), targets.to(DEV), lengths.to(DEV)).cpu()
    ref = X.ctc_viterbi_alignments(x.double(), targets, lengths, state_len).float()
    print(f"k={state_len} quantised={quantise}: {(got != ref).sum().item()} differing entries")
    assert torch.equal(got, ref)
    bad = _infeasible(lengths, state_len, T)
    assert torch.all(got[:, bad] == 0) and torch.all(got[:, ~bad].sum(-1) == 1)


def test_target_lattice_max_semiring_gradient():
    T, N, L = 90, 5, 40
    g = torch.Generator().manual_seed(41)
    stay, move = torch.randn(T, N, L, generator=g), torch.randn(T, N, L - 1, generator=g)
    lengths = torch.tensor([40, 1, 0, 92, 25], dtype=torch.int32)
    s, m = stay.to(DEV).requires_grad_(), move.to(DEV).requires_grad_()
    logz = target_logz(s, m, lengths.to(DEV), Max)
    logz.sum().backward()
    ref_stay, ref_move = X.target_max_onehot(stay.double(), move.double(), lengths)
    ref_lz = X.target_logz(stay.double(), move.double(), lengths, "max")
    assert torch.equal(s.grad.cpu(), ref_stay.float()) and torch.equal(m.grad.cpu(), ref_move.float())
    assert _logz_err(logz[torch.isfinite(ref_lz)], ref_lz[torch.isfinite(ref_lz)]) <= 1.0
    assert torch.equal(torch.isinf(logz.cpu()), torch.isinf(ref_lz))


def test_bitwise_repeatable():
    state_len, T, N = 4, 300, 9
    x = _scores(T, N, state_len, seed=51).to(DEV)
    seqdist = CTC_CRF(state_len, "NACGT")
    targets, lengths = _targets(N, T, state_len, seed=52)
    stay, move = seqdist.prepare_ctc_scores(seqdist.normalise(x), targets.to(DEV))
    lt = (lengths + 1 - state_len).to(DEV)

    def run():
        out = [seqdist.logZ(x), seqdist.logZ(x, Max), seqdist.forward_scores(x), seqdist.backward_scores(x),
               seqdist.posteriors(x), seqdist.posteriors(x, Max)]
        s, m = stay.detach().requires_grad_(), move.detach().requires_grad_()
        lz = target_logz(s, m, lt)
        lz.sum().backward()
        return out + [lz.detach(), s.grad, m.grad, *target_viterbi(stay, move, lt)]

    a, b = run(), run()
    assert all(torch.equal(u, v) for u, v in zip(a, b))


def test_logz_beyond_2_31_score_elements():
    """One forward logZ over more than 2^31 fp32 scores (8.6 GB): the last chunk equals, bitwise, the same chunk alone."""
    state_len, T, N = 5, 2000, 210
    assert T * N * 5 * 4 ** state_len > 2 ** 31
    seqdist = CTC_CRF(state_len, "NACGT")
    g = torch.Generator(device=DEV).manual_seed(61)
    x = torch.randn(T, N, 5 * 4 ** state_len, device=DEV, generator=g)
    with torch.no_grad():
        logz = seqdist.logZ(x)
        last = x[:, -1:].contiguous()
        alone = seqdist.logZ(last)
        first = seqdist.logZ(x[:, :1].contiguous())
    del x
    print(f"logZ last chunk {float(logz[-1]):.6f} alone {float(alone[0]):.6f}")
    assert torch.isfinite(logz).all()
    assert torch.equal(logz[-1:], alone) and torch.equal(logz[:1], first)


def test_target_max_logz_without_gradient():
    """The Max-semiring target forward with no workspace (inputs that need no gradient) equals the oracle."""
    T, N, L = 90, 5, 40
    g = torch.Generator().manual_seed(43)
    stay, move = torch.randn(T, N, L, generator=g), torch.randn(T, N, L - 1, generator=g)
    lengths = torch.tensor([40, 1, 0, 92, 25], dtype=torch.int32)
    with torch.no_grad():
        logz = target_logz(stay.to(DEV), move.to(DEV), lengths.to(DEV), Max).cpu()
    ref = X.target_logz(stay.double(), move.double(), lengths, "max")
    fin = torch.isfinite(ref)
    assert torch.equal(torch.isfinite(logz), fin) and torch.all(logz[~fin] == float("-inf"))
    assert _logz_err(logz[fin], ref[fin]) <= 1.0


@pytest.mark.parametrize("T,bases", [(1400, (1100, 1300)), (2800, (2300, 2700))])
def test_long_targets(T, bases):
    """Targets of more than 1024 (two states per thread) and more than 2048 k-mers (four states per thread): loss value and
    gradient, the Max logZ without a workspace, and the Viterbi alignment."""
    state_len, N = 2, 3
    x = _scores(T, N, state_len, seed=T)
    g = torch.Generator().manual_seed(T + 1)
    lengths = torch.randint(bases[0], bases[1], (N,), generator=g)
    targets = torch.zeros(N, bases[1], dtype=torch.long)
    for n in range(N):
        targets[n, :lengths[n]] = torch.randint(1, 5, (int(lengths[n]),), generator=g)
    L = targets.shape[1] - state_len + 1
    assert L > (2048 if T > 2000 else 1024)
    seqdist = CTC_CRF(state_len, "NACGT")

    xg = x.to(DEV).requires_grad_()
    per = seqdist.ctc_loss(xg, targets.to(DEV), lengths.to(DEV), reduction="none")
    per.sum().backward()
    xd = x.double().requires_grad_()
    per_ref = X.ctc_loss(xd, targets, lengths, state_len, reduction="none")
    per_ref.sum().backward()
    rel = float(((per.detach().double().cpu() - per_ref.detach()) / per_ref.detach().abs()).abs().max())
    gerr = float((xg.grad.double().cpu() - xd.grad).abs().max())

    stay, move = X.prepare_ctc_scores(x.double(), targets, state_len)
    lt = lengths + 1 - state_len
    with torch.no_grad():
        lz_max = target_logz(stay.float().to(DEV), move.float().to(DEV), lt.to(DEV), Max).cpu()
    max_err = _logz_err(lz_max, X.target_logz(stay, move, lt, "max"))
    align = seqdist.ctc_viterbi_alignments(x.to(DEV), targets.to(DEV), lengths.to(DEV)).cpu()
    ref_align = X.ctc_viterbi_alignments(x.double(), targets, lengths, state_len).float()
    print(f"T={T} L={L}: per-chunk loss rel {rel:.2e}; grad max|d| {gerr:.2e}; Max logZ relative to bound {max_err:.3f}; "
          f"{(align != ref_align).sum().item()} differing alignment entries")
    assert rel <= 1e-5 and gerr <= 1e-4 and max_err <= 1.0
    assert torch.equal(align, ref_align)


@pytest.mark.parametrize("S", ["Log", "Max"])
def test_second_backward_with_retained_graph(S):
    """backward(retain_graph=True) then backward() again gives the same gradients, bitwise, for both lattices: the
    workspace lives as long as the graph."""
    from bonito_b200.crf.model import Log
    semiring = Log if S == "Log" else Max
    state_len, T, N = 3, 50, 4
    seqdist = CTC_CRF(state_len, "NACGT")
    x = _scores(T, N, state_len, seed=71).to(DEV)
    targets, lengths = _targets(N, T, state_len, seed=72)
    stay, move = seqdist.prepare_ctc_scores(x, targets.to(DEV))
    x, stay, move = (t.detach().requires_grad_() for t in (x, stay, move))
    tz = target_logz(stay, move, (lengths + 1 - state_len).to(DEV), semiring)
    out = seqdist.logZ(x, semiring).sum() + tz[torch.isfinite(tz)].sum()
    out.backward(retain_graph=True)
    first = [t.grad.clone() for t in (x, stay, move)]
    for t in (x, stay, move):
        t.grad = None
    out.backward()
    assert all(torch.equal(a, t.grad) for a, t in zip(first, (x, stay, move)))
