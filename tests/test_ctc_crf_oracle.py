"""The float64 CTC-CRF oracle (tests/_oracle_ctc_crf.py) against path enumeration, the crf_oracle restatement and finite
differences, and the CPU-side contract of the CTC_CRF scoring API (no GPU needed)."""
import itertools

import numpy as np
import pytest
import torch

import _oracle_ctc_crf as X
from bonito_b200 import native
from bonito_b200.crf.model import CTC_CRF, Log, Max, SeqdistModel
from oracle import crf_oracle as O


def _paths_sparse(state_len, T):
    """Every path of the k-mer lattice as (start state, [(state, edge)] * T)."""
    idx = O.crf_idx(state_len)
    S = idx.shape[0]
    out_edges = [[(s, e) for s in range(S) for e in range(5) if idx[s, e] == p] for p in range(S)]

    def walk(p, t):
        if t == T:
            yield []
            return
        for s, e in out_edges[p]:
            for rest in walk(s, t + 1):
                yield [(s, e)] + rest
    for p in range(S):
        for path in walk(p, 0):
            yield path


@pytest.mark.parametrize("state_len,T", [(1, 1), (1, 3), (2, 2)])
def test_sparse_lattice_equals_path_enumeration(state_len, T):
    torch.manual_seed(0)
    N = 2
    scores = torch.randn(T, N, 5 * 4 ** state_len, dtype=torch.float64)
    paths = list(_paths_sparse(state_len, T))
    assert len(paths) == 4 ** state_len * 5 ** T
    cols = torch.tensor([[s * 5 + e for s, e in p] for p in paths])            # [P, T]
    tot = scores[torch.arange(T), :, cols].sum(1)                               # [P, N]
    logz_log, logz_max = torch.logsumexp(tot, 0), tot.amax(0)
    torch.testing.assert_close(X.sparse_logz(scores, state_len, "log"), logz_log, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(X.sparse_logz(scores, state_len, "max"), logz_max, rtol=1e-12, atol=1e-12)
    # posteriors: the probability mass of the paths through each edge
    w = torch.softmax(tot, 0)
    post = torch.zeros_like(scores)
    for p in range(len(paths)):
        for t in range(T):
            post[t, :, cols[p, t]] += w[p]
    torch.testing.assert_close(X.sparse_posteriors(scores, state_len), post, rtol=1e-10, atol=1e-12)
    # the Max one-hot marks the best path (continuous scores: no ties)
    best = tot.argmax(0)
    onehot = torch.zeros_like(scores)
    for n in range(N):
        for t in range(T):
            onehot[t, n, cols[best[n], t]] = 1
    assert torch.equal(X.sparse_max_onehot(scores, state_len), onehot)
    # alpha_T and beta_0 both give logZ
    torch.testing.assert_close(torch.logsumexp(X.sparse_beta(scores, state_len)[0], -1), logz_log, rtol=1e-12, atol=1e-12)


def test_target_lattice_equals_path_enumeration():
    torch.manual_seed(1)
    T, N, L = 6, 6, 4
    stay = torch.randn(T, N, L, dtype=torch.float64)
    move = torch.randn(T, N, L - 1, dtype=torch.float64)
    lengths = torch.tensor([1, 2, 4, 3, 0, 8])                                  # 0: no state; 8 > L: infeasible
    lz = X.target_logz(stay, move, lengths)
    lz_max = X.target_logz(stay, move, lengths, "max")
    dstay, dmove = X.target_max_onehot(stay, move, lengths)
    for n in range(N):
        ln = int(lengths[n])
        tots, routes = [], []
        for steps in itertools.product((0, 1), repeat=T):                     # 1 = move
            if not (1 <= ln <= L) or sum(steps) != ln - 1:
                continue
            j, sc = 0, 0.0
            for t, m in enumerate(steps):
                sc += float(move[t, n, j]) if m else float(stay[t, n, j])
                j += m
            tots.append(sc)
            routes.append(steps)
        if not tots:
            assert lz[n] == -np.inf and lz_max[n] == -np.inf
            assert not dstay[:, n].any() and not dmove[:, n].any()
            continue
        assert abs(float(lz[n]) - float(np.logaddexp.reduce(tots))) < 1e-12
        assert abs(float(lz_max[n]) - max(tots)) < 1e-12
        steps = routes[int(np.argmax(tots))]
        j = 0
        for t, m in enumerate(steps):
            assert (dmove if m else dstay)[t, n, j] == 1
            j += m
        assert dstay[:, n].sum() + dmove[:, n].sum() == T


def test_target_max_ties_go_to_the_stay():
    T, N, L = 4, 1, 3
    stay = torch.zeros(T, N, L, dtype=torch.float64)
    move = torch.zeros(T, N, L - 1, dtype=torch.float64)
    dstay, dmove = X.target_max_onehot(stay, move, torch.tensor([2]))
    # every alignment scores 0; traced back from the end every tie takes the stay, so the one move is the first frame
    assert dmove[0, 0, 0] == 1 and dstay[1:, 0, 1].tolist() == [1, 1, 1]
    assert dstay.sum() + dmove.sum() == T


@pytest.mark.parametrize("state_len", [1, 2, 3])
def test_log_semiring_equals_crf_oracle(state_len):
    torch.manual_seed(2)
    scores = torch.randn(9, 3, 5 * 4 ** state_len, dtype=torch.float64)
    Ms = scores.numpy().reshape(9, 3, -1, 5)
    idx = O.crf_idx(state_len)
    np.testing.assert_allclose(X.sparse_logz(scores, state_len).numpy(), O.logZ(Ms, idx), rtol=1e-12)
    np.testing.assert_allclose(X.sparse_logz(scores, state_len, "max").numpy(), O.logZ(Ms, idx, "max"), rtol=1e-12)
    np.testing.assert_allclose(X.sparse_posteriors(scores, state_len).numpy().reshape(Ms.shape), O.posteriors(Ms, idx),
                               rtol=1e-9, atol=1e-14)
    alpha, beta = O.fwd_bwd(Ms, idx)
    np.testing.assert_allclose(X.sparse_alpha(scores, state_len).numpy(), alpha, rtol=1e-12)
    np.testing.assert_allclose(X.sparse_beta(scores, state_len).numpy(), beta, rtol=1e-12)


@pytest.mark.parametrize("quantised", [False, True])
@pytest.mark.parametrize("state_len", [1, 2, 3])
def test_max_path_equals_crf_oracle_viterbi(state_len, quantised):
    torch.manual_seed(3)
    scores = torch.randn(12, 4, 5 * 4 ** state_len, dtype=torch.float64)
    if quantised:
        scores = torch.round(scores * 2) / 2                                   # many ties
    states, edges = X.sparse_max_path(scores, state_len)
    o_states, o_edges = O.viterbi_edges(scores.numpy().reshape(12, 4, -1, 5), O.crf_idx(state_len))
    assert np.array_equal(states.numpy(), o_states) and np.array_equal(edges.numpy(), o_edges)


def _loss_inputs(seed=4, state_len=2, T=7, N=4):
    g = torch.Generator().manual_seed(seed)
    scores = torch.randn(T, N, 5 * 4 ** state_len, dtype=torch.float64, generator=g)
    lengths = torch.tensor([5, 3, 4, 2])[:N]
    targets = torch.zeros(N, 5, dtype=torch.long)
    for n in range(N):
        targets[n, :lengths[n]] = torch.randint(1, 5, (int(lengths[n]),), generator=g)
    return scores, targets, lengths


@pytest.mark.parametrize("normalise_scores", [True, False])
def test_loss_gradient_matches_central_differences(normalise_scores):
    scores, targets, lengths = _loss_inputs()
    x = scores.clone().requires_grad_()
    loss = X.ctc_loss(x, targets, lengths, 2, normalise_scores=normalise_scores)
    grad, = torch.autograd.grad(loss, x)
    h = 1e-6
    flat = scores.reshape(-1)
    rng = np.random.default_rng(0)
    for i in rng.choice(flat.numel(), 60, replace=False):
        up, dn = flat.clone(), flat.clone()
        up[i] += h
        dn[i] -= h
        fd = (X.ctc_loss(up.view_as(scores), targets, lengths, 2, normalise_scores=normalise_scores)
              - X.ctc_loss(dn.view_as(scores), targets, lengths, 2, normalise_scores=normalise_scores)) / (2 * h)
        assert abs(float(fd) - float(grad.reshape(-1)[i])) < 1e-7, i


def test_prepare_ctc_scores_matches_the_index_by_index_oracle():
    scores, targets, lengths = _loss_inputs(state_len=3, T=3)
    stay, move = CTC_CRF(3, "NACGT").prepare_ctc_scores(scores, targets)
    o_stay, o_move = X.prepare_ctc_scores(scores.float(), targets, 3)
    assert torch.equal(stay, o_stay) and torch.equal(move, o_move)


def test_api_contract_without_gpu():
    seqdist = CTC_CRF(2, "NACGT")
    assert Log is not Max
    with pytest.raises(ValueError, match="80"):
        seqdist.logZ(torch.zeros(4, 2, 81))
    with pytest.raises(ValueError, match="Unknown reduction"):
        seqdist.ctc_loss(torch.zeros(4, 2, 80), torch.ones(2, 3, dtype=torch.long), torch.tensor([3, 3]),
                         reduction="sum")
    if not torch.cuda.is_available():
        with pytest.raises(native.NativeError):
            seqdist.logZ(torch.zeros(4, 2, 80))
        with pytest.raises(native.NativeError):
            seqdist.posteriors(torch.zeros(4, 2, 80))
        with pytest.raises(native.NativeError):
            seqdist.ctc_loss(torch.zeros(4, 2, 80), torch.ones(2, 3, dtype=torch.long), torch.tensor([3, 3]))
    assert hasattr(SeqdistModel, "loss")


def test_native_wrappers_refuse_host_tensors():
    x = torch.zeros(3, 2, 80)
    with pytest.raises(native.NativeError):
        native.ctc_crf_sparse_fwd(x, 2, native.SEMIRING_LOG, torch.zeros(2))
    with pytest.raises(native.NativeError):
        native.ctc_crf_target_fwd(torch.zeros(3, 2, 4), torch.zeros(3, 2, 3), torch.ones(2, dtype=torch.int32),
                                  native.SEMIRING_LOG, torch.zeros(2))
