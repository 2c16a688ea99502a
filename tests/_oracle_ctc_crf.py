"""
Float64 CPU restatement of the two CTC-CRF lattices (test infrastructure; the GPU kernels are checked against it).

  * the k-mer lattice of CTC_CRF (graph from `oracle.crf_oracle.crf_idx`): alpha, beta, logZ in the Log / Max semiring,
    posteriors by autograd, the Max path by back-pointers (ties: lowest in-edge, then lowest final state);
  * the target lattice of ctc_loss: logZ by autograd-friendly recursion, the Max path by back-pointers (ties: the stay);
  * ctc_loss composed from them the way bonito/crf/model.py:110-143 writes it.

Scores are torch float64 tensors in the reference layout [T, N, 5 * 4**state_len].
"""
import numpy as np
import torch

from oracle import crf_oracle

NEG = -1e300          # stands in for -inf inside the target recursion, so that autograd never sees inf - inf


def graph(state_len):
    idx = torch.as_tensor(crf_oracle.crf_idx(state_len))
    S, E = idx.shape
    succ = [[] for _ in range(S)]
    for s in range(S):
        for e in range(E):
            succ[int(idx[s, e])].append((s, e))
    succ = torch.as_tensor(succ)                                  # [S, 5, (s, e)]
    return idx, succ[..., 0], succ[..., 1]


def _red(x, semiring):
    return torch.logsumexp(x, -1) if semiring == "log" else x.amax(-1)


def sparse_alpha(scores, state_len, semiring="log"):
    T, N, _ = scores.shape
    idx, _, _ = graph(state_len)
    Ms = scores.reshape(T, N, -1, 5).unbind(0)       # one unbind: indexing frame by frame costs O(T^2) in backward
    a = scores.new_zeros(N, idx.shape[0])
    rows = [a]
    for t in range(T):
        a = _red(Ms[t] + a[:, idx], semiring)
        rows.append(a)
    return torch.stack(rows)


def sparse_beta(scores, state_len, semiring="log"):
    T, N, _ = scores.shape
    idx, succ_s, succ_e = graph(state_len)
    Ms = scores.reshape(T, N, -1, 5)
    b = scores.new_zeros(N, idx.shape[0])
    rows = [b]
    for t in range(T - 1, -1, -1):
        b = _red(Ms[t][:, succ_s, succ_e] + b[:, succ_s], semiring)
        rows.append(b)
    return torch.stack(rows[::-1])


def sparse_logz(scores, state_len, semiring="log"):
    return _red(sparse_alpha(scores, state_len, semiring)[-1], semiring)


def sparse_posteriors(scores, state_len):
    x = scores.detach().clone().requires_grad_()
    grad, = torch.autograd.grad(sparse_logz(x, state_len).sum(), x)
    return grad


def sparse_max_path(scores, state_len):
    """(state [T, N], edge [T, N]) of the best path: first maximum over in-edges, first maximum over final states."""
    T, N, _ = scores.shape
    idx, _, _ = graph(state_len)
    Ms = scores.reshape(T, N, -1, 5)
    v = scores.new_zeros(N, idx.shape[0])
    bps = []
    for t in range(T):
        cand = Ms[t] + v[:, idx]
        bp = cand.argmax(-1)                                      # first maximum
        v = cand.gather(-1, bp[..., None])[..., 0]
        bps.append(bp)
    s = v.argmax(-1)
    states = torch.empty(T, N, dtype=torch.long)
    edges = torch.empty(T, N, dtype=torch.long)
    for t in range(T - 1, -1, -1):
        e = bps[t].gather(1, s[:, None])[:, 0]
        states[t], edges[t] = s, e
        s = idx[s, e]
    return states, edges


def sparse_max_onehot(scores, state_len):
    """d logZ_Max / d scores: 1 on the best path's edges."""
    states, edges = sparse_max_path(scores, state_len)
    out = torch.zeros_like(scores)
    out.scatter_(2, (states * 5 + edges)[..., None], 1.0)
    return out


def viterbi(scores, state_len):
    """CTC_CRF.viterbi: [T, N], 0 on a stay, else 1 + the emitted base."""
    states, edges = sparse_max_path(scores, state_len)
    return torch.where(edges != 0, 1 + states % 4, 0)


def feasible(lengths, T, L):
    lengths = torch.as_tensor(lengths)
    return (lengths >= 1) & (lengths <= L) & (lengths - 1 <= T)


def target_logz(stay, move, lengths, semiring="log"):
    """logZ [N] of the target lattice (differentiable in the Log semiring); -inf for infeasible chunks."""
    T, N, L = stay.shape
    lengths = torch.as_tensor(lengths).long()
    a = torch.full((N, L), NEG, dtype=stay.dtype)
    a = torch.cat([stay.new_zeros(N, 1), a[:, 1:]], 1)
    neg = torch.full((N, 1), NEG, dtype=stay.dtype)
    stay, move = stay.unbind(0), move.unbind(0)        # one unbind: indexing frame by frame costs O(T^2) in backward
    for t in range(T):
        s = a + stay[t]
        m = torch.cat([neg, a[:, :-1] + move[t]], 1)
        a = torch.logaddexp(s, m) if semiring == "log" else torch.maximum(s, m)
    ok = feasible(lengths, T, L)
    lz = a.gather(1, (lengths - 1).clamp(0, L - 1)[:, None])[:, 0]
    return torch.where(ok, lz, torch.full_like(lz, -np.inf))


def target_max_onehot(stay, move, lengths):
    """(dstay, dmove) one-hot on the best path of the target lattice (ties: the stay); zeros for infeasible chunks."""
    T, N, L = stay.shape
    lengths = torch.as_tensor(lengths).long()
    a = torch.full((N, L), -np.inf, dtype=torch.float64)
    a[:, 0] = 0
    bps = []
    for t in range(T):
        s = a + stay[t]
        m = torch.cat([torch.full((N, 1), -np.inf, dtype=torch.float64), a[:, :-1] + move[t]], 1)
        bps.append(m > s)
        a = torch.where(m > s, m, s)
    dstay, dmove = torch.zeros_like(stay), torch.zeros_like(move)
    ok = feasible(lengths, T, L)
    for n in range(N):
        if not ok[n]:
            continue
        j = int(lengths[n]) - 1
        for t in range(T - 1, -1, -1):
            if bps[t][n, j]:
                j -= 1
                dmove[t, n, j] = 1
            else:
                dstay[t, n, j] = 1
    return dstay, dmove


def prepare_ctc_scores(scores, targets, state_len):
    """Stay / move scores of the k-mers along each target row, built index by index."""
    T, N, _ = scores.shape
    tg = (torch.as_tensor(targets).long() - 1).clamp(min=0)
    L = tg.shape[1] - (state_len - 1)
    stay = torch.empty(T, N, L, dtype=scores.dtype)
    move = torch.empty(T, N, L - 1, dtype=scores.dtype)
    stay_cols = torch.empty(N, L, dtype=torch.long)
    move_cols = torch.empty(N, max(L - 1, 0), dtype=torch.long)
    for n in range(N):
        for j in range(L):
            kmer = 0
            for i in range(state_len):
                kmer = kmer * 4 + int(tg[n, j + i])
            stay_cols[n, j] = kmer * 5
            if j >= 1:
                move_cols[n, j - 1] = kmer * 5 + 1 + int(tg[n, j - 1])
    stay = scores.gather(2, stay_cols.expand(T, -1, -1))
    move = scores.gather(2, move_cols.expand(T, -1, -1))
    return stay, move


def normalise(scores, state_len):
    return scores - sparse_logz(scores, state_len)[:, None] / len(scores)


def ctc_loss(scores, targets, target_lengths, state_len, loss_clip=None, reduction="mean", normalise_scores=True):
    target_lengths = torch.as_tensor(target_lengths)
    if normalise_scores:
        scores = normalise(scores, state_len)
    stay, move = prepare_ctc_scores(scores, targets, state_len)
    logz = target_logz(stay, move, target_lengths + 1 - state_len)
    loss = -(logz / target_lengths)
    if loss_clip:
        loss = torch.clamp(loss, 0.0, loss_clip)
    return loss.mean() if reduction == "mean" else loss


def ctc_viterbi_alignments(scores, targets, target_lengths, state_len):
    stay, move = prepare_ctc_scores(scores, targets, state_len)
    dstay, dmove = target_max_onehot(stay, move, torch.as_tensor(target_lengths) + 1 - state_len)
    return dstay + torch.nn.functional.pad(dmove, (0, 1))
