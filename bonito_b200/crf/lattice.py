"""
The two lattices of the CTC-CRF sequence distribution as autograd functions over the sm_90a kernels of
`csrc/ctc_crf.cu` (the parts of koi.ctc that bonito/crf/model.py:30-143 calls).

  * `sparse_logz(scores, state_len, S)`: logZ of the k-mer lattice, scores [T, N, 5 * 4**state_len] fp32;
  * `target_logz(stay, move, lengths, S)`: logZ of the target-constrained lattice of ctc_loss.

`S` is one of the semiring markers `Log` (logsumexp) and `Max`.  The gradient of a Max logZ is the one-hot of its best path
(ties: the lowest in-edge at every frame then the lowest final state; in the target lattice the stay).  Nothing here falls
back to the CPU: tensors off the GPU raise `NativeError`.
"""

import torch

from bonito_b200 import native


class Semiring:
    """Marker of a semiring; `one` is its multiplicative unit (the boundary value alpha_0 = beta_T)."""

    def __init__(self, name, code):
        self.name, self.code, self.one = name, code, 0.0

    def __repr__(self):
        return self.name


Log = Semiring("Log", native.SEMIRING_LOG)
Max = Semiring("Max", native.SEMIRING_MAX)


def _code(S):
    if S is Log or S is Max:
        return S.code
    raise ValueError(f"unknown semiring {S!r}: use Log or Max")


class SparseLogZ(torch.autograd.Function):
    @staticmethod
    def forward(ctx, scores, state_len, code):
        t, n, _ = scores.shape
        logz = scores.new_empty(n)
        workspace = None
        if ctx.needs_input_grad[0]:
            workspace = torch.empty(native.ctc_crf_sparse_workspace_bytes(n, t, state_len, code), dtype=torch.uint8,
                                    device=scores.device)
        native.ctc_crf_sparse_fwd(scores, state_len, code, logz, workspace=workspace)
        ctx.state_len, ctx.code, ctx.workspace = state_len, code, workspace
        ctx.save_for_backward(scores)
        return logz

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        scores, = ctx.saved_tensors
        grad = torch.empty_like(scores)
        native.ctc_crf_sparse_grad(scores, ctx.state_len, ctx.code, g.float().contiguous(), ctx.workspace, grad)
        return grad, None, None


class TargetLogZ(torch.autograd.Function):
    @staticmethod
    def forward(ctx, stay, move, lengths, code):
        t, n, l = stay.shape
        logz = stay.new_empty(n)
        workspace = None
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
            workspace = torch.empty(native.ctc_crf_target_workspace_bytes(n, t, l, code), dtype=torch.uint8,
                                    device=stay.device)
        native.ctc_crf_target_fwd(stay, move, lengths, code, logz, workspace=workspace)
        ctx.code, ctx.workspace = code, workspace
        ctx.save_for_backward(stay, move, lengths)
        return logz

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        stay, move, lengths = ctx.saved_tensors
        dstay, dmove = torch.empty_like(stay), torch.empty_like(move)
        native.ctc_crf_target_grad(stay, move, lengths, ctx.code, g.float().contiguous(), ctx.workspace, dstay, dmove)
        return dstay, dmove, None, None


def _cuda_f32(x, name):
    if not x.is_cuda:
        raise native.NativeError(f"{name} must be on a CUDA device (the CTC-CRF lattices run on the sm_90a kernels only)")
    return x.float().contiguous()


def sparse_scores(scores, state_len):
    """Reference-layout scores [T, N, 5 * 4**state_len] as the kernels take them: CUDA, fp32, contiguous."""
    if scores.dim() != 3 or scores.shape[2] != 5 * 4 ** state_len:
        raise ValueError(f"scores must be [T, N, {5 * 4 ** state_len}] (n_score() for state_len {state_len}), "
                         f"got {tuple(scores.shape)}")
    if scores.shape[0] < 1:
        raise ValueError("scores must hold at least one frame")
    scores = _cuda_f32(scores, "scores")
    if scores.data_ptr() % 16:
        scores = scores.clone()
    return scores


def sparse_logz(scores, state_len, S=Log):
    return SparseLogZ.apply(sparse_scores(scores, state_len), state_len, _code(S))


def sparse_forward_scores(scores, state_len, S=Log):
    scores = sparse_scores(scores, state_len)
    t, n, _ = scores.shape
    alpha = scores.new_empty(t + 1, n, 4 ** state_len)
    native.ctc_crf_sparse_fwd(scores, state_len, _code(S), scores.new_empty(n), alpha=alpha)
    return alpha


def sparse_backward_scores(scores, state_len, S=Log):
    scores = sparse_scores(scores, state_len)
    t, n, _ = scores.shape
    beta = scores.new_empty(t + 1, n, 4 ** state_len)
    native.ctc_crf_sparse_bwd(scores, state_len, _code(S), beta)
    return beta


def _target_args(stay, move, lengths):
    stay, move = _cuda_f32(stay, "stay"), _cuda_f32(move, "move")
    if stay.dim() != 3 or stay.shape[0] < 1 or stay.shape[2] < 1:
        raise ValueError(f"stay scores must be [T >= 1, N, L >= 1], got {tuple(stay.shape)}")
    t, n, l = stay.shape
    if tuple(move.shape) != (t, n, l - 1):
        raise ValueError(f"move scores must be {(t, n, l - 1)}, got {tuple(move.shape)}")
    if l > native.ctc_crf_target_max_states():
        raise ValueError(f"targets of {l} states are longer than the {native.ctc_crf_target_max_states()} supported")
    lengths = torch.as_tensor(lengths).to(device=stay.device, dtype=torch.int32).contiguous()
    if lengths.shape != (n,):
        raise ValueError(f"lengths must have {n} entries, got shape {tuple(lengths.shape)}")
    return stay, move, lengths


def target_logz(stay, move, lengths, S=Log):
    """logZ [N] of the target lattice; -inf for an infeasible chunk (lengths < 1, lengths > L or lengths - 1 > T)."""
    stay, move, lengths = _target_args(stay, move, lengths)
    return TargetLogZ.apply(stay, move, lengths, _code(S))


def target_viterbi(stay, move, lengths):
    """The best path of the target lattice as its one-hot edges (dstay [T, N, L], dmove [T, N, L-1]); all zeros for an
    infeasible chunk."""
    stay, move, lengths = _target_args(stay, move, lengths)
    t, n, l = stay.shape
    workspace = torch.empty(native.ctc_crf_target_workspace_bytes(n, t, l, Max.code), dtype=torch.uint8,
                            device=stay.device)
    native.ctc_crf_target_fwd(stay, move, lengths, Max.code, stay.new_empty(n), workspace=workspace)
    dstay, dmove = torch.empty_like(stay), torch.empty_like(move)
    native.ctc_crf_target_grad(stay, move, lengths, Max.code, stay.new_ones(n), workspace, dstay, dmove)
    return dstay, dmove
