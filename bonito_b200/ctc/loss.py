"""
The CTC loss of the QuartzNet CTC models as one autograd function over the sm_90a kernels of `csrc/ctc_loss.cu`.

`ctc_loss` has the contract of `torch.nn.functional.ctc_loss` (which the reference calls in
bonito/ctc/model.py:48-53), with these differences:
  * it is deterministic: the gradient sums in a fixed order, where torch's CUDA backward accumulates with atomics;
  * labels are checked: a label equal to `blank` or outside [0, C) raises `ValueError` (torch does not check them);
  * targets hold at most `native.ctc_loss_max_target()` labels and C is at most 256;
  * the loss is fp32 whatever the input's floating dtype (fp16 log-probs are upcast), and there is no CPU path: tensors
    off the GPU raise `NativeError`.
"""

import numpy as np
import torch

from bonito_b200 import native

MAX_CLASSES = 256  # B200_CTC_LOSS_MAX_CLASSES


class CtcLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, log_probs, targets, target_off, input_lengths, target_lengths, max_target, blank, zero_infinity):
        t, n, _ = log_probs.shape
        nll = log_probs.new_empty(n)
        workspace = None
        if ctx.needs_input_grad[0]:
            workspace = torch.empty(native.ctc_loss_workspace_bytes(n, t, max_target), dtype=torch.uint8,
                                    device=log_probs.device)
        native.ctc_loss_fwd(log_probs, input_lengths, targets, target_off, target_lengths, max_target, blank, nll,
                            workspace=workspace)
        ctx.max_target, ctx.blank, ctx.zero_infinity, ctx.workspace = max_target, blank, zero_infinity, workspace
        ctx.save_for_backward(log_probs, targets, target_off, input_lengths, target_lengths)
        return nll

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        log_probs, targets, target_off, input_lengths, target_lengths = ctx.saved_tensors
        grad = torch.empty(log_probs.shape, dtype=torch.float32, device=log_probs.device)
        native.ctc_loss_grad(log_probs, input_lengths, targets, target_off, target_lengths, ctx.max_target, ctx.blank,
                             g.float().contiguous(), ctx.zero_infinity, ctx.workspace, grad)
        return grad, None, None, None, None, None, None, None


def _lengths(x, n, name):
    x = torch.as_tensor(x).detach().cpu()
    if x.dtype.is_floating_point or x.dtype.is_complex or x.dtype == torch.bool:
        raise ValueError(f"{name} must hold integers, got {x.dtype}")
    if tuple(x.shape) != (n,):
        raise ValueError(f"{name} must have {n} entries (one per sample), got shape {tuple(x.shape)}")
    return x.to(torch.int64)


def ctc_loss(log_probs, targets, input_lengths, target_lengths, blank=0, reduction="mean", zero_infinity=False):
    """
    CTC loss of `log_probs` [T, N, C] (a CUDA tensor; fp16 is upcast to fp32; any strides) against `targets`, padded
    [N, S] or concatenated 1-D, with per-sample `input_lengths` (each in 1..T) and `target_lengths` (each in
    0..min(S, native.ctc_loss_max_target())).  `reduction`: 'mean' divides each sample's loss by its target length
    (at least 1) and averages over the batch, 'sum' adds the losses, 'none' returns them [N].  A sample that no alignment
    fits (input length < target length + adjacent repeats) has an infinite loss and a NaN gradient, or 0 for both with
    `zero_infinity`.  See the module docstring for how this differs from torch's.
    """
    if not isinstance(log_probs, torch.Tensor) or log_probs.dim() != 3:
        raise ValueError(f"log_probs must be a [T, N, C] tensor, got {getattr(log_probs, 'shape', type(log_probs))}")
    if not log_probs.is_cuda:
        raise native.NativeError("log_probs must be on a CUDA device (the CTC loss runs on the sm_90a kernels only)")
    if not log_probs.dtype.is_floating_point:
        raise ValueError(f"log_probs must be floating point, got {log_probs.dtype}")
    if reduction not in ("mean", "sum", "none"):
        raise ValueError(f"unknown reduction {reduction!r}: use 'mean', 'sum' or 'none'")
    T, N, C = log_probs.shape
    if T < 1 or not 1 <= C <= MAX_CLASSES:
        raise ValueError(f"log_probs must have T >= 1 frames and 1..{MAX_CLASSES} classes, got {tuple(log_probs.shape)}")
    if not isinstance(blank, int) or not 0 <= blank < C:
        raise ValueError(f"blank must be an integer in [0, {C}), got {blank!r}")
    il = _lengths(input_lengths, N, "input_lengths")
    tl = _lengths(target_lengths, N, "target_lengths")
    if N and (int(il.min()) < 1 or int(il.max()) > T):
        raise ValueError(f"input_lengths must be in 1..{T}")
    if N and int(tl.min()) < 0:
        raise ValueError("target_lengths must not be negative")
    max_target = int(tl.max()) if N else 0
    if max_target > native.ctc_loss_max_target():
        raise ValueError(f"a target of {max_target} labels is longer than the {native.ctc_loss_max_target()} supported")

    if not isinstance(targets, torch.Tensor) or targets.dtype.is_floating_point or targets.dtype == torch.bool:
        raise ValueError("targets must be an integer tensor")
    dev = log_probs.device
    if targets.dim() == 2:
        if targets.shape[0] != N or targets.shape[1] < max_target:
            raise ValueError(f"padded targets must be [N = {N}, S >= {max_target}], got {tuple(targets.shape)}")
        off = np.arange(N, dtype=np.int64) * targets.shape[1]
        valid = torch.arange(targets.shape[1])[None, :] < tl[:, None]
    elif targets.dim() == 1:
        total = int(tl.sum())
        if targets.shape[0] < total:
            raise ValueError(f"concatenated targets hold {targets.shape[0]} labels, the target lengths add up to {total}")
        off = np.concatenate([[0], np.cumsum(tl.numpy())[:-1]]).astype(np.int64) if N else np.zeros(0, np.int64)
        valid = torch.arange(targets.shape[0]) < total
    else:
        raise ValueError(f"targets must be padded [N, S] or concatenated 1-D, got {tuple(targets.shape)}")
    targets = targets.to(device=dev, dtype=torch.int64)
    bad = ((targets < 0) | (targets >= C) | (targets == blank)) & valid.to(dev)
    if bool(bad.any()):
        raise ValueError(f"targets hold a label equal to blank ({blank}) or outside [0, {C})")

    lp = log_probs.float()
    if lp.stride(2) != 1 and C != 1:
        lp = lp.contiguous()
    nll = CtcLoss.apply(lp, targets.to(torch.int32).contiguous(), torch.from_numpy(off).to(dev),
                        il.to(device=dev, dtype=torch.int32), tl.to(device=dev, dtype=torch.int32), max_target, blank,
                        bool(zero_infinity))
    if zero_infinity:
        nll = torch.where(nll == float("inf"), torch.zeros_like(nll), nll)
    if reduction == "none":
        return nll
    if reduction == "sum":
        return nll.sum()
    return (nll / tl.to(dev).clamp_min(1)).mean()
