"""
QuartzNet CTC model package (`package = "bonito.ctc"`: dna_r9.4.1@v1 and @v2).

`Model(config)` mirrors the reference's module tree (bonito/ctc/model.py: `Encoder`, `Block`, `TCSConv1d`, `Decoder`, with
the same attribute names and registration order), so a reference `weights_N.tar` loads through `match_names` unchanged,
BatchNorm running statistics included.  On the CPU without `use_koi` the module tree runs and returns `[T, N, 5]`
log-probs, as the reference's `forward` does.  With `use_koi` the native engine (`bonito_b200.engine_ctc.CtcPlan`) runs
it on the GPU and returns batch-first `[N, T, 5]` fp16 log-probs; there is no eager CUDA path.  The plan holds folded
copies of the weights and BatchNorm statistics: it remembers the `_version` of every parameter and buffer it folded and is
rebuilt when any of them changes (an optimizer step, a `load_state_dict`, a training forward's statistics update).

Training: in train mode with grad enabled, a CUDA input runs `bonito_b200.engine_ctc.CtcTrainPlan` through one autograd
node (`CtcTrainFunction`): batch-statistics BatchNorm, dropout, fp16 operands with fp32 accumulation, and fp32
`[N, T, 5]` log-probs that backpropagate into every parameter on native kernels.

Decoding: `greedy_step` / `greedy_collapse` (host, the default) and `beam_search`, the CTC prefix beam search on the GPU
(`b200_ctc_beam_search`; cut, merge, tie, move and quality rules in bonito_b200/csrc/ctc_beam.cu).  The reference decodes
with fast_ctc_decode's beam search of width 5 (bonito/ctc/model.py:39-46).  Deviations: the default here is the greedy
decode; the beam search returns qualities and emission frames, which the reference's has not, so `qscores=True` keeps the
beam search where the reference switches to its Viterbi decode; there is no CPU path for the beam search.

Loss: `loss` / `ctc_label_smoothing_loss` as in the reference, with the CTC loss on the GPU (`bonito_b200.ctc.loss`).
"""

import numpy as np
import torch
from torch.nn import BatchNorm1d, Conv1d, Dropout, Module, ModuleList, Sequential
from torch.nn.functional import log_softmax

from bonito_b200.nn import Permute, layers


class Model(Module):
    """QuartzNet-style CTC model (reference: bonito/ctc/model.py:15-60)."""

    def __init__(self, config):
        super().__init__()
        if "qscore" not in config:
            self.qbias, self.qscale = 0.0, 1.0
        else:
            self.qbias, self.qscale = config["qscore"]["bias"], config["qscore"]["scale"]
        self.config = config
        self.stride = config["block"][0]["stride"][0]
        self.alphabet = config["labels"]["labels"]
        self.features = config["block"][-1]["filters"]
        self.encoder = Encoder(config)
        self.decoder = Decoder(self.features, len(self.alphabet))
        self._native = None        # set by use_koi(): dict of basecaller settings
        self._plan = None          # built lazily, after the weights are loaded
        self._plan_state = None    # (data_ptr, _version) of every parameter and buffer when the plan was built
        self._train_plan = None

    def forward(self, x):
        """[N, 1, L] -> log-probs: [T, N, 5] from the module tree on the CPU, [N, T, 5] fp16 from the native engine, and
        [N, T, 5] fp32 from the native training path (train mode, grad enabled, CUDA input)."""
        if self._native is None:
            if x.is_cuda:
                raise RuntimeError("bonito_b200: CUDA model called without use_koi(); call model.use_koi(...) "
                                   "(load_model(..., use_koi=True)) or run the module tree on the CPU")
            return self.decoder(self.encoder(x))
        if self.training and torch.is_grad_enabled() and x.is_cuda:
            from bonito_b200 import native
            from bonito_b200.engine_ctc import CtcTrainFunction, CtcTrainPlan
            native.require()
            if self._train_plan is None:
                self._train_plan = CtcTrainPlan(self)
            seed = int(torch.randint(0, 2**62, (1,)).item())
            return CtcTrainFunction.apply(self._train_plan, seed, x, *self._train_plan.params)
        return self.native_plan(x.device if x.is_cuda else None).forward(x)

    def _state(self):
        return [(t.data_ptr(), t._version) for t in list(self.parameters()) + list(self.buffers())]

    def native_plan(self, device=None):
        from bonito_b200 import native
        from bonito_b200.engine_ctc import CtcPlan
        native.require()
        if device is None:
            device = next(self.parameters()).device
        if torch.device(device).type != "cuda":
            raise native.NativeError("the native path was requested (use_koi) but the model is not on a CUDA device")
        state = self._state()
        if self._plan is None or self._plan.device != torch.device(device) or self._plan_state != state:
            self._plan = CtcPlan(self, device, quantize=bool((self._native or {}).get("quantize")))
            self._plan_state = state
        return self._plan

    def invalidate_plan(self):
        self._plan = self._train_plan = None

    def _apply(self, fn, *args, **kwargs):
        self._plan = self._train_plan = None  # .half()/.to() change the tensors the plans were packed from / refer to
        return super()._apply(fn, *args, **kwargs)

    def apply(self, fn):
        self._plan = self._train_plan = None
        return super().apply(fn)

    def load_state_dict(self, *args, **kwargs):
        self._plan = None  # the plan holds folded copies of the weights
        return super().load_state_dict(*args, **kwargs)

    def use_koi(self, **kwargs):
        """Arm the native engine (the hook `_load_model` calls)."""
        self._native = dict(kwargs)
        self._plan = self._train_plan = None

    def decode(self, x, beamsize=1, threshold=1e-3, qscores=False, return_path=False):
        """
        Decode one `[T, 5]` log-prob tensor: greedily on the host with `beamsize=1` (see `greedy_collapse`), with the prefix
        beam search on the GPU with `beamsize` in 2..32 (`beam_search`; x must be a CUDA tensor, `threshold` is its
        probability cut).  Returns the sequence, with the quality string appended when `qscores` (the layout of the
        reference's viterbi_search), and the emission frames when `return_path`.  `qscores` does not change the sequence:
        the beam search has qualities of its own (the reference's has none and falls back to Viterbi).
        """
        check_beamsize(beamsize)
        if beamsize > 1:
            check_alphabet(self.alphabet)
            seq, qstring, moves = beam_search(x.detach(), [0, x.shape[0]], beamsize, threshold, self.qscale, self.qbias).cpu().numpy()
        else:
            logp = x.detach().float().cpu().numpy()
            labels, probs = greedy_step(logp)
            seq, qstring, moves = greedy_collapse(labels, probs, self.alphabet, self.qscale, self.qbias)
        seq = seq[seq != 0].tobytes().decode()
        if qscores:
            seq += qstring[qstring != 0].tobytes().decode()
        if return_path:
            return seq, np.flatnonzero(moves)
        return seq

    def ctc_label_smoothing_loss(self, log_probs, targets, lengths, weights=None):
        """
        CTC loss plus label smoothing (reference: bonito/ctc/model.py:48-54).  `log_probs` is the reference layout
        [T, N, C] on a CUDA device; the native forward's [N, T, C] output becomes it by `permute(1, 0, 2)`, which the
        loss reads in place.  Every input length is T, the CTC loss (`bonito_b200.ctc.loss.ctc_loss`, on the GPU) has
        reduction 'mean', and the smoothing term is -(log_probs * weights).mean() in torch's type promotion, as in the
        reference; `weights` defaults to [0.4, 0.1 / (C - 1), ...].  Deviation: a given `weights` tensor is used as it
        is, where the reference's `weights or ...` raises for one of more than one element.
        Returns {'total_loss', 'loss', 'label_smooth_loss'}.
        """
        from bonito_b200.ctc.loss import ctc_loss
        T, N, C = log_probs.shape
        if weights is None:
            weights = torch.cat([torch.tensor([0.4]), (0.1 / (C - 1)) * torch.ones(C - 1)])
        log_probs_lengths = torch.full(size=(N,), fill_value=T, dtype=torch.int64)
        loss = ctc_loss(log_probs.to(torch.float32), targets, log_probs_lengths, lengths, reduction="mean")
        label_smoothing_loss = -((log_probs * weights.to(log_probs.device)).mean())
        return {"total_loss": loss + label_smoothing_loss, "loss": loss, "label_smooth_loss": label_smoothing_loss}

    def loss(self, log_probs, targets, lengths):
        """`ctc_label_smoothing_loss` with the default weights (reference: bonito/ctc/model.py:56-57)."""
        return self.ctc_label_smoothing_loss(log_probs, targets, lengths)


MAX_BEAMSIZE = 32


def check_beamsize(beamsize):
    if not isinstance(beamsize, int) or not 1 <= beamsize <= MAX_BEAMSIZE:
        raise ValueError(f"beamsize must be an integer in 1..{MAX_BEAMSIZE}, got {beamsize!r}")


def check_alphabet(alphabet):
    if "".join(alphabet) != "NACGT":
        raise ValueError(f"the CTC beam search writes the bases of the alphabet NACGT, the model has {''.join(alphabet)!r}")


def beam_search(logp, offsets, beamsize=5, threshold=1e-3, qscale=1.0, qbias=0.0):
    """
    CTC prefix beam search of a batch of reads in one launch of `b200_ctc_beam_search`.  `logp`: CUDA `[frames, 5]`
    log-probs (class 0 = blank) of the reads packed back to back; `offsets`: the len(reads) + 1 frame boundaries, read r
    being frames offsets[r]:offsets[r + 1].  Returns a CUDA uint8 tensor `[3, frames]` = sequence, qstring, moves in the
    byte layout of `greedy_collapse`.  There is no CPU path.
    """
    from bonito_b200 import native
    check_beamsize(beamsize)
    if not isinstance(logp, torch.Tensor) or not logp.is_cuda:
        raise NotImplementedError("CTC beam search has no CPU path: it needs CUDA log-probs (use beamsize=1 for the greedy decode)")
    if logp.dim() != 2 or logp.shape[1] != 5:
        raise ValueError(f"beam_search: logp must be [frames, 5], got {tuple(logp.shape)}")
    offsets = np.asarray(offsets, dtype=np.int64)
    if offsets.ndim != 1 or offsets.size < 1 or offsets[0] != 0 or offsets[-1] != logp.shape[0] or (np.diff(offsets) < 0).any():
        raise ValueError("beam_search: offsets must rise from 0 to the number of frames")
    logp = logp.to(torch.float16).contiguous()
    frames, reads = logp.shape[0], offsets.size - 1
    with torch.cuda.device(logp.device):
        out = torch.empty(3, frames, dtype=torch.uint8, device=logp.device)
        workspace = torch.empty(native.ctc_beam_workspace_bytes(reads, frames, beamsize), dtype=torch.uint8, device=logp.device)
        native.ctc_beam_search(logp, offsets[:-1], np.diff(offsets), beamsize, threshold, qscale, qbias, workspace,
                               out[0], out[1], out[2])
    return out


def greedy_step(logp):
    """Per-frame argmax of [..., 5] log-probs (equal values: the highest index wins) and its probability exp(logp)."""
    logp = np.asarray(logp, dtype=np.float32)
    labels = (logp.shape[-1] - 1 - np.argmax(logp[..., ::-1], axis=-1)).astype(np.uint8)
    probs = np.exp(np.take_along_axis(logp, labels[..., None].astype(np.int64), axis=-1)[..., 0]).astype(np.float32)
    return labels, probs


def greedy_collapse(labels, probs, alphabet, qscale=1.0, qbias=0.0):
    """
    Greedy CTC collapse of one read's per-frame labels [T] (uint8, 0 = blank) and probabilities [T] (fp32):
      * frame t emits a base when labels[t] != 0 and labels[t] != labels[t - 1] (frame -1 has no label; blanks reset, so
        A _ A emits two A);
      * the quality of a base is phred(mean of probs over the non-blank frames from its emission up to the next emission),
        phred(p) = clip(rint(-10 log10(max(1 - p, 1e-4)) * qscale + qbias) + 33, 33, 126).
    Returns (sequence, qstring, moves) as uint8 [T] arrays: the character / quality on emitting frames and 0 elsewhere,
    moves 1 on emitting frames (the byte layout of the CRF decoder's outputs).
    """
    labels = np.asarray(labels, dtype=np.uint8)
    probs = np.asarray(probs, dtype=np.float32)
    T = labels.shape[0]
    seq = np.zeros(T, dtype=np.uint8)
    qual = np.zeros(T, dtype=np.uint8)
    moves = np.zeros(T, dtype=np.uint8)
    if T == 0:
        return seq, qual, moves
    prev = np.concatenate([[0], labels[:-1]]).astype(np.uint8)
    emit = (labels != 0) & (labels != prev)
    starts = np.flatnonzero(emit)
    if starts.size == 0:
        return seq, qual, moves
    moves[starts] = 1
    letters = np.frombuffer("".join(alphabet).encode(), dtype=np.uint8)
    seq[starts] = letters[labels[starts]]
    # run means over the non-blank frames of each emission's span [start_i, start_{i+1})
    nonblank = (labels != 0).astype(np.float64)
    sums = np.add.reduceat(probs.astype(np.float64) * nonblank, starts)
    counts = np.add.reduceat(nonblank, starts)
    mean = sums / counts
    err = np.maximum(1.0 - mean, 1e-4)
    q = np.rint(-10.0 * np.log10(err) * qscale + qbias) + 33
    qual[starts] = np.clip(q, 33, 126).astype(np.uint8)
    return seq, qual, moves


class Encoder(Module):
    """The blocks of a `[[block]]` config (reference: bonito/ctc/model.py:63-87)."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        features = self.config["input"]["features"]
        activation = layers[self.config["encoder"]["activation"]]()
        encoder_layers = []
        for layer in self.config["block"]:
            encoder_layers.append(Block(features, layer["filters"], activation, repeat=layer["repeat"],
                                        kernel_size=layer["kernel"], stride=layer["stride"], dilation=layer["dilation"],
                                        dropout=layer["dropout"], residual=layer["residual"], separable=layer["separable"]))
            features = layer["filters"]
        self.encoder = Sequential(*encoder_layers)

    def forward(self, x):
        return self.encoder(x)


class TCSConv1d(Module):
    """Time-channel separable Conv1d: depthwise then pointwise, or one dense Conv1d (reference: bonito/ctc/model.py:90-121)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=False,
                 separable=False):
        super().__init__()
        self.separable = separable
        if separable:
            self.depthwise = Conv1d(in_channels, in_channels, kernel_size=kernel_size, stride=stride, padding=padding,
                                    dilation=dilation, bias=bias, groups=in_channels)
            self.pointwise = Conv1d(in_channels, out_channels, kernel_size=1, stride=1, dilation=dilation, bias=bias,
                                    padding=0)
        else:
            self.conv = Conv1d(in_channels, out_channels, kernel_size=kernel_size, stride=stride, padding=padding,
                               dilation=dilation, bias=bias)

    def forward(self, x):
        if self.separable:
            return self.pointwise(self.depthwise(x))
        return self.conv(x)


class Block(Module):
    """repeat x [TCSConv1d, BatchNorm1d(eps=1e-3)] with activation + Dropout between repeats, the optional residual
    [Conv1d 1x1, BatchNorm1d] of the block input added before the last activation (reference: bonito/ctc/model.py:124-192)."""

    def __init__(self, in_channels, out_channels, activation, repeat=5, kernel_size=1, stride=1, dilation=1, dropout=0.0,
                 residual=False, separable=False):
        super().__init__()
        self.use_res = residual
        self.conv = ModuleList()
        _in_channels = in_channels
        padding = self.get_padding(kernel_size[0], stride[0], dilation[0])
        for _ in range(repeat - 1):
            self.conv.extend(self.get_tcs(_in_channels, out_channels, kernel_size=kernel_size, stride=stride,
                                          dilation=dilation, padding=padding, separable=separable))
            self.conv.extend(self.get_activation(activation, dropout))
            _in_channels = out_channels
        self.conv.extend(self.get_tcs(_in_channels, out_channels, kernel_size=kernel_size, stride=stride, dilation=dilation,
                                      padding=padding, separable=separable))
        if self.use_res:
            self.residual = Sequential(*self.get_tcs(in_channels, out_channels))
        self.activation = Sequential(*self.get_activation(activation, dropout))

    def get_activation(self, activation, dropout):
        return activation, Dropout(p=dropout)

    def get_padding(self, kernel_size, stride, dilation):
        if stride > 1 and dilation > 1:
            raise ValueError("Dilation and stride can not both be greater than 1")
        return (kernel_size // 2) * dilation

    def get_tcs(self, in_channels, out_channels, kernel_size=1, stride=1, dilation=1, padding=0, bias=False, separable=False):
        return [TCSConv1d(in_channels, out_channels, kernel_size, stride=stride, dilation=dilation, padding=padding, bias=bias,
                          separable=separable),
                BatchNorm1d(out_channels, eps=1e-3, momentum=0.1)]

    def forward(self, x):
        _x = x
        for layer in self.conv:
            _x = layer(_x)
        if self.use_res:
            _x = _x + self.residual(x)
        return self.activation(_x)


class Decoder(Module):
    """Conv1d(features -> classes, k1, bias) -> Permute([2, 0, 1]) -> log_softmax (reference: bonito/ctc/model.py:195-208)."""

    def __init__(self, features, classes):
        super().__init__()
        self.layers = Sequential(Conv1d(features, classes, kernel_size=1, bias=True), Permute([2, 0, 1]))

    def forward(self, x):
        return log_softmax(self.layers(x), dim=-1)
