"""
CTC-CRF model package (`Model`, `basecall` are what `load_symbol` looks up:
`bonito/util.py:223-234`, `bonito/cli/basecaller.py:71`).

Mirror of `bonito/crf/model.py`: the sequence distribution `CTC_CRF` with its scoring API and CTC
loss (logZ, normalise, forward / backward scores, posteriors, viterbi, ctc_loss, ctc_viterbi_alignments:
the koi.ctc calls of bonito/crf/model.py:47-143, here on the sm_90a kernels of csrc/ctc_crf.cu),
`SeqdistModel` with `loss`, and `Model` with the `use_koi` swap-in hook.  The scoring API takes
reference-layout scores [T, N, n_score()] on a CUDA device; gradients flow through autograd.
"""

import numpy as np
import torch
import torch.nn.functional as F

from bonito_b200.crf.lattice import Log, Max, sparse_backward_scores, sparse_forward_scores, sparse_logz, \
    target_logz, target_viterbi
from bonito_b200.nn import (Module, Convolution, LinearCRFEncoder, Serial, Permute, layers, to_dict, from_dict,
                            register)


def get_stride(m, stride=1):
    """Total down-sampling of a module tree (reference: bonito/crf/model.py:15-27)."""
    if hasattr(m, "output_stride"):
        return m.output_stride(stride)
    if hasattr(m, "stride"):
        s = m.stride
        if isinstance(s, tuple):
            assert len(s) == 1
            s = s[0]
        return stride * s
    for child in m.children():
        stride = get_stride(child, stride)
    return stride


class CTC_CRF:
    """
    State graph of the k-mer CRF: 4**state_len states, 5 in-edges per state
    (`idx[s, 0] = s` stay; `idx[s, 1+j] = j * 4**(state_len-1) + s // 4` move),
    flat score index `s * 5 + e` (reference: bonito/crf/model.py:30-45).
    """

    def __init__(self, state_len, alphabet):
        self.alphabet = alphabet
        self.state_len = state_len
        self.n_base = len(alphabet[1:])
        n_states = self.n_base ** state_len
        states = torch.arange(n_states)
        moves = states.repeat_interleave(self.n_base).reshape(self.n_base, -1).T
        self.idx = torch.cat([states[:, None], moves], dim=1).to(torch.int32)

    def n_score(self):
        return len(self.alphabet) * self.n_base ** self.state_len

    def reverse_complement(self, scores):
        """Scores of the reverse-complement strand (reference: bonito/crf/model.py:84-96); [T, N, C] layout."""
        T, N, C = scores.shape
        k, nb = self.state_len, self.n_base
        x = scores.reshape(T, N, *([nb] * k), nb + 1)
        blanks = torch.flip(x[..., 0].permute(0, 1, *range(k + 1, 1, -1)).reshape(T, N, -1, 1), [0, 2])
        emissions = torch.flip(
            x[..., 1:].permute(0, 1, *range(k, 1, -1), k + 2, k + 1).reshape(T, N, -1, nb), [0, 2, 3])
        return torch.cat([blanks, emissions], dim=-1).reshape(T, N, -1)

    def path_to_str(self, path):
        letters = np.frombuffer("".join(self.alphabet).encode(), dtype="u1")
        return letters[path[path != 0]].tobytes().decode()

    # -- scoring API (reference: bonito/crf/model.py:47-82, 98-103, 110-143) ------------------------------------------
    # scores: [T, N, n_score()] on a CUDA device, the edge from idx[s, e] into s at column s*5 + e; fp16 is upcast to fp32
    def logZ(self, scores, S=Log):
        """logZ [N] of the whole lattice (alpha_0 = beta_T = S.one for every state)."""
        return sparse_logz(scores, self.state_len, S)

    def normalise(self, scores):
        return scores - self.logZ(scores)[:, None] / len(scores)

    def forward_scores(self, scores, S=Log):
        """alpha [T+1, N, 4**state_len]."""
        return sparse_forward_scores(scores, self.state_len, S)

    def backward_scores(self, scores, S=Log):
        """beta [T+1, N, 4**state_len]."""
        return sparse_backward_scores(scores, self.state_len, S)

    def compute_transition_probs(self, scores, betas):
        T, N, C = scores.shape
        log_trans = scores.reshape(T, N, -1, self.n_base + 1) + betas[1:, :, :, None]
        # (new state, dropped base) -> (old state, emitted base)
        log_trans = torch.cat([log_trans[:, :, :, [0]],
                               log_trans[:, :, :, 1:].transpose(3, 2).reshape(T, N, -1, self.n_base)], dim=-1)
        return torch.softmax(log_trans, dim=-1), torch.softmax(betas[0], dim=-1)

    def posteriors(self, scores, S=Log):
        """d logZ(scores, S).sum() / d scores, [T, N, n_score()]: edge marginals (Log) or the best path's one-hot (Max)."""
        with torch.enable_grad():
            x = scores.detach().requires_grad_()
            grad, = torch.autograd.grad(self.logZ(x, S).sum(), x)
        return grad

    def viterbi(self, scores):
        """Best path [T, N]: 0 on a stay, else 1 + the emitted base."""
        a = self.posteriors(scores, Max).argmax(2)
        moves = (a % len(self.alphabet)) != 0
        return torch.where(moves, 1 + torch.div(a, len(self.alphabet), rounding_mode="floor") % self.n_base, 0)

    def prepare_ctc_scores(self, scores, targets):
        """Stay and move scores [T, N, L] / [T, N, L-1] of the k-mers along zero-padded targets [N, max_len] (1 + base)."""
        targets = torch.clamp(targets - 1, 0)          # CTC labels (blank = 0) -> bases
        T, N, C = scores.shape
        scores = scores.to(torch.float32)
        n = targets.size(1) - (self.state_len - 1)
        stay_idx = sum(targets[:, i:n + i] * self.n_base ** (self.state_len - i - 1)
                       for i in range(self.state_len)) * len(self.alphabet)
        move_idx = stay_idx[:, 1:] + targets[:, :n - 1] + 1
        return scores.gather(2, stay_idx.expand(T, -1, -1)), scores.gather(2, move_idx.expand(T, -1, -1))

    def ctc_loss(self, scores, targets, target_lengths, loss_clip=None, reduction="mean", normalise_scores=True):
        if reduction not in ("mean", "none", None):
            raise ValueError("Unknown reduction type {}".format(reduction))
        if normalise_scores:
            scores = self.normalise(scores)
        stay, move = self.prepare_ctc_scores(scores, targets)
        logz = target_logz(stay, move, target_lengths + 1 - self.state_len)
        loss = -(logz / target_lengths)
        if loss_clip:
            loss = torch.clamp(loss, 0.0, loss_clip)
        return loss.mean() if reduction == "mean" else loss

    def ctc_viterbi_alignments(self, scores, targets, target_lengths):
        """One-hot [T, N, L] of the best alignment: a stay at j and the move j -> j+1 both mark column j."""
        stay, move = self.prepare_ctc_scores(scores, targets)
        dstay, dmove = target_viterbi(stay, move, target_lengths + 1 - self.state_len)
        return dstay + F.pad(dmove, (0, 1))


def conv(c_in, c_out, ks, stride=1, bias=False, activation=None, norm=None):
    return Convolution(c_in, c_out, ks, stride=stride, padding=ks // 2, bias=bias, activation=activation, norm=norm)


def rnn_encoder(n_base, state_len, insize=1, first_conv_size=4, stride=5, winlen=19, activation="swish",
                rnn_type="lstm", features=768, scale=5.0, blank_score=None, expand_blanks=True, num_layers=5,
                norm=None):
    """Old-style ([encoder] without `type`) config -> module tree (reference: bonito/crf/model.py:150-162)."""
    rnn = layers[rnn_type]
    return Serial([
        conv(insize, first_conv_size, ks=5, bias=True, activation=activation, norm=norm),
        conv(first_conv_size, 16, ks=5, bias=True, activation=activation, norm=norm),
        conv(16, features, ks=winlen, stride=stride, bias=True, activation=activation, norm=norm),
        Permute([2, 0, 1]),
        *(rnn(features, features, reverse=(num_layers - i) % 2) for i in range(num_layers)),
        LinearCRFEncoder(features, n_base, state_len, activation="tanh", scale=scale,
                         blank_score=blank_score, expand_blanks=expand_blanks),
    ])


@register
class SeqdistModel(Module):
    def __init__(self, encoder, seqdist, n_pre_post_context_bases=None, target_projection=None):
        super().__init__()
        self.seqdist = seqdist
        self.encoder = encoder
        self.stride = get_stride(encoder)
        self.alphabet = seqdist.alphabet
        if n_pre_post_context_bases is None:
            self.n_pre_context_bases, self.n_post_context_bases = seqdist.state_len - 1, 1
        else:
            self.n_pre_context_bases, self.n_post_context_bases = n_pre_post_context_bases
        if target_projection is None:
            self.target_projection = None
        else:
            self.register_buffer("target_projection", torch.tensor([0] + target_projection), persistent=False)
        self._native = None        # set by use_koi(): dict of basecaller settings
        self._plan = None          # built lazily, after the weights are loaded / fused

    @classmethod
    def from_dict(cls, model_dict, layer_types=None):
        kwargs = dict(model_dict, encoder=from_dict(model_dict["encoder"], layer_types),
                      seqdist=CTC_CRF(**model_dict["seqdist"]))
        return cls(**kwargs)

    # -- forward -----------------------------------------------------------------------------------
    def forward(self, x, *args, slot=0):
        """
        Plain module tree ([T, N, C+blanks], the reference's non-koi path) unless `use_koi` armed the
        native engine, in which case the result is [N, T, C] fp16 without blank column and any failure to
        reach the sm_90a kernels raises (no CPU fallback).
        """
        if self._native is None:
            if x.is_cuda:
                # the only CUDA path of this package is the native engine; an eager-torch forward here would be a silent
                # non-native result with a different layout ([T, N, C+blanks])
                raise RuntimeError("bonito_b200: CUDA model called without use_koi(); call model.use_koi(...) "
                                   "(load_model(..., use_koi=True)) or run the module tree on the CPU")
            return self.encoder(x)
        # `slot`: independent buffer set of the native plan, for callers that keep several batches in flight on
        # different streams (score_batches)
        return self.native_plan(x.device if x.is_cuda else None).forward(x, slot=slot)

    def native_plan(self, device=None):
        from bonito_b200 import native
        from bonito_b200.engine import compile_lstm_crf
        from bonito_b200.engine_tf import compile_transformer, find_transformer_encoder
        native.require()
        if device is None:
            device = next(self.parameters()).device
        if torch.device(device).type != "cuda":
            raise native.NativeError("the native path was requested (use_koi) but the model is not on a CUDA device")
        if self._plan is None or self._plan.device != torch.device(device):
            if find_transformer_encoder(self.encoder) is not None:
                self._plan = compile_transformer(self.encoder, device)
            else:
                self._plan = compile_lstm_crf(self.encoder, device, quantize=bool((self._native or {}).get("quantize")))
        return self._plan

    def invalidate_plan(self):
        self._plan = None

    def _apply(self, fn, *args, **kwargs):
        self._plan = None  # .half()/.to() change the tensors the plan was packed from
        return super()._apply(fn, *args, **kwargs)

    def apply(self, fn):
        self._plan = None  # e.g. model.apply(fuse_bn_) rewrites the conv weights
        return super().apply(fn)

    def load_state_dict(self, *args, **kwargs):
        self._plan = None  # the plan holds packed copies of the weights
        return super().load_state_dict(*args, **kwargs)

    def use_koi(self, **kwargs):
        """Arm the native engine (the hook `_load_model` calls: bonito/util.py:292-296)."""
        self._native = dict(kwargs)
        self._plan = None

    # -- decode ------------------------------------------------------------------------------------
    def decode_batch(self, x):
        """
        x: scores.  Native layout [N, T, C] on CUDA (no blank column, or the [state][stay, m0..m3] layout of a head with
        learned blank scores) -> list of N strings, via the sm_90a posterior-Viterbi kernel (same maths as the reference's decode_batch, bonito/crf/model.py:196-199).
        """
        from bonito_b200.decode import beam_search, to_str
        if not x.is_cuda:
            raise NotImplementedError("decode_batch runs on the native CUDA decoder only")
        blank = self._blank_score()
        if blank is None:        # learned blank scores: the stay scores are columns of x, there is no fixed one to pass
            seq, _, _ = beam_search(x.contiguous())
        else:
            seq, _, _ = beam_search(x.contiguous(), blank_score=blank)
        return [to_str(row) for row in seq]

    def decode(self, x):
        return self.decode_batch(x.unsqueeze(0))[0]

    def loss(self, scores, targets, target_lengths, **kwargs):
        """CTC-CRF loss of reference-layout scores [T, N, n_score()] (reference: bonito/crf/model.py:204-207)."""
        if self.target_projection is not None:
            targets = self.target_projection[targets]
        return self.seqdist.ctc_loss(scores.to(torch.float32), targets, target_lengths, **kwargs)

    def _blank_score(self):
        """The head's fixed blank score; None when the head learns its blank scores (blank_score=None)."""
        for m in self.encoder.modules():
            if isinstance(m, LinearCRFEncoder):
                return None if m.blank_score is None else float(m.blank_score)
        return 2.0

    def to_dict(self, include_weights=False):
        if include_weights:
            raise NotImplementedError
        out = {
            "encoder": to_dict(self.encoder),
            "seqdist": {"state_len": self.seqdist.state_len, "alphabet": self.seqdist.alphabet},
            "n_pre_post_context_bases": (self.n_pre_context_bases, self.n_post_context_bases),
        }
        if self.target_projection is not None:
            out["target_projection"] = self.target_projection.tolist()[1:]
        return out


class Model(SeqdistModel):
    """`Model(config)` for `package = "bonito.crf"` configs (reference: bonito/crf/model.py:225-246)."""

    def __init__(self, config):
        seqdist = CTC_CRF(state_len=config["global_norm"]["state_len"], alphabet=config["labels"]["labels"])
        if "type" in config["encoder"]:
            encoder = from_dict(config["encoder"])
        else:
            encoder = rnn_encoder(seqdist.n_base, seqdist.state_len, insize=config["input"]["features"],
                                  **config["encoder"])
        super().__init__(encoder, seqdist, n_pre_post_context_bases=config["input"].get("n_pre_post_context_bases"))
        self.config = config
