"""
CPU oracle of the layers that dna_r10.4.1@v4.0 and dna_r9.4.1@v3 add to the LSTM-CRF stack (test infrastructure, built on
oracle/crf_oracle.py):
  * `lstm_crf_forward`: crf_oracle.lstm_crf_forward plus a Clamp behind every convolution (spec "conv_clamp", exact on the
    fp16 activation), a Linear in front of the head (spec "bottleneck", with bias) and heads with learned blank scores
    (blank_score None: the full [state][stay, m0..m3] layout, reference bonito/crf/model.py:150-162, bonito/nn.py:283-298);
  * `decode_native_lb`: crf_oracle.decode_native on learned-blank scores -- the same posterior-Viterbi decode and output
    conventions, with the stay edges read from the scores instead of a fixed blank_score.
"""
import numpy as np
import torch.nn.functional as F

from oracle import crf_oracle as O


def lstm_crf_forward(weights, spec, x, expand_blanks=False, return_features=False, fp16=False):
    """x [N, 1, L] -> scores [T, N, C] as crf_oracle.lstm_crf_forward, for specs with conv_clamp / bottleneck / learned
    blanks; `expand_blanks` only concerns fixed-blank heads."""
    feats = {}
    h = x
    for i, (_, _, _, stride, pad, act) in enumerate(spec["convs"]):
        h = O.convolution(h, weights[f"conv{i}.weight"], weights[f"conv{i}.bias"], stride, pad, act, fp16)
        if spec.get("conv_clamp") is not None:
            h = h.clamp(*spec["conv_clamp"])
        feats[f"conv{i}"] = h
    h = h.permute(2, 0, 1)
    for i in range(spec["n_lstm"]):
        h = O.lstm_layer(h, weights[f"lstm{i}.w_ih"], weights[f"lstm{i}.w_hh"], weights[f"lstm{i}.b_ih"],
                         weights[f"lstm{i}.b_hh"], spec["reverse"][i], fp16)
        feats[f"lstm{i}"] = h
    if spec.get("bottleneck") is not None:
        h = O._r16(F.linear(O._r16(h, fp16), weights["linear.weight"], weights["linear.bias"]), fp16)
        feats["linear"] = h
    s = O.linear_crf(O._r16(h, fp16), weights["crf.weight"], weights.get("crf.bias"), activation=spec.get("crf_activation"),
                     scale=spec.get("crf_scale"), blank_score=spec["blank_score"], expand_blanks=False, fp16=fp16)
    s = O._r16(s, fp16)
    if expand_blanks and spec["blank_score"] is not None:
        T_, N_, C_ = s.shape
        s = F.pad(s.view(T_, N_, C_ // 4, 4), (1, 0), value=spec["blank_score"]).view(T_, N_, -1)
    if spec.get("clamp") is not None:
        s = s.clamp(*spec["clamp"])
    return (s, feats) if return_features else s


def decode_native_lb(scores_ntc, state_len, qscale=1.0, qbias=0.0, n_base=4):
    """Oracle for b200_crf_decode_lb: scores [N, T, S*5] in the [state][stay, m0..m3] layout (fp16-valued) ->
    (moves, sequence, qstring) uint8 [N, T] and the move-mass table, as crf_oracle.decode_native returns them."""
    x = np.asarray(scores_ntc, dtype=np.float64)
    N, T, C = x.shape
    idx = O.crf_idx(state_len, n_base)
    Ms = x.transpose(1, 0, 2).reshape(T, N, -1, n_base + 1)
    post = O.posteriors(Ms, idx)
    lp = np.log(post.astype(np.float32) + np.float32(1e-8))
    states, edges = O.viterbi_edges(lp, idx)
    move = edges != 0
    base = states % n_base
    S = Ms.shape[2]
    mass = post[..., 1:].sum(-1).reshape(T, N, S // n_base, n_base).sum(2)  # [T, N, 4]
    p = np.take_along_axis(mass, base[..., None], axis=-1)[..., 0]
    err = np.maximum(1.0 - p, 1e-4)
    q = np.clip(np.rint(-10.0 * np.log10(err) * qscale + qbias).astype(np.int64) + 33, 33, 126)
    letters = np.frombuffer(b"ACGT", dtype="u1")
    moves = move.T.astype(np.uint8)
    seq = np.where(move, letters[base], 0).T.astype(np.uint8)
    qual = np.where(move, q, 0).T.astype(np.uint8)
    return moves, seq, qual, mass.transpose(1, 0, 2)


def strings(seq):
    """Decoded strings of a sequence array [N, T] (0 = no emission)."""
    return [r[r != 0].tobytes().decode() for r in np.asarray(seq)]
