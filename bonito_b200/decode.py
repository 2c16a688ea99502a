"""
Decoder op with the call contract of `koi.decode.beam_search` / `to_str`
(`bonito/crf/basecall.py:7,36-40,50-54`).

koi's beam search is a closed binary with no pinned outputs (SURVEY.md section 8c), so the default
arithmetic here is the reference's in-repo decode definition (`SeqdistModel.decode_batch`,
`bonito/crf/model.py:196-199`): exact forward-backward posteriors followed by a Viterbi
pass over the log-posteriors; `beam_width` and `beam_cut` are then unused (the search is exact).

`decoder="beam"` (or `B200_DECODER=beam` in the environment) runs this repository's own beam search
instead -- a backward-guided prefix search with `beam_width` (<= 32) entries and the `beam_cut`
pruning threshold, one warp per chunk (`b200_crf_beam_search`); quality strings come from the same
posterior move mass.  It is an approximation of the most probable SEQUENCE (alignments of a prefix are
summed), not of koi's implementation; on peaked score distributions it returns the same calls as the
exact decoder (tests/test_gpu_kernels.py::test_beam_search_*).
"""

import os

import numpy as np
import torch

from bonito_b200.engine import CrfDecoder, score_layout

_decoder = CrfDecoder()


def beam_search(scores, beam_width=32, beam_cut=100.0, scale=1.0, offset=0.0, blank_score=2.0, decoder=None):
    """
    scores: CUDA fp16 contiguous, either [N, T, 4**(k+1)] (fixed blank: no blank column, [state][m0..m3], the stay score is
    `blank_score`) or [N, T, 5 * 4**k] (learned blank scores: the CTC_CRF layout [state][stay, m0..m3]; `blank_score` is
    ignored).  The width picks the layout and k.  The beam search (`decoder="beam"`) needs a fixed blank score.
    Returns (sequence, qstring, moves): three CPU uint8 tensors [N, T]; sequence / qstring carry an
    ASCII character on frames that emit a base and 0 elsewhere.  `scale` / `offset` are the qscore
    scale and bias (q = -10 log10(max(1-p, 1e-4)) * scale + offset).
    """
    n, t, c = scores.shape
    state_len, _ = score_layout(c)
    decoder = decoder or os.environ.get("B200_DECODER", "exact")
    if decoder not in ("exact", "beam"):
        raise ValueError(f"unknown decoder {decoder!r} (exact, beam)")
    beam = (min(int(beam_width), 32), float(beam_cut)) if decoder == "beam" else None
    moves, sequence, qstring = _decoder(scores, state_len, blank_score=blank_score, qscale=scale, qbias=offset, beam=beam)
    return sequence.cpu(), qstring.cpu(), moves.cpu()


def to_str(x, encoding="ascii"):
    """Bytes of the non-zero entries of a uint8 tensor/array, decoded."""
    arr = x.numpy() if isinstance(x, torch.Tensor) else np.asarray(x)
    return arr[arr != 0].tobytes().decode(encoding)
