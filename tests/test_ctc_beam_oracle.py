"""
The CTC prefix beam search definition (bonito_b200/csrc/ctc_beam.cu) as stated by its CPU oracle, tests/_oracle_ctc_beam.py:
hand-worked cases, the brute force over every label sequence, and the argument checks of the host layers that run
without a GPU.
"""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import _oracle_ctc as oc  # noqa: E402
import _oracle_ctc_beam as ob  # noqa: E402
from bonito_b200 import native, synth  # noqa: E402
from bonito_b200.ctc.model import Model, beam_search  # noqa: E402


def _logp(rows, hi=0.8):
    """Log-probs whose argmax follows `rows` (labels): `hi` on the label, the rest shared equally."""
    out = np.full((len(rows), 5), np.log((1 - hi) / 4), dtype=np.float32)
    out[np.arange(len(rows)), rows] = np.log(hi)
    return out


def _phred(p):
    return chr(int(np.rint(-10 * np.log10(1 - p))) + 33)


def test_hand_worked_cases():
    # all blank
    s, q, mv = ob.beam_search(_logp([0, 0, 0]))
    assert (s, q, mv.tolist()) == ("", "", [0, 0, 0])
    # T = 1, and no frames at all
    s, q, mv = ob.beam_search(_logp([2]))
    assert (s, q, mv.tolist()) == ("C", _phred(0.8), [1])
    s, q, mv = ob.beam_search(np.zeros((0, 5), dtype=np.float32))
    assert (s, q, mv.tolist()) == ("", "", [])
    # A A _ A: the repeat collapses, the blank separates -> two A, the first on frame 0
    s, q, mv = ob.beam_search(_logp([1, 1, 0, 1]))
    assert s == "AA" and mv[0] == 1 and mv.sum() == 2 and len(q) == 2
    # a base enters the beam at the first frame where its class passes the cut, which can be before the frame the greedy
    # decode emits it on; with the other classes below the cut the frames are the greedy ones, and so are the qualities
    rows = [0, 1, 1, 0, 0, 2, 2, 2, 0, 1, 0, 0, 1, 3, 4, 4, 0]
    early = ob.beam_search(_logp(rows, hi=0.97))
    assert early[0] == "ACAAGT" and early[2][0] == 1 and oc.greedy(_logp(rows, hi=0.97))[2][0] == 0
    lp = _logp(rows, hi=0.998).astype(np.float16).astype(np.float32)
    assert ob.beam_search(lp)[0] == oc.greedy(lp)[0] == "ACAAGT"
    s, q, mv = ob.beam_search(lp, qscale=1.5, qbias=-0.5)
    gs, gq, gmv = oc.greedy(lp, qscale=1.5, qbias=-0.5)
    assert (s, q) == (gs, gq) and np.array_equal(mv, gmv)


def test_beam_beats_greedy():
    """Two frames of p = [0.40, 0.35, 0.25, 0, 0]: the best path is blank-blank (0.16), so greedy calls "", but "A" sums
    A_, _A and AA to 0.4025; the A enters the beam at frame 0."""
    with np.errstate(divide="ignore"):
        lp = np.log(np.array([[0.40, 0.35, 0.25, 0.0, 0.0]] * 2, dtype=np.float64))
    assert oc.greedy(lp)[0] == ""
    s, q, mv = ob.beam_search(lp)
    assert (s, mv.tolist()) == ("A", [1, 0])
    assert abs(np.exp(ob.ctc_log_prob(lp, (1,))) - 0.4025) < 1e-7 and abs(np.exp(ob.ctc_log_prob(lp, ())) - 0.16) < 1e-7
    # no frame of the span has A as its argmax: the quality is that of the emission frame alone
    assert q == _phred(0.35)
    assert ob.most_probable_sequence(lp)[0] == (1,)


def test_threshold_rules():
    p = np.array([[0.05, 0.90, 0.05, 0.0, 0.0], [0.0008, 0.0002, 0.999, 0.0, 0.0]])
    with np.errstate(divide="ignore"):
        lp = np.log(p)
    # frame 1: blank and A are below 1e-3 and skipped, so every survivor ends in C
    assert ob.beam_search(lp)[0] == "AC"
    assert ob.search(lp, beam_width=32)[0] == (1, 2)
    # the blank is not exempt: with a cut of 0.1 frame 0 can only emit A, and the empty prefix leaves the beam
    assert ob.beam_search(lp, threshold=0.1)[0] == "AC"
    assert ob.beam_search(lp[:1], threshold=0.1)[0] == "A"
    # every class below the cut: the frame changes nothing
    flat = np.log(np.full((3, 5), 0.2))
    s, q, mv = ob.beam_search(flat, threshold=0.5)
    assert (s, q, mv.tolist()) == ("", "", [0, 0, 0])
    mixed = np.concatenate([_logp([3]), flat, _logp([3])])
    s, q, mv = ob.beam_search(mixed, threshold=0.5)
    assert (s, mv.tolist()) == ("G", [1, 0, 0, 0, 0])            # G G with nothing between them is one G
    assert ob.beam_search(mixed, threshold=0.0)[0] != "G"             # without the cut the flat frames do change the beam


def test_ties_follow_rank_then_kept_then_class():
    # one frame, four labels at 0.25 each and no blank: the lowest class wins
    with np.errstate(divide="ignore"):
        lp = np.log(np.array([[0.0, 0.25, 0.25, 0.25, 0.25]]))
    assert ob.beam_search(lp)[0] == "A"
    # blank and A tie at 0.5: the kept (empty) prefix comes before its child
    with np.errstate(divide="ignore"):
        lp = np.log(np.array([[0.5, 0.5, 0.0, 0.0, 0.0]]))
    assert ob.beam_search(lp)[0] == ""


def test_width_one_is_not_the_greedy_decode_but_a_valid_search():
    rows = [1, 1, 0, 2, 2, 0, 0, 3]
    assert ob.beam_search(_logp(rows, hi=0.99), beam_width=1)[0] == "ACG"


@pytest.mark.parametrize("seed", range(12))
def test_wide_beam_without_cut_is_the_most_probable_sequence(seed):
    rng = np.random.default_rng(seed)
    T = 3 + seed % 4
    logits = rng.normal(size=(T, 5)) * (1.0 + seed % 3)
    lp = (logits - np.log(np.exp(logits).sum(-1, keepdims=True))).astype(np.float16).astype(np.float64)
    best, top, second = ob.most_probable_sequence(lp)
    if top - second <= 1e-9:
        pytest.skip("the two most probable sequences tie")
    labels, frames = ob.search(lp, beam_width=10 ** 6, threshold=0.0)
    assert labels == best
    assert len(frames) == len(labels) and list(frames) == sorted(set(frames))


def test_long_read_does_not_underflow():
    rows = ([1] * 2 + [0] + [2] * 3 + [0] * 2 + [3] + [4] * 2) * 400
    s, q, mv = ob.beam_search(_logp(rows, hi=0.9))
    assert s == "ACGT" * 400 and len(q) == len(s) and int(mv.sum()) == len(s)


def test_argument_checks_without_a_gpu():
    spec = synth.quartznet_spec("v1", max_repeat=2)
    m = Model(synth.quartznet_config(spec)).eval()
    for bad in (0, -1, 33, 2.5, "5"):
        with pytest.raises(ValueError, match="beamsize"):
            m.decode(torch.zeros(4, 5), beamsize=bad)
        with pytest.raises(ValueError, match="beamsize"):
            beam_search(torch.zeros(4, 5), [0, 4], beamsize=bad)
    from bonito_b200.ctc.basecall import basecall
    with pytest.raises(ValueError, match="beamsize"):
        basecall(m, [], beamsize=33)
    consumed = []

    def reads():
        consumed.append(1)
        yield None
    with pytest.raises(NotImplementedError, match="no CPU path"):
        basecall(m, reads(), beamsize=5)
    assert not consumed
    with pytest.raises(NotImplementedError, match="no CPU path"):
        m.decode(torch.zeros(4, 5), beamsize=2)
    with pytest.raises(NotImplementedError, match="no CPU path"):
        beam_search(torch.zeros(4, 5), [0, 4])
    # the workspace query: per-read arrays (padded to 256 bytes) + 8 bytes for each of the 1 + width * frames nodes of a read
    assert native.ctc_beam_workspace_bytes(3, 100, 5) == 256 + 8 * (3 + 5 * 100)
    assert native.ctc_beam_workspace_bytes(0, 0, 5) == 0 and native.ctc_beam_workspace_bytes(3, 100, 33) == 0
