"""
The two alignment kernels on batches larger than their grids.  b200_pair_align runs at most 1024 warps and b200_sw_align
at most 2048; above that, pair p shares a warp -- its workspace row and shared traceback tile -- with pair p + warps.
Each batch below puts a long pair (several 256-row strips; for GLOBAL_EDIT a band wider than the 128-diagonal traceback
tile) and a short one (empty or 1-40 bases) on the same warp, in both orders.  Results are integers and op strings, so
every comparison is exact: short pairs against the CPU oracles, long pairs against the same pair launched alone (and a
few against the oracles), and the batch against its own reversal.
"""
import random

import numpy as np
import pytest

import _oracle_align as OA
import _oracle_duplex as OD

pytestmark = pytest.mark.gpu

PA_WARPS, SW_WARPS, EXTRA = 1024, 2048, 77
LONG_BAND = 150              # GLOBAL_EDIT band of the long pairs: 2 * 150 + 1 diagonals, wider than one 128-diagonal tile


def _mutate(rng, s, rate):
    out = []
    for ch in s:
        x = rng.random()
        if x < rate / 2:
            out.append(rng.choice([b for b in "ACGT" if b != ch]))
        elif x < 3 * rate / 4:
            out.append(ch + rng.choice("ACGT"))
        elif x >= rate:
            out.append(ch)
    return "".join(out)


def _short(rng, i):
    if i % 7 == 0:
        return "", "".join(rng.choice("ACGT") for _ in range(rng.randint(0, 9)))
    if i % 7 == 1:
        return "".join(rng.choice("ACGT") for _ in range(rng.randint(1, 9))), ""
    base = "".join(rng.choice("ACGT") for _ in range(rng.randint(1, 40)))
    return _mutate(rng, base, 0.2), _mutate(rng, base, 0.2)


def _long(rng, length):
    base = "".join(rng.choice("ACGT") for _ in range(length))
    return _mutate(rng, base, 0.08), _mutate(rng, base, 0.08)


def _batch(seed, warps, first_long_lengths):
    """warps + EXTRA pairs: warp w < EXTRA holds pairs w and w + warps, one long and one short (long first on even w);
    every other pair is short.  Returns queries, targets and the indices of the long pairs."""
    rng = random.Random(seed)
    n = warps + EXTRA
    qs, rs, long_idx = [None] * n, [None] * n, []
    for w in range(EXTRA):
        lp, sp = (w, w + warps) if w % 2 == 0 else (w + warps, w)
        length = first_long_lengths[w] if w < len(first_long_lengths) else rng.randint(600, 1500)
        qs[lp], rs[lp] = _long(rng, length)
        qs[sp], rs[sp] = _short(rng, w)
        long_idx.append(lp)
    for p in range(EXTRA, warps):
        qs[p], rs[p] = _short(rng, p)
    return qs, rs, sorted(long_idx)


@pytest.fixture(scope="module")
def pair_batch():
    from bonito_b200.align import PairAligner
    qs, rs, long_idx = _batch(5, PA_WARPS, [520, 560, 480, 590])
    return qs, rs, long_idx, PairAligner(qs, rs)


def _bands(qs, rs, long_idx):
    band = np.array([max(len(q), len(r)) for q, r in zip(qs, rs)], dtype=np.int32)
    band[long_idx] = LONG_BAND
    return band


@pytest.mark.parametrize("mode", [pytest.param("edit-traceback", id="GLOBAL_EDIT-traceback"),
                                  pytest.param("edit-score", id="GLOBAL_EDIT-score-only"),
                                  pytest.param("affine", id="SEMIGLOBAL_AFFINE")])
def test_pair_align_shared_warps(pair_batch, mode):
    """b200_pair_align on 1024 + 77 pairs: 77 warps align a long and a short pair one after the other.  Short pairs equal
    the oracle (distance / score and ops), long pairs equal their launch alone, the first four long pairs (<= 600 bases,
    distance within the band) equal the oracle, and the reversed batch gives the same rows."""
    from bonito_b200 import native
    qs, rs, long_idx, al = pair_batch
    n = len(qs)
    idx = np.arange(n)
    long_set = set(long_idx)
    if mode == "affine":
        kind, band, tb = native.PAIR_SEMIGLOBAL_AFFINE, None, True
        oracle = OD.semiglobal_affine
    else:
        kind, band, tb = native.PAIR_GLOBAL_EDIT, _bands(qs, rs, long_idx), mode == "edit-traceback"
        oracle = OD.global_edit
    assert max(len(qs[p]) for p in long_idx) > 2 * 256 and all(len(qs[p]) > 256 for p in long_idx)
    score, ops = al._launch(kind, idx, band, tb)
    for p in range(n):
        if p in long_set:
            continue
        want = oracle(qs[p], rs[p])
        assert score[p] == want[0], (p, qs[p], rs[p])
        if tb:
            assert ops[p] == want[1], (p, qs[p], rs[p])
    for p in long_idx:
        s1, o1 = al._launch(kind, [p], None if band is None else band[[p]], tb)
        assert score[p] == s1[0], p
        if tb:
            assert ops[p] == o1[0], p
    for p in long_idx[:4]:
        if len(qs[p]) > 600 or len(rs[p]) > 600:
            continue
        want = oracle(qs[p], rs[p])
        if mode != "affine":
            assert want[0] <= LONG_BAND
        assert score[p] == want[0], p
        if tb:
            assert ops[p] == want[1], p
    rev = idx[::-1].copy()
    s_rev, o_rev = al._launch(kind, rev, None if band is None else band[rev], tb)
    assert np.array_equal(s_rev[::-1], score)
    if tb:
        assert o_rev[::-1] == ops


def test_sw_align_shared_warps():
    """b200_sw_align on 2048 + 77 pairs: 77 warps align a long and a short pair one after the other.  Every row (score,
    ends, CIGAR counts) equals the Gotoh oracle, long pairs also equal their launch alone, and the reversed batch gives
    the same rows."""
    from bonito_b200.align import sw_align_batch
    qs, rs, long_idx = _batch(9, SW_WARPS, [])
    assert all(len(qs[p]) > 2 * 256 for p in long_idx)
    got = sw_align_batch(rs, qs)
    for p in range(len(qs)):
        assert list(got[p]) == OA.as_row(OA.align(qs[p], rs[p])), (p, len(qs[p]), len(rs[p]))
    for p in long_idx[::8]:
        assert np.array_equal(sw_align_batch([rs[p]], [qs[p]])[0], got[p]), p
    rev = sw_align_batch(rs[::-1], qs[::-1])
    assert np.array_equal(rev[::-1], got)
