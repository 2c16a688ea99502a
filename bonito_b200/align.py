"""
Alignment of basecalls to their references for `evaluate`: the fields of the reference's `AlignResult`
(bonito/cli/evaluate.py:22-67), computed from one batched Smith-Waterman launch on the GPU (`b200_sw_align`, the
scoring and tie rules are in bonito_b200/csrc/align.cu) instead of parasail one pair at a time.

Deviation: a pair whose best local score is 0 (no base in common) gives `accuracy 0.0` with `ref_len` / `seq_len` set
and every other field 0; the reference divides by an empty CIGAR there and raises ZeroDivisionError.
"""

from dataclasses import dataclass

import numpy as np
import torch

from bonito_b200 import native

MAX_LEN = 65535                  # the kernel packs each count into 16 bits

_ACGT = np.zeros(256, dtype=bool)
_ACGT[np.frombuffer(b"ACGT", dtype=np.uint8)] = True


@dataclass
class AlignResult:
    accuracy: float = 0
    num_correct: int = 0
    num_mismatches: int = 0
    num_insertions: int = 0
    num_deletions: int = 0
    ref_len: int = 0
    seq_len: int = 0
    align_ref_start: int = 0
    align_ref_end: int = 0
    align_seq_start: int = 0
    align_seq_end: int = 0


def _pack(strings, what):
    """Strings -> (uint8 bytes, int64 offsets, int32 lengths); refuses non-ACGT bytes and sequences over MAX_LEN."""
    raw = [s.encode() if isinstance(s, str) else bytes(s) for s in strings]
    lengths = np.fromiter((len(b) for b in raw), dtype=np.int64, count=len(raw))
    if lengths.size and lengths.max() > MAX_LEN:
        i = int(np.argmax(lengths))
        raise ValueError(f"{what} {i} has {lengths[i]} bases; at most {MAX_LEN} can be aligned")
    data = np.frombuffer(b"".join(raw), dtype=np.uint8)
    if not _ACGT[data].all():
        bad = int(np.flatnonzero(~_ACGT[data])[0])
        i = int(np.searchsorted(np.cumsum(lengths), bad, side="right"))
        raise ValueError(f"{what} {i} has a byte other than A, C, G, T ({bytes(data[bad:bad + 1])!r})")
    offsets = np.zeros(len(raw), dtype=np.int64)
    if len(raw) > 1:
        np.cumsum(lengths[:-1], out=offsets[1:])
    return data, offsets, lengths.astype(np.int32)


def _pinned(array):
    """A pinned copy with at least one element (all-empty strings still give the kernel a non-null buffer)."""
    t = torch.zeros(max(array.size, 1), dtype=torch.from_numpy(np.empty(0, array.dtype)).dtype, pin_memory=True)
    t.numpy()[:array.size] = array
    return t


def sw_align_batch(refs, seqs, device="cuda"):
    """Raw kernel output for each pair (query = seq, target = ref): int32 numpy [n, 7] of score, end_query, end_ref, n_eq,
    n_x, n_ins, n_del.  Every input is checked before anything is launched."""
    if len(refs) != len(seqs):
        raise ValueError(f"{len(refs)} references for {len(seqs)} sequences")
    q, q_off, q_len = _pack(seqs, "sequence")
    r, r_off, r_len = _pack(refs, "reference")
    n = len(seqs)
    if n == 0:
        return np.zeros((0, 7), dtype=np.int32)
    device = torch.device(device)
    native.require()
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream()
        query = _pinned(q).to(device, non_blocking=True)
        ref = _pinned(r).to(device, non_blocking=True)
        meta = [_pinned(a) for a in (q_off, q_len, r_off, r_len)]
        workspace = torch.empty(native.sw_align_workspace_bytes(n, int(r_len.max())), dtype=torch.uint8, device=device)
        out = torch.empty(n, 7, dtype=torch.int32, device=device)
        native.sw_align(query, meta[0], meta[1], ref, meta[2], meta[3], workspace, out, stream=stream)
        result = out.cpu()               # synchronises the stream, so the pinned arrays may be released after this
    return result.numpy()


# ------------------------------------------------------------------------------------------------ pairwise, with ops
# `duplex` aligns whole reads (b200_pair_align, rules in bonito_b200/csrc/pair_align.cu): GLOBAL_EDIT stands in for
# edlib.align(task="path"), SEMIGLOBAL_AFFINE for parasail.sg_trace_scan_32(q, r, 10, 2, dnafull).

EDIT_BAND0 = 256                 # first band half-width of GLOBAL_EDIT; a pair whose distance exceeds it is re-run at 2k


def _pack_bytes(strings):
    """Byte strings -> (uint8 bytes, int64 offsets, int32 lengths), any byte values."""
    raw = [s.encode() if isinstance(s, str) else bytes(s) for s in strings]
    lengths = np.fromiter((len(b) for b in raw), dtype=np.int64, count=len(raw))
    offsets = np.zeros(len(raw), dtype=np.int64)
    if len(raw) > 1:
        np.cumsum(lengths[:-1], out=offsets[1:])
    return np.frombuffer(b"".join(raw), dtype=np.uint8), offsets, lengths.astype(np.int32)


def band_cells(m, n, k):
    """Cells of the GLOBAL_EDIT band of one pair (rows 1..m, columns 1..n, diagonals [min(0,n-m)-k, max(0,n-m)+k])."""
    if m == 0 or n == 0:
        return 0
    k = min(k, max(m, n))
    lo, hi = min(0, n - m) - k, max(0, n - m) + k
    i = np.arange(1, m + 1, dtype=np.int64)
    return int(np.clip(np.minimum(n, i + hi) - np.maximum(1, i + lo) + 1, 0, None).sum())


class PairAligner:
    """Pairs (query p, target p) uploaded once; GLOBAL_EDIT / SEMIGLOBAL_AFFINE launches over any subset of them.
    `stats` counts launches, computed cells and kernel milliseconds (CUDA events) per mode."""

    def __init__(self, queries, targets, device="cuda"):
        if len(queries) != len(targets):
            raise ValueError(f"{len(queries)} queries for {len(targets)} targets")
        q, self.q_off, self.q_len = _pack_bytes(queries)
        r, self.r_off, self.r_len = _pack_bytes(targets)
        self.device = torch.device(device)
        native.require()
        with torch.cuda.device(self.device):
            self.query = _pinned(q).to(self.device, non_blocking=True)
            self.ref = _pinned(r).to(self.device, non_blocking=True)
        self.stats = {"edit_passes": 0, "edit_cells": 0, "edit_ms": 0.0, "affine_launches": 0, "affine_cells": 0,
                      "affine_ms": 0.0}

    def trace_bytes(self, mode, idx, band=None):
        return [native.pair_align_trace_bytes(mode, self.q_len[p], self.r_len[p], 0 if band is None else band[t])
                for t, p in enumerate(idx)]

    def _launch(self, mode, idx, band, traceback):
        """One b200_pair_align launch over pairs `idx` -> (scores int32 [len(idx)], list of op strings or None)."""
        idx = np.asarray(idx, dtype=np.int64)
        ql, rl = self.q_len[idx], self.r_len[idx]
        bd = None if band is None else np.asarray(band, dtype=np.int32)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream()
            ws = torch.empty(native.pair_align_workspace_bytes(mode, ql, rl, bd, traceback), dtype=torch.uint8,
                             device=self.device)
            out = torch.empty(len(idx), 2, dtype=torch.int32, device=self.device)
            ops = ops_off = None
            if traceback:
                slot = ql.astype(np.int64) + rl
                ops_off = np.zeros(len(idx), dtype=np.int64)
                np.cumsum(slot[:-1], out=ops_off[1:])
                ops = torch.empty(max(int(slot.sum()), 1), dtype=torch.uint8, device=self.device)
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record(stream)
            native.pair_align(mode, self.query, self.q_off[idx], ql, self.ref, self.r_off[idx], rl, bd, ws, out, ops=ops,
                              ops_off=ops_off, traceback=traceback, stream=stream)
            end.record(stream)
            res = out.cpu().numpy()
            host_ops = ops.cpu().numpy() if traceback else None
            ms = start.elapsed_time(end)
        key = "edit" if mode == native.PAIR_GLOBAL_EDIT else "affine"
        self.stats[f"{key}_ms"] += ms
        if not traceback:
            return res[:, 0], None
        strings = []
        for t in range(len(idx)):
            end_at = int(ops_off[t] + slot[t])
            strings.append(host_ops[end_at - int(res[t, 1]):end_at].tobytes().decode("ascii"))
        return res[:, 0], strings

    def global_edit(self, idx, k0=EDIT_BAND0, trace_budget=None):
        """Banded GLOBAL_EDIT of pairs `idx`: score-only passes at k0, 2 k0, ... until every distance is <= its band (or
        the band covers the matrix), then one traceback pass per group of pairs whose traceback fits `trace_budget` bytes.
        -> (distances, op strings (None for a pair whose traceback alone exceeds the budget), passes per pair)."""
        idx = np.asarray(idx, dtype=np.int64)
        full = np.maximum(self.q_len[idx], self.r_len[idx]).astype(np.int64)
        band = np.minimum(k0, full)
        passes = np.zeros(len(idx), dtype=np.int64)
        pending = np.arange(len(idx))
        while len(pending):
            scores, _ = self._launch(native.PAIR_GLOBAL_EDIT, idx[pending], band[pending], traceback=False)
            self.stats["edit_passes"] += 1
            self.stats["edit_cells"] += sum(band_cells(self.q_len[p], self.r_len[p], k)
                                            for p, k in zip(idx[pending], band[pending]))
            passes[pending] += 1
            done = (scores <= band[pending]) | (band[pending] >= full[pending])
            pending = pending[~done]
            band[pending] = np.minimum(2 * band[pending], full[pending])
        dist = np.zeros(len(idx), dtype=np.int64)
        ops = [None] * len(idx)
        sizes = self.trace_bytes(native.PAIR_GLOBAL_EDIT, idx, band)
        for group in _budget_groups(sizes, trace_budget):
            scores, strings = self._launch(native.PAIR_GLOBAL_EDIT, idx[group], band[group], traceback=True)
            self.stats["edit_passes"] += 1
            self.stats["edit_cells"] += sum(band_cells(self.q_len[p], self.r_len[p], k)
                                            for p, k in zip(idx[group], band[group]))
            for t, g in enumerate(group):
                dist[g], ops[g] = scores[t], strings[t]
        return dist, ops, passes

    def semiglobal_affine(self, idx, trace_budget=None):
        """SEMIGLOBAL_AFFINE of pairs `idx` -> (scores, op strings (None for a pair over `trace_budget`))."""
        idx = np.asarray(idx, dtype=np.int64)
        score = np.zeros(len(idx), dtype=np.int64)
        ops = [None] * len(idx)
        sizes = self.trace_bytes(native.PAIR_SEMIGLOBAL_AFFINE, idx)
        for group in _budget_groups(sizes, trace_budget):
            scores, strings = self._launch(native.PAIR_SEMIGLOBAL_AFFINE, idx[group], None, traceback=True)
            self.stats["affine_launches"] += 1
            self.stats["affine_cells"] += int(sum(int(self.q_len[p]) * int(self.r_len[p]) for p in idx[group]))
            for t, g in enumerate(group):
                score[g], ops[g] = scores[t], strings[t]
        return score, ops


def _budget_groups(sizes, budget):
    """Consecutive groups of indices whose sizes sum to at most `budget` (None: one group); an index whose own size
    exceeds the budget is left out of every group."""
    if budget is None:
        return [list(range(len(sizes)))] if len(sizes) else []
    groups, cur, used = [], [], 0
    for i, s in enumerate(sizes):
        if s > budget:
            continue
        if used + s > budget and cur:
            groups.append(cur)
            cur, used = [], 0
        cur.append(i)
        used += s
    if cur:
        groups.append(cur)
    return groups


def align_batch(refs, seqs, device="cuda"):
    """Align every seq (basecall) to its ref on the device in one launch -> list of AlignResult, as the reference's
    align(ref=..., seq=...) computes them from parasail's CIGAR (bonito/cli/evaluate.py:37-67)."""
    raw = sw_align_batch(refs, seqs, device)
    results = []
    for ref, seq, (score, end_q, end_r, n_eq, n_x, n_ins, n_del) in zip(refs, seqs, raw.tolist()):
        if not seq:
            results.append(AlignResult())
            continue
        if score == 0:
            results.append(AlignResult(accuracy=0.0, ref_len=len(ref), seq_len=len(seq)))
            continue
        # the reference drops a leading run of D from the counts; a path traced under these tie rules never starts with
        # a gap, so the run is always empty
        del_start = 0
        n_del -= del_start
        results.append(AlignResult(
            accuracy=n_eq / (n_eq + n_x + n_ins + n_del),
            num_correct=n_eq,
            num_mismatches=n_x,
            num_insertions=n_ins,
            num_deletions=n_del,
            ref_len=len(ref),
            seq_len=len(seq),
            align_ref_start=end_r - n_eq - n_x - n_del + 1,
            align_ref_end=end_r,
            align_seq_start=end_q - n_eq - n_x - n_ins + 1,
            align_seq_end=end_q,
        ))
    return results
