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
