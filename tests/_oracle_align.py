"""
CPU oracle of b200_sw_align: Gotoh local alignment with full H / E / F matrices (numpy, vectorised over anti-diagonals)
and an explicit traceback under the tie rules of bonito_b200/csrc/align.cu.  The counts come from the CIGAR the traceback
writes, so agreement with the kernel (which carries the counts forward instead) also checks that argument.
"""
import re

import numpy as np

MATCH, MISMATCH, OPEN, EXTEND = 5, -4, 8, 4
NEG = -(1 << 29)


def matrices(q, r):
    """H, E, F as int64 [(m + 1), (n + 1)] arrays; rows are query bases, columns reference bases."""
    qa = np.frombuffer(q.encode(), dtype=np.uint8)
    ra = np.frombuffer(r.encode(), dtype=np.uint8)
    m, n = len(qa), len(ra)
    H = np.zeros((m + 1, n + 1), dtype=np.int64)
    E = np.full((m + 1, n + 1), NEG, dtype=np.int64)
    F = np.full((m + 1, n + 1), NEG, dtype=np.int64)
    for d in range(2, m + n + 1):
        i = np.arange(max(1, d - n), min(m, d - 1) + 1)
        if i.size == 0:
            continue
        j = d - i
        E[i, j] = np.maximum(H[i, j - 1] - OPEN, E[i, j - 1] - EXTEND)
        F[i, j] = np.maximum(H[i - 1, j] - OPEN, F[i - 1, j] - EXTEND)
        s = np.where(qa[i - 1] == ra[j - 1], MATCH, MISMATCH)
        H[i, j] = np.maximum.reduce([np.zeros_like(i), H[i - 1, j - 1] + s, E[i, j], F[i, j]])
    return H, E, F


def align(q, r):
    """-> dict(score, end_query, end_ref, cigar, n_eq, n_x, n_ins, n_del); score 0 gives ends -1 and an empty CIGAR."""
    m, n = len(q), len(r)
    if m == 0 or n == 0:
        return dict(score=0, end_query=-1, end_ref=-1, cigar="", n_eq=0, n_x=0, n_ins=0, n_del=0)
    H, E, F = matrices(q, r)
    flat = int(np.argmax(H[1:, 1:]))              # first maximum in query-major order
    i, j = divmod(flat, n)
    i, j = i + 1, j + 1
    score = int(H[i, j])
    if score == 0:
        return dict(score=0, end_query=-1, end_ref=-1, cigar="", n_eq=0, n_x=0, n_ins=0, n_del=0)
    end_query, end_ref = i - 1, j - 1
    ops, state = [], "H"
    while True:
        if state == "H":
            h = H[i, j]
            if h == 0:
                break
            same = q[i - 1] == r[j - 1]
            if h == H[i - 1, j - 1] + (MATCH if same else MISMATCH):
                ops.append("=" if same else "X")
                i, j = i - 1, j - 1
            elif h == E[i, j]:
                state = "E"
            else:
                assert h == F[i, j]
                state = "F"
        elif state == "E":
            ops.append("D")
            state = "H" if H[i, j - 1] - OPEN >= E[i, j - 1] - EXTEND else "E"
            j -= 1
        else:
            ops.append("I")
            state = "H" if H[i - 1, j] - OPEN >= F[i - 1, j] - EXTEND else "F"
            i -= 1
    ops.reverse()
    cigar = "".join(f"{len(run.group())}{run.group()[0]}" for run in re.finditer(r"(.)\1*", "".join(ops)))
    counts = {op: 0 for op in "=XID"}
    for cnt, op in re.findall(r"(\d+)([=XID])", cigar):
        counts[op] += int(cnt)
    return dict(score=score, end_query=end_query, end_ref=end_ref, cigar=cigar, n_eq=counts["="], n_x=counts["X"],
                n_ins=counts["I"], n_del=counts["D"])


def as_row(res):
    """The kernel's output row: score, end_query, end_ref, n_eq, n_x, n_ins, n_del."""
    return [res[k] for k in ("score", "end_query", "end_ref", "n_eq", "n_x", "n_ins", "n_del")]


def align_result_fields(ref, seq):
    """The AlignResult fields the reference's formulas give from this oracle's CIGAR (bonito/cli/evaluate.py:37-67), with
    the score-0 rule of bonito_b200.align."""
    from bonito_b200.align import AlignResult
    if not seq:
        return AlignResult()
    res = align(seq, ref)
    if res["score"] == 0:
        return AlignResult(accuracy=0.0, ref_len=len(ref), seq_len=len(seq))
    lead = re.match(r"^(\d+)D", res["cigar"])
    n_del = res["n_del"] - (int(lead.group(1)) if lead else 0)
    eq, x, ins = res["n_eq"], res["n_x"], res["n_ins"]
    return AlignResult(accuracy=eq / (eq + x + ins + n_del), num_correct=eq, num_mismatches=x, num_insertions=ins,
                       num_deletions=n_del, ref_len=len(ref), seq_len=len(seq),
                       align_ref_start=res["end_ref"] - eq - x - n_del + 1, align_ref_end=res["end_ref"],
                       align_seq_start=res["end_query"] - eq - x - ins + 1, align_seq_end=res["end_query"])
