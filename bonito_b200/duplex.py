"""
Base-space duplex consensus, the per-pair logic of the reference's `bonito duplex` (bonito/cli/duplex.py:109-301)
restated from its behaviour, with the alignments batched on the GPU (bonito_b200.align.PairAligner, b200_pair_align):

  1. each strand's qualities are shifted (+1 template, -1 complement, edge padded), min-pooled over 5 (edge padded) and
     every homopolymer run of 2 or more is set to its float32 mean; then the complement is reverse-complemented and its
     qualities reversed;
  2. the template is aligned to the reverse complement with GLOBAL_EDIT (for edlib); the ops before the first '=' run of
     11 or more, through that run, are re-aligned with SEMIGLOBAL_AFFINE (for parasail) and spliced in front of the rest,
     then the same from the end with the last such run; with no such run the whole pair is re-aligned;
  3. the ops are trimmed to the first and last '=' run of 11 or more, and the sequences and qualities with them;
  4. the consensus takes, column by column, the base of the strand with the higher quality (the template on a tie), with
     the sum of the qualities where the bases agree; gap columns are dropped.

Deviations: alignment ties follow this project's rules (bonito_b200/csrc/pair_align.cu), not edlib's or parasail's; a
pair whose traceback alone needs more than TRACE_BUDGET bytes gets an empty consensus (the reference would align it);
empty reads give an empty consensus (the reference raises).
"""

import numpy as np

MIN_LONG_MATCH = 11
TRACE_BUDGET = 8 << 30          # bytes of traceback bits per GPU launch (GLOBAL_EDIT and SEMIGLOBAL_AFFINE alike)

_COMPLEMENT = str.maketrans("ACGTacgt", "TGCAtgca")


def revcomp(seq):
    return seq.translate(_COMPLEMENT)[::-1]


def adjust_qscores(qscores, seq, shift, window=5):
    """Shift by `shift` with edge padding, min-pool over `window` with edge padding, then the float32 mean over every
    homopolymer run of 2 or more bases of `seq` -> float32 array."""
    q = np.asarray(qscores, dtype=np.uint8)
    if shift > 0:
        q = np.concatenate([np.full(shift, q[0], dtype=np.uint8), q[:-shift]])
    elif shift < 0:
        q = np.concatenate([q[-shift:], np.full(-shift, q[-1], dtype=np.uint8)])
    padded = np.pad(q.astype(np.float32), window // 2, mode="edge")
    pooled = np.lib.stride_tricks.sliding_window_view(padded, window).min(axis=1)
    s = np.frombuffer(seq.encode("ascii"), dtype=np.uint8)
    if len(s) < 2:
        return pooled
    starts = np.flatnonzero(np.concatenate([[True], s[1:] != s[:-1]]))
    lengths = np.diff(np.append(starts, len(s)))
    # the pooled values are integers, so the float32 run sums are exact in any order and the correctly rounded quotient
    # is np.mean's float32 result
    means = (np.add.reduceat(pooled, starts).astype(np.float64) / lengths).astype(np.float32)
    return np.where(np.repeat(lengths >= 2, lengths), np.repeat(means, lengths), pooled)


def runs(ops):
    """Op string -> [(op, count)] with maximal runs."""
    if not ops:
        return []
    a = np.frombuffer(ops.encode("ascii"), dtype=np.uint8)
    starts = np.flatnonzero(np.concatenate([[True], a[1:] != a[:-1]]))
    counts = np.diff(np.append(starts, len(a)))
    return [(chr(a[s]), int(c)) for s, c in zip(starts, counts)]


def run_lens(rs):
    """(query bases, target bases) consumed by runs."""
    q = sum(c for op, c in rs if op != "D")
    r = sum(c for op, c in rs if op != "I")
    return q, r


def splice(*parts):
    """Concatenate run lists, merging equal ops where two parts meet."""
    out = []
    for part in parts:
        for op, c in part:
            if c == 0:
                continue
            if out and out[-1][0] == op:
                out[-1] = (op, out[-1][1] + c)
            else:
                out.append((op, c))
    return out


def _long(run):
    return run[0] == "=" and run[1] >= MIN_LONG_MATCH


def first_long(rs):
    return next((i for i, r in enumerate(rs) if _long(r)), None)


def last_long(rs):
    """Index of the last long '=' run counted from the end (0: the last run), or None."""
    return next((i for i, r in enumerate(reversed(rs)) if _long(r)), None)


def trim(rs):
    """Drop the runs before the first and after the last long '=' run -> (runs, q_start, r_start, q_end, r_end)."""
    f, b = first_long(rs), last_long(rs)
    if f is None:
        q, r = run_lens(rs)
        return [], q, r, 0, 0
    head, tail = rs[:f], rs[len(rs) - b:] if b else []
    q_st, r_st = run_lens(head)
    q_en, r_en = run_lens(tail)
    return rs[f:len(rs) - b], q_st, r_st, q_en, r_en


def consensus(rs, temp_seq, temp_q, comp_seq, comp_q):
    """Column-by-column consensus of an alignment (runs) of template and complement -> (sequence, qstring)."""
    ops = np.frombuffer("".join(op * c for op, c in rs).encode("ascii"), dtype=np.uint8)
    is_t, is_c = ops != ord("D"), ops != ord("I")
    gap = np.uint8(ord("-"))
    col_t = np.full(len(ops), gap, dtype=np.uint8)
    col_c = np.full(len(ops), gap, dtype=np.uint8)
    col_t[is_t] = np.frombuffer(temp_seq.encode("ascii"), dtype=np.uint8)
    col_c[is_c] = np.frombuffer(comp_seq.encode("ascii"), dtype=np.uint8)
    # each strand's quality is that of its last consumed base (its first base before any)
    qs = np.stack([temp_q[np.maximum(np.cumsum(is_t) - 1, 0)], comp_q[np.maximum(np.cumsum(is_c) - 1, 0)]])
    pick = qs.argmax(axis=0)                      # a tie picks the template
    cons = np.where(pick, col_c, col_t)
    q = np.where(col_c == col_t, qs.sum(axis=0), qs[pick, np.arange(qs.shape[1])])
    keep = cons != gap
    # rounded after the +33, in float32, as the reference does
    qstring = np.round(np.clip(q[keep], 0, 60) + 33).astype(np.uint8)
    return cons[keep].tobytes().decode("ascii"), qstring.tobytes().decode("ascii")


def prepare(temp_seq, temp_q, comp_seq, comp_q):
    """Step 1: (template, adjusted template qualities, revcomp complement, adjusted and reversed complement qualities)."""
    tq = adjust_qscores(temp_q, temp_seq, shift=1)
    cq = adjust_qscores(comp_q, comp_seq, shift=-1)
    return temp_seq, tq, revcomp(comp_seq), cq[::-1]


def finish(rs, temp_seq, temp_q, comp_seq, comp_q):
    """Steps 3 and 4 on the final alignment runs of a prepared pair."""
    rs, t_st, c_st, t_en, c_en = trim(rs)
    if not rs:
        return "", ""
    return consensus(rs, temp_seq[t_st:len(temp_seq) - t_en], temp_q[t_st:len(temp_q) - t_en],
                     comp_seq[c_st:len(comp_seq) - c_en], comp_q[c_st:len(comp_q) - c_en])


def realign(edit_runs, temp_seqs, comp_seqs, affine):
    """Step 2 after GLOBAL_EDIT: the end re-alignments of every pair.  `affine(list of (query, target))` -> list of op
    strings (None: not aligned) is called at most twice: once for every whole-pair re-alignment, prefix and suffix that
    the GLOBAL_EDIT result fixes, and once for the suffixes that depend on a re-aligned prefix (a pair whose only long
    match is its first).  -> list of runs (None where a re-alignment was not done)."""
    result = list(edit_runs)
    jobs, later = [], []                           # (pair, kind, query, target, cut)

    for p, rs in enumerate(edit_runs):
        if rs is None:
            continue
        t, c = temp_seqs[p], comp_seqs[p]
        f = first_long(rs)
        if f is None:
            jobs.append((p, "full", t, c, None))
            continue
        if f > 0:
            q_st, r_st = run_lens(rs[:f + 1])
            jobs.append((p, "prefix", t[:q_st], c[:r_st], f))
        b = last_long(rs)
        if f > 0 and len(rs) - 1 - b == f:
            later.append(p)                        # the last long match is the re-aligned prefix's
        elif b > 0:
            q_en, r_en = run_lens(rs[-(b + 1):])
            jobs.append((p, "suffix", t[len(t) - q_en:], c[len(c) - r_en:], b))

    def apply(jobs):
        ops = affine([(q, r) for _, _, q, r, _ in jobs]) if jobs else []
        for (p, kind, _, _, cut), o in zip(jobs, ops):
            if result[p] is None:
                continue
            if o is None:
                result[p] = None
            elif kind == "full":
                result[p] = runs(o)
            elif kind == "prefix":
                result[p] = splice(runs(o), result[p][cut + 1:])
            else:
                result[p] = splice(result[p][:len(result[p]) - (cut + 1)], runs(o))

    # prefixes before suffixes of the same pair: a suffix cut counts runs from the end, which a prefix splice keeps
    jobs.sort(key=lambda j: j[1] == "suffix")
    apply(jobs)
    jobs = []
    for p in later:
        rs = result[p]
        if rs is None:
            continue
        b = last_long(rs)
        if b is None:
            jobs.append((p, "full", temp_seqs[p], comp_seqs[p], None))
        elif b > 0:
            q_en, r_en = run_lens(rs[-(b + 1):])
            t, c = temp_seqs[p], comp_seqs[p]
            jobs.append((p, "suffix", t[len(t) - q_en:], c[len(c) - r_en:], b))
    apply(jobs)
    return result


def align_pairs(prepared, device="cuda", k0=None, budget=TRACE_BUDGET, stats=None):
    """Step 2 for a batch of prepared pairs on the GPU -> list of runs (None: over the traceback budget)."""
    from bonito_b200.align import EDIT_BAND0, PairAligner
    if not prepared:
        return []
    temps = [t for t, _, _, _ in prepared]
    comps = [c for _, _, c, _ in prepared]
    aligner = PairAligner(temps, comps, device)
    _, ops, passes = aligner.global_edit(np.arange(len(prepared)), k0=EDIT_BAND0 if k0 is None else k0,
                                         trace_budget=budget)
    edit_runs = [None if o is None else runs(o) for o in ops]

    def affine(pairs):
        sub = PairAligner([q for q, _ in pairs], [r for _, r in pairs], device)
        _, out = sub.semiglobal_affine(np.arange(len(pairs)), trace_budget=budget)
        if stats is not None:
            for key in ("affine_launches", "affine_cells", "affine_ms"):
                stats[key] = stats.get(key, 0) + sub.stats[key]
        return out

    result = realign(edit_runs, temps, comps, affine)
    if stats is not None:
        for key in ("edit_passes", "edit_cells", "edit_ms"):
            stats[key] = stats.get(key, 0) + aligner.stats[key]
        hist = stats.setdefault("pass_histogram", {})
        for n in passes.tolist():
            hist[n] = hist.get(n, 0) + 1
    return result


def call_pairs(pairs, device="cuda", k0=None, budget=TRACE_BUDGET, stats=None):
    """(temp_seq, temp_qscores, comp_seq, comp_qscores) per pair (qualities as uint8 Q values; None for a missing pair)
    -> list of (sequence, qstring); the whole pipeline, synchronously (the CLI overlaps the steps across batches)."""
    prepared = [prepare_pair(p) for p in pairs]
    ok = [i for i, p in enumerate(prepared) if p is not None]
    aligned = align_pairs([prepared[i] for i in ok], device, k0, budget, stats)
    out = [("", "")] * len(pairs)
    for i, rs in zip(ok, aligned):
        out[i] = ("", "") if rs is None else finish(rs, *prepared[i])
    return out


def prepare_pair(pair):
    """`prepare` for one input pair, or None when a read is missing or empty (an empty consensus)."""
    if pair is None:
        return None
    temp_seq, temp_q, comp_seq, comp_q = pair
    if not temp_seq or not comp_seq:
        return None
    return prepare(temp_seq, temp_q, comp_seq, comp_q)
