"""
ORACLE -- TEST INFRASTRUCTURE ONLY.  The CTC prefix beam search of `bonito_b200` (rules in bonito_b200/csrc/ctc_beam.cu)
as plain loops over dicts, float64 sums, written from the definition and not from the kernel (a prefix is a record
(parent, label, frame) in a list, so that reads of thousands of frames stay cheap to hash):

  * `class_probs(logp)`      p[t][c] = exp(logp[t][c]) rounded to fp32, the one rounding the definition prescribes;
  * `beam_search(logp, ...)`  -> (sequence str, qstring str, moves uint8 [T]);
  * `ctc_log_prob(logp, labels)`       log P(labels | logp) by the CTC forward algorithm in the log domain;
  * `most_probable_sequence(logp)`     brute force over every label sequence, for T <= 6.

A prefix is identified by its labels AND the frames at which they entered the beam: a prefix that was dropped and is
proposed again later is a new record, and descendants of the dropped one that are still in the beam are not its children.
"""
import itertools

import numpy as np


def class_probs(logp):
    return np.exp(np.asarray(logp).astype(np.float64)).astype(np.float32)


def argmax_high(row):
    """Index of the largest value; equal values: the highest index."""
    row = [float(v) for v in row]
    return max(i for i in range(len(row)) if row[i] == max(row))


def phred(p, qscale=1.0, qbias=0.0):
    q = np.rint(-10.0 * np.log10(max(1.0 - p, 1e-4)) * qscale + qbias) + 33
    return chr(int(min(max(q, 33), 126)))


def search(logp, beam_width=5, threshold=1e-3):
    """The top prefix after the last frame: (labels tuple, frames tuple)."""
    probs = class_probs(logp)
    cut = np.float32(threshold)
    prefixes = [(None, 0, -1)]                      # id -> (parent id, label, frame at which it entered the beam)
    beam = [(0, 0.0, 1.0)]                          # (prefix id, p_label, p_blank), by rank
    for t in range(len(probs)):
        p = probs[t]
        alive = [c for c in range(len(p)) if not p[c] < cut]
        if not alive:
            continue
        rank_of = {pid: rank for rank, (pid, _, _) in enumerate(beam)}
        in_beam = {prefixes[pid][:2]: pid for pid in rank_of}            # (parent id, label) -> prefix id
        cand = {}                                   # prefix id, or (parent id, label) of a new one -> [p_label, p_blank, order]

        def propose(key, order, d_label, d_blank):
            entry = cand.setdefault(key, [0.0, 0.0, order])
            entry[0] += d_label
            entry[1] += d_blank

        for rank, (pid, pl, pb) in enumerate(beam):
            last = prefixes[pid][1]
            for c in alive:
                pc = float(p[c])
                if c == 0:
                    propose(pid, (rank, 0), 0.0, (pl + pb) * pc)
                    continue
                if last == c:
                    propose(pid, (rank, 0), pl * pc, 0.0)
                    mass = pb * pc
                else:
                    mass = (pl + pb) * pc
                kin = in_beam.get((pid, c))         # the child is an entry of the beam already: it is that entry
                if kin is not None:
                    propose(kin, (rank_of[kin], 0), mass, 0.0)
                else:
                    propose((pid, c), (rank, c), mass, 0.0)
        ranked = sorted((kv for kv in cand.items() if kv[1][0] + kv[1][1] > 0),
                        key=lambda kv: (-(kv[1][0] + kv[1][1]), kv[1][2]))[:beam_width]
        if not ranked:
            continue
        top = ranked[0][1][0] + ranked[0][1][1]
        beam = []
        for key, (pl, pb, _) in ranked:
            if isinstance(key, tuple):              # a new prefix enters the beam at this frame
                prefixes.append((key[0], key[1], t))
                key = len(prefixes) - 1
            beam.append((key, pl / top, pb / top))
    labels, frames = [], []
    pid = beam[0][0]
    while pid:
        pid, lab, frame = prefixes[pid]
        labels.append(lab)
        frames.append(frame)
    return tuple(labels[::-1]), tuple(frames[::-1])


def beam_search(logp, beam_width=5, threshold=1e-3, alphabet="NACGT", qscale=1.0, qbias=0.0):
    logp = np.asarray(logp)
    T = len(logp)
    labels, frames = search(logp, beam_width, threshold)
    probs = class_probs(logp)
    moves = np.zeros(T, dtype=np.uint8)
    qual = []
    for i, (lab, start) in enumerate(zip(labels, frames)):
        moves[start] = 1
        end = frames[i + 1] if i + 1 < len(frames) else T
        vals = [float(probs[u][lab]) for u in range(start, end) if argmax_high(logp[u]) == lab]
        if not vals:
            vals = [float(probs[start][lab])]
        total = 0.0
        for v in vals:
            total += v
        qual.append(phred(total / len(vals), qscale, qbias))
    return "".join(alphabet[c] for c in labels), "".join(qual), moves


def ctc_log_prob(logp, labels):
    """log of the summed probability of every alignment of `labels` (a sequence of classes 1..4), from class_probs."""
    with np.errstate(divide="ignore"):
        lp = np.log(class_probs(logp).astype(np.float64))
    ext = [0]
    for c in labels:
        ext += [int(c), 0]
    alpha = np.full(len(ext), -np.inf)
    alpha[0] = 0.0                                  # before the first frame: in the leading blank, nothing emitted
    first = True
    for row in lp:
        new = np.full(len(ext), -np.inf)
        for s, c in enumerate(ext):
            if first:
                a = 0.0 if s <= 1 else -np.inf
            else:
                a = alpha[s]
                if s >= 1:
                    a = np.logaddexp(a, alpha[s - 1])
                if s >= 2 and c != 0 and ext[s - 2] != c:
                    a = np.logaddexp(a, alpha[s - 2])
            new[s] = a + row[c]
        alpha, first = new, False
    if first:
        return 0.0 if not labels else -np.inf
    return float(np.logaddexp(alpha[-1], alpha[-2]) if len(ext) > 1 else alpha[-1])


def most_probable_sequence(logp):
    """(best labels, its log-prob, the runner-up's log-prob) over every sequence of up to T labels; T <= 6."""
    T = len(logp)
    assert T <= 6
    scored = []
    for n in range(T + 1):
        for labels in itertools.product((1, 2, 3, 4), repeat=n):
            scored.append((ctc_log_prob(logp, labels), labels))
    scored.sort(key=lambda x: -x[0])
    return scored[0][1], scored[0][0], scored[1][0]
