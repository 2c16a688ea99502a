"""
Write tests/golden/duplex_pairs.npz: seeded synthetic (template, complement) read pairs and the consensus the reference's
own `call_basespace_duplex` (bonito/cli/duplex.py) computes for them, with the CPU alignment oracle standing in for edlib
and parasail (tests/_reference_duplex.py).  Needs the reference checkout; run from the repository root:

    python scripts/make_golden_duplex.py

The pairs cover: no long match at all (the whole pair re-aligned), prefix and suffix re-alignment, a suffix that depends on
the re-aligned prefix, homopolymer-rich reads, equal qualities on both strands (the template wins every tie), and reads
that trim to nothing.  Arrays: ids (template, complement), sequences and Q-value qualities concatenated with offsets,
and the expected consensus sequence / qstring per pair.
"""
import os
import random
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import _reference_duplex as R  # noqa: E402
from bonito_b200 import duplex as D  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "duplex_pairs.npz")


def rand(rng, n, alphabet="ACGT"):
    return "".join(rng.choice(alphabet) for _ in range(n))


def mutate(rng, s, sub, ins, dele):
    out = []
    for c in s:
        x = rng.random()
        if x < sub:
            out.append(rng.choice([b for b in "ACGT" if b != c]))
        elif x < sub + ins:
            out.append(c)
            out.append(rng.choice("ACGT"))
        elif x >= sub + ins + dele:
            out.append(c)
    return "".join(out)


def homopolymers(rng, n):
    out = []
    while len(out) < n:
        out.extend(rng.choice("ACGT") * rng.randint(1, 7))
    return "".join(out[:n])


def quals(rng, n, lo=2, hi=40):
    return np.array([rng.randint(lo, hi) for _ in range(n)], dtype=np.uint8)


def make_pairs(seed=11):
    rng = random.Random(seed)
    pairs = []                                      # (kind, template, complement as sequenced, tq, cq)

    def add(kind, t, c_fwd, tq=None, cq=None):
        c = D.revcomp(c_fwd)
        pairs.append((kind, t, c, quals(rng, len(t)) if tq is None else tq, quals(rng, len(c)) if cq is None else cq))

    for _ in range(4):                              # ordinary pairs
        truth = rand(rng, rng.randint(200, 700))
        add("plain", mutate(rng, truth, .03, .02, .02), mutate(rng, truth, .03, .02, .02))
    for _ in range(3):                              # unrelated flanks: prefix and suffix re-alignment
        truth = rand(rng, rng.randint(200, 500))
        add("flanks", rand(rng, rng.randint(5, 30)) + mutate(rng, truth, .03, .01, .01) + rand(rng, rng.randint(5, 30)),
            rand(rng, rng.randint(5, 30)) + mutate(rng, truth, .03, .01, .01) + rand(rng, rng.randint(5, 30)))
    for _ in range(2):                              # one long match only, after noise: the suffix depends on the prefix
        core = rand(rng, 14)
        add("one_match", rand(rng, 25) + core + mutate(rng, rand(rng, 40), 0, 0, 0),
            rand(rng, 22) + core + rand(rng, 37))
    for _ in range(2):                              # no long match anywhere: the whole pair re-aligned
        truth = rand(rng, 60)
        add("no_match", mutate(rng, truth, .3, .05, .05), mutate(rng, truth, .3, .05, .05))
    for _ in range(4):                              # homopolymer-rich
        truth = homopolymers(rng, rng.randint(150, 500))
        add("homopolymer", mutate(rng, truth, .02, .03, .03), mutate(rng, truth, .02, .03, .03))
    for _ in range(3):                              # equal qualities: the template wins every tie
        truth = rand(rng, rng.randint(150, 400))
        t, c = mutate(rng, truth, .04, .02, .02), mutate(rng, truth, .04, .02, .02)
        q = rng.randint(5, 30)
        add("quality_ties", t, c, np.full(len(t), q, np.uint8), np.full(len(c), q, np.uint8))
    for _ in range(2):                              # high divergence and a length difference
        truth = rand(rng, rng.randint(300, 600))
        add("divergent", mutate(rng, truth, .08, .06, .02), mutate(rng, truth[40:], .08, .02, .06))
    return pairs


def paths(t, tq, c, cq):
    """Which re-alignments the pair takes: (first long match index, last long match index from the end, long matches)."""
    import _oracle_duplex as O
    prep = D.prepare(t, tq, c, cq)
    rs = D.runs(O.global_edit(prep[0], prep[2])[1])
    return D.first_long(rs), D.last_long(rs), sum(D._long(r) for r in rs)


def main():
    ref = R.load_duplex()
    pairs = make_pairs()
    kinds, t_ids, c_ids, seqs, qs, cons, cons_q = [], [], [], [], [], [], []
    seen = set()
    for n, (kind, t, c, tq, cq) in enumerate(pairs):
        seq, qstring = ref.call_basespace_duplex(t, tq, c, cq)
        f, b, n_long = paths(t, tq, c, cq)
        seen.update({"full" if f is None else None, "prefix" if f else None, "suffix" if b else None,
                     "dependent" if f and n_long == 1 else None})
        kinds.append(kind)
        t_ids.append(f"read{2 * n:03d}")
        c_ids.append(f"read{2 * n + 1:03d}")
        seqs += [t, c]
        qs += [tq, cq]
        cons.append(seq)
        cons_q.append(qstring)
        print(f"{kind:13s} {len(t):4d} {len(c):4d} -> {len(seq):4d}  first {f} last {b} long {n_long}")
    missing = {"full", "prefix", "suffix", "dependent"} - seen
    assert not missing, f"no pair takes the {missing} path"
    lens = np.array([len(s) for s in seqs], dtype=np.int64)
    np.savez_compressed(
        OUT, kinds=np.array(kinds), temp_ids=np.array(t_ids), comp_ids=np.array(c_ids),
        seq_data=np.frombuffer("".join(seqs).encode(), dtype=np.uint8), qual_data=np.concatenate(qs), lengths=lens,
        consensus=np.array(cons, dtype=object).astype(str), consensus_q=np.array(cons_q, dtype=object).astype(str))
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes, {len(pairs)} pairs)")


if __name__ == "__main__":
    main()
