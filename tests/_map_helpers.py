"""Sequence helpers shared by the mapping tests: random bases, planted errors, reverse complements and FASTA files."""
import numpy as np

import _oracle_map as O

ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)


def _rand(rng, n):
    return ACGT[rng.integers(0, 4, n)]


def _mutate(rng, s, sub, ins, dele):
    """Substitutions, insertions after a base and deletions at the given per-base rates (uint8 ACGT arrays)."""
    code = np.searchsorted(ACGT, s)
    u = rng.random(len(s))
    keep = u >= dele
    subm = keep & (u < dele + sub)
    code[subm] = (code[subm] + rng.integers(1, 4, int(subm.sum()))) % 4
    insm = keep & (rng.random(len(s)) < ins)
    counts = keep.astype(np.int64) + insm
    out = np.repeat(code, counts)
    out[np.cumsum(counts)[insm] - 1] = rng.integers(0, 4, int(insm.sum()))
    return ACGT[out]


def _rc(s):
    return np.frombuffer(O.revcomp(np.asarray(s, dtype=np.uint8).tobytes()), dtype=np.uint8)


def _fasta(path, contigs):
    with open(path, "w") as fh:
        for name, seq in contigs:
            fh.write(f">{name} planted\n")
            s = np.asarray(seq, dtype=np.uint8).tobytes().decode()
            fh.write("\n".join(s[i:i + 70] for i in range(0, len(s), 70)) + "\n")
