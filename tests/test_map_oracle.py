"""CPU checks of the mapping rules: the oracle (tests/_oracle_map.py) against brute-force definitions, FASTA parsing,
presets, MAPQ, CIGAR / NM / MD and the aligned SAM record and header (bonito_b200.aligner, bonito_b200.io)."""
import gzip
import random

import numpy as np
import pytest

import _oracle_map as O
from bonito_b200 import aligner as A
from bonito_b200.io import sam_header, sam_record


def _rand(rng, n, alphabet="ACGT"):
    return "".join(rng.choice(alphabet) for _ in range(n)).encode()


# ------------------------------------------------------------------------------------------------ minimizers
def _brute_minimizers(seq, k, w):
    """Every window, every k-mer, the canonical code and hash from the definitions."""
    comp = {"A": "T", "C": "G", "G": "C", "T": "A"}
    code = {"A": 0, "C": 1, "G": 2, "T": 3}
    s = seq.decode()
    keys = []
    for p in range(len(s) - k + 1):
        kmer = s[p:p + k]
        if any(c not in code for c in kmer):
            keys.append(None)
            continue
        fwd = sum(code[c] << 2 * (k - 1 - t) for t, c in enumerate(kmer))
        rc = "".join(comp[c] for c in reversed(kmer))
        rev = sum(code[c] << 2 * (k - 1 - t) for t, c in enumerate(rc))
        keys.append((O.hash64(min(fwd, rev), (1 << 2 * k) - 1), int(fwd > rev)))
    found = {}
    for st in range(len(keys) - w + 1):
        best = None
        for p in range(st, st + w):
            if keys[p] is not None and (best is None or keys[p][0] < keys[best][0]):
                best = p
        if best is not None:
            found[best] = keys[best][0] << 1 | keys[best][1]
    return sorted(found.items())


@pytest.mark.parametrize("k,w", [(19, 19), (15, 10), (5, 3)])
def test_minimizers_are_the_exhaustive_window_minima(k, w):
    rng = random.Random(k * 100 + w)
    for n in (0, k - 1, k + w - 2, k + w - 1, 200, 600):
        seq = bytearray(_rand(rng, n))
        if n >= 200:
            seq[50:70] = b"N" * 20                  # an N run breaks every k-mer over it
            seq[120:121] = b"n"
        assert O.minimizers(bytes(seq), k, w) == _brute_minimizers(bytes(seq), k, w), n
    assert O.minimizers(_rand(rng, k + w - 2), k, w) == []      # shorter than one window


def test_low_complexity_ties_go_left():
    seq = b"A" * 60
    got = O.minimizers(seq, 5, 4)
    assert got == _brute_minimizers(seq, 5, 4)
    assert [p for p, _ in got] == list(range(0, 60 - 5 - 4 + 2))   # one tie per window: its first k-mer


# ------------------------------------------------------------------------------------------------ chaining
def test_hand_built_chain():
    k = 15
    # strand 0 anchors (s, r, q) of one contig: a colinear run, one off-diagonal decoy, one too far away
    anc = [(0, 100, 10), (0, 130, 40), (0, 160, 72), (0, 165, 20), (0, 30000, 100)]
    anc.sort(key=lambda a: (a[0], a[1]))
    f, pred = O.chain_dp(anc, np.array([0, 100000]), k)
    # anchor 1: 15 + (15 + min(30, 30, 15) - gamma(0)) = 45; anchor 2: dq 32, dr 30, gamma(2) = 0 + 0 -> 15 + 45 + 15 = 75
    assert f[:3] == [15, 45, 75] and pred[:3] == [-1, 0, 1]
    # the decoy (r 165, q 20) can only follow anchor 0: dq 10, dr 65 -> 15 + 10 - (15 * 55 // 100 + 5 // 2) = 15
    assert f[3] == 30 and pred[3] == 0
    assert f[4] == 15 and pred[4] == -1                          # dr > 10000
    ch = O.extract(anc, f, pred, 200, k)
    # the decoy's chain stops at the taken anchor 0: 30 - 15; its span [20, 35) lies inside the primary's [10, 87)
    assert ch["n"] == 3 and ch["f1"] == 75 and ch["f2"] == 15 and ch["chain"] == [(10, 100), (40, 130), (72, 160)]
    assert ch["W"] == 64 + 2
    # a contig boundary between two anchors cuts the chain
    f, pred = O.chain_dp(anc, np.array([0, 120, 100000]), k)
    assert pred[1] == -1


def test_chain_ties_go_to_the_nearest_predecessor():
    k = 15
    anc = [(0, 100, 0), (0, 100, 0), (0, 140, 40)]      # two identical predecessors
    f, pred = O.chain_dp(anc, np.array([0, 1000]), k)
    assert pred[2] == 1


def test_mapq():
    assert A.mapq(100, 100, 20) == 0 and A.mapq(100, 150, 20) == 0
    assert A.mapq(1000, 0, 50) == 60
    assert A.mapq(100, 50, 5) == int(np.floor(40 * 0.5 * 0.5 * np.log(100)))
    assert O.mapq(321, 17, 7) == A.mapq(321, 17, 7)


# ------------------------------------------------------------------------------------------------ alignment
def _brute_local(q, t, allowed):
    """Full (m+1) x (n+1) matrices of the local affine recurrences with the band as a mask."""
    m, n = len(q), len(t)
    NEG = O.NEG
    H = [[0] * (n + 1) for _ in range(m + 1)]
    E = [[NEG] * (n + 1) for _ in range(m + 1)]
    F = [[NEG] * (n + 1) for _ in range(m + 1)]
    S = [[0] * (n + 1) for _ in range(m + 1)]
    EO = [[False] * (n + 1) for _ in range(m + 1)]
    FO = [[False] * (n + 1) for _ in range(m + 1)]
    best = (0, 0, 0)
    for i in range(1, m + 1):
        for j in range(1, n + 1):
            if not allowed(i, j):
                H[i][j] = E[i][j] = F[i][j] = NEG
                continue
            EO[i][j] = H[i][j - 1] - 6 >= E[i][j - 1] - 2
            E[i][j] = max(H[i][j - 1] - 6, E[i][j - 1] - 2)
            FO[i][j] = H[i - 1][j] - 6 >= F[i - 1][j] - 2
            F[i][j] = max(H[i - 1][j] - 6, F[i - 1][j] - 2)
            a, b = chr(q[i - 1]), chr(t[j - 1])
            s = -1 if a not in "ACGT" or b not in "ACGT" else (2 if a == b else -4)
            d = H[i - 1][j - 1] + s
            m3 = max(d, E[i][j], F[i][j])
            if m3 <= 0:
                H[i][j], S[i][j] = 0, 1
            else:
                H[i][j], S[i][j] = m3, 0 if m3 == d else (3 if m3 == E[i][j] else 2)
            if H[i][j] > 0 and (H[i][j], i, j) > best:
                best = (H[i][j], i, j)
    score, i, j = best
    if not score:
        return 0, 0, 0, 0, 0, b""
    ops, state, ei, ej = [], 0, i, j
    while i > 0 and j > 0:
        if state == 0:
            if S[i][j] == 1:
                break
            if S[i][j] == 0:
                ops.append(b"=" if q[i - 1] == t[j - 1] and chr(q[i - 1]) in "ACGT" else b"X")
                i, j = i - 1, j - 1
            else:
                state = 1 if S[i][j] == 3 else 2
        elif state == 1:
            ops.append(b"D")
            state = 0 if EO[i][j] else 1
            j -= 1
        else:
            ops.append(b"I")
            state = 0 if FO[i][j] else 2
            i -= 1
    return score, i, ei, j, ej, b"".join(ops[::-1])


def _mutate(rng, s, sub, ins, dele):
    out = bytearray()
    for c in s:
        x = rng.random()
        if x < dele:
            continue
        if x < dele + sub:
            out += rng.choice([b for b in b"ACGT" if b != c]).to_bytes(1, "little")
        else:
            out.append(c)
        if rng.random() < ins:
            out += rng.choice(b"ACGT").to_bytes(1, "little")
    return bytes(out)


@pytest.mark.parametrize("seed", range(6))
def test_band_align_equals_full_matrix(seed):
    rng = random.Random(seed)
    t = bytearray(_rand(rng, rng.randint(30, 70)))
    q = bytearray(_mutate(rng, bytes(t[5:-5]), 0.08, 0.05, 0.05))
    if seed % 2:
        q[3:6] = b"NNN"
        t[20:22] = b"NN"
    q = bytes(rng.choice([b"", _rand(rng, 4)])) + bytes(q)
    chain = [(2, 7), (len(q) - 3, len(t) - 8)] if seed % 3 else [(0, 0), (len(q) - 1, len(t) - 1)]
    for W in (3, 6, 200):
        got = O.band_align(q, t, chain, W)
        cen = O.centres(chain, len(q))
        want = _brute_local(q, bytes(t), lambda i, j: 0 <= j - (cen[i - 1] + 1 - W) <= 2 * W)
        assert got == want, (seed, W)


@pytest.mark.parametrize("W", [0, 1, 5, 16])
def test_band_align_equals_full_matrix_at_band_edges(W):
    """First rows whose band starts at column 0, 1 or 2, a steep chain segment (the centre jumps by more than 2W + 1), a
    flat one, and query overhangs that leave whole rows outside the target."""
    rng = random.Random(100 + W)
    t = _rand(rng, 60)
    cases = [(t[:40], t[:50], [(0, 0), (39, 39)]), (t[W:W + 30], t, [(0, W), (29, W + 29)]),
             (t[W + 1:W + 31], t, [(0, W + 1), (29, W + 30)]),
             (t[:15] + t[45:60], t, [(0, 0), (14, 14), (15, 45), (29, 59)]),
             (t[:10] + _rand(rng, 20) + t[10:25], t[:25], [(0, 0), (9, 9), (30, 10), (44, 24)]),
             (_rand(rng, 12) + t[:30] + _rand(rng, 12), t[:30], [(12, 0), (41, 29)])]
    for q, tt, chain in cases:
        cen = O.centres(chain, len(q))
        want = _brute_local(q, tt, lambda i, j: 0 <= j - (cen[i - 1] + 1 - W) <= 2 * W)
        assert O.band_align(q, tt, chain, W) == want, (W, chain)


def test_band_align_zero_score():
    assert O.band_align(b"AAAA", b"CCCC", [(0, 0), (3, 3)], 4) == (0, 0, 0, 0, 0, b"")


# ------------------------------------------------------------------------------------------------ CIGAR / NM / MD
def test_cigar_nm_md_product_equals_oracle():
    rng = random.Random(5)
    for _ in range(200):
        n = rng.randint(1, 60)
        ops = bytes(rng.choice(b"==========XID") for _ in range(n))
        ref = _rand(rng, sum(o != ord("I") for o in ops))
        assert A.cigar_nm_md(np.frombuffer(ops, np.uint8), np.frombuffer(ref, np.uint8)) == O.cigar_nm_md(ops, ref)
    assert O.cigar_nm_md(b"==X=DD=I==", b"ACGTAC" + b"GAC") == ("4M2D1M1I2M", 4, "2G1^AC3")
    assert O.cigar_nm_md(b"XDD=", b"ACGT") == ("1M2D1M", 3, "0A0^CG1")


# ------------------------------------------------------------------------------------------------ FASTA
def test_fasta_parsing(tmp_path):
    fa = tmp_path / "ref.fa"
    fa.write_bytes(b">chr1 first contig\nACGTacgt\nNNRY\n\n>chr2\nggcc\n>empty\n\n>chr3\tx\nA\n")
    contigs = A.read_fasta(str(fa))
    assert [(n, s.tobytes()) for n, s in contigs] == [("chr1", b"ACGTACGTNNNN"), ("chr2", b"GGCC"), ("chr3", b"A")]
    gz = tmp_path / "ref.fa.gz"
    gz.write_bytes(gzip.compress(fa.read_bytes()))
    assert [(n, s.tobytes()) for n, s in A.read_fasta(str(gz))] == [(n, s.tobytes()) for n, s in contigs]
    crlf = tmp_path / "crlf.fa"
    crlf.write_bytes(b">a\r\nAC\r\nGT\r\n")
    assert [(n, s.tobytes()) for n, s in A.read_fasta(str(crlf))] == [("a", b"ACGT")]
    for name, data in (("e.fa", b""), ("h.fa", b">only\n\n"), ("x.fa", b"ACGT\n"), ("i.mmi", b"MMI\x02")):
        (tmp_path / name).write_bytes(data)
        with pytest.raises(A.IndexBuildError):
            A.read_fasta(str(tmp_path / name))
    with pytest.raises(A.IndexBuildError):
        A.read_fasta(str(tmp_path / "missing.fa"))


def test_presets():
    assert A.PRESETS == {"lr:hq": (19, 19), "map-ont": (15, 10)}
    assert all(k % 2 for k, _ in A.PRESETS.values())
    with pytest.raises(ValueError, match="preset"):
        A.Aligner("unused.fa", preset="sr")


# ------------------------------------------------------------------------------------------------ SAM
def _md_check(rec, contig):
    """NM / MD of a SAM line recomputed from its CIGAR, SEQ and the contig."""
    import re
    f = rec.split("\t")
    cigar, seq, pos = f[5], f[9].encode(), int(f[3]) - 1
    clips = re.findall(r"(\d+)S", cigar)
    lead = int(cigar.split("S")[0]) if re.match(r"^\d+S", cigar) else 0
    core = re.sub(r"\d+S", "", cigar)
    tail = int(clips[-1]) if cigar.endswith("S") else 0
    span = sum(int(n) for n, op in re.findall(r"(\d+)([MD])", core))
    nm, md = O.nm_md_from_cigar(core, seq[lead:len(seq) - tail], contig[pos:pos + span])
    return f"NM:i:{nm}" in f and f"MD:Z:{md}" in f


def test_sam_record_both_strands():
    contig = b"TTTTACGTACGAACGTTTTT"
    read = "GGACGTACGAACGTCC"                      # clips GG / CC around ACGTACGAACGT = contig[4:16]
    fwd = A.Mapping("c1", 4, 16, 2, 14, 1, 60, "12M", 0, "12")
    rec = sam_record("r", read, "ABCDEFGHIJKLMNOP", fwd, tags=["qs:i:9"])
    assert rec.split("\t") == ["r", "0", "c1", "5", "60", "2S12M2S", "*", "0", "0", read, "ABCDEFGHIJKLMNOP", "NM:i:0",
                               "MD:Z:12", "qs:i:9"]
    assert _md_check(rec, contig)
    # reverse strand: the read is the reverse complement of GGG + contig[4:16] with one mismatch + C
    core = bytearray(contig[4:16])
    core[5] = ord("T")                             # contig has C at 9
    rc_read = A.revcomp("GGG" + core.decode() + "C")
    # in the read's own orientation the leading clip is the 1 C-complement base, the trailing clip the 3 G's
    rev = A.Mapping("c1", 4, 16, 1, 13, -1, 7, "12M", 1, "5C6")
    rec = sam_record("r2", rc_read, "0123456789abcdef", rev)
    f = rec.split("\t")
    assert f[1] == "16" and f[5] == "3S12M1S" and f[9] == "GGG" + core.decode() + "C" and f[10] == "fedcba9876543210"
    assert _md_check(rec, contig)
    assert sam_record("u", "ACGT", "5555", None, tags=["qs:i:20"]) == \
        "u\t4\t*\t0\t0\t*\t*\t0\t0\tACGT\t5555\tNM:i:0\tqs:i:20"


def test_sam_header():
    plain = sam_header(["@RG\tID:x"], argv=["a", "b"])
    assert plain == ("@HD\tVN:1.5\tSO:unknown\tob:0.0.2\n"
                     "@PG\tID:basecaller\tPN:bonito_b200\tVN:0.2.0\tCL:bonito_b200 a b\n@RG\tID:x\n")
    assert sam_header(["@RG\tID:x"], argv=["a", "b"], contigs=None) == plain
    lines = sam_header(["@RG\tID:x"], argv=["a"], contigs=[("chr1", 100), ("chr2", 7)]).splitlines()
    assert lines[0].startswith("@HD") and lines[1:3] == ["@SQ\tSN:chr1\tLN:100", "@SQ\tSN:chr2\tLN:7"]
    assert lines[3].startswith("@PG\tID:basecaller") and lines[4].startswith("@PG\tID:aligner") and lines[5] == "@RG\tID:x"


# ------------------------------------------------------------------------------------------------ whole rule chain
def test_oracle_maps_a_planted_read():
    rng = random.Random(11)
    contigs = [("a", _rand(rng, 6000)), ("b", _rand(rng, 3000))]
    index = O.Index(contigs, 15, 10)
    read = _mutate(rng, contigs[0][1][1000:2500], 0.02, 0.01, 0.01)
    m = O.map_read(index, read)
    assert m[0] == "a" and m[5] == 1 and abs(m[1] - 1000) < 20 and m[6] > 0
    m = O.map_read(index, O.revcomp(read))
    assert m[0] == "a" and m[5] == -1 and abs(m[1] - 1000) < 20
    assert O.map_read(index, _rand(rng, 1500)) is None
    assert O.map_read(index, contigs[1][1][:20]) is None           # shorter than k + w - 1: no minimizers
