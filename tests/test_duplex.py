"""`duplex`: the CPU alignment oracle by hand, the host pipeline against the reference (when its checkout is present) and the
golden fixture, the readers and the CLI surface; on the GPU b200_pair_align against the oracle and the whole subcommand
against the fixture."""
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import _oracle_duplex as O
from bonito_b200 import duplex as D
from bonito_b200.cli import duplex as cli

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "duplex_pairs.npz")


def _cpu_affine(pairs):
    return [O.semiglobal_affine(q, r)[1] for q, r in pairs]


def _cpu_call(t, tq, c, cq):
    prep = D.prepare(t, tq, c, cq)
    rs = D.realign([D.runs(O.global_edit(prep[0], prep[2])[1])], [prep[0]], [prep[2]], _cpu_affine)[0]
    return D.finish(rs, *prep)


def load_golden():
    g = np.load(GOLDEN)
    lens = g["lengths"]
    offs = np.concatenate([[0], np.cumsum(lens)])
    data = g["seq_data"].tobytes().decode()
    seqs = [data[offs[i]:offs[i + 1]] for i in range(len(lens))]
    quals = [g["qual_data"][offs[i]:offs[i + 1]] for i in range(len(lens))]
    pairs = []
    for n, (tid, cid) in enumerate(zip(g["temp_ids"], g["comp_ids"])):
        pairs.append((str(tid), str(cid), seqs[2 * n], quals[2 * n], seqs[2 * n + 1], quals[2 * n + 1],
                      str(g["consensus"][n]), str(g["consensus_q"][n])))
    return pairs


# ------------------------------------------------------------------------------------------------ oracle, by hand
@pytest.mark.parametrize("q,r,want", [
    ("", "", (0, "")),
    ("", "ACG", (3, "DDD")),
    ("ACG", "", (3, "III")),
    ("A", "A", (0, "=")),
    ("A", "C", (1, "X")),
    ("ACGT", "TGCA", (4, "XXXX")),                     # all mismatch: the diagonal wins the ties with I / D
    ("AAAA", "AAA", (1, "I===")),                      # homopolymer indels: see the test below
    ("AAA", "AAAA", (1, "D===")),
    ("ACGTT", "ACGT", (1, "===I=")),                   # the walk matches the last T diagonally, the I goes before it
])
def test_global_edit_oracle_by_hand(q, r, want):
    dist, ops = O.global_edit(q, r)
    assert (dist, ops) == want
    O.check_ops(q, r, ops)
    assert O.edit_cost(ops) == dist


def test_global_edit_homopolymer_tie_rule():
    """Traced from (m, n) with the diagonal preferred, then I, then D: an extra base of a homopolymer is placed at the
    run's start (the walk keeps matching diagonally from the end and takes the gap last)."""
    assert O.global_edit("CAAAG", "CAAG") == (1, "=I===")
    assert O.global_edit("CAAG", "CAAAG") == (1, "=D===")
    assert O.global_edit("AAAA", "AAA") == (1, "I===")


@pytest.mark.parametrize("q,r,want", [
    ("", "", (0, "")),
    ("", "ACG", (0, "DDD")),
    ("ACG", "", (0, "III")),
    ("A", "A", (5, "=")),
    ("A", "C", (0, "ID")),                             # -4 < 0: the free end gaps win; end cell H[1][0]
    ("ACGTACGT", "ACGTACGT", (40, "========")),
    ("TTACGTACGT", "ACGTACGT", (40, "II========")),    # free leading query bases
    ("ACGTACGT", "ACGTACGTGG", (40, "========DD")),    # free trailing target bases
    ("ACGTACGTAC", "ACGTTACGTAC", (40, "===D=======")),   # 10 matches and one gap: 50 - 10
    ("AAAACCCC", "AAAAGGCCCC", (28, "====DD====")),       # a gap of 2: 40 - 10 - 2
])
def test_semiglobal_affine_oracle_by_hand(q, r, want):
    score, ops = O.semiglobal_affine(q, r)
    O.check_ops(q, r, ops)
    assert score == O.affine_score(ops)
    assert (score, ops) == want


def test_oracles_are_optimal_on_random_pairs():
    rng = random.Random(3)
    for _ in range(30):
        q = "".join(rng.choice("ACGT") for _ in range(rng.randint(0, 25)))
        r = "".join(rng.choice("ACGT") for _ in range(rng.randint(0, 25)))
        dist, ops = O.global_edit(q, r)
        O.check_ops(q, r, ops)
        assert O.edit_cost(ops) == dist
        score, ops = O.semiglobal_affine(q, r)
        O.check_ops(q, r, ops)
        assert O.affine_score(ops) == score


# ------------------------------------------------------------------------------------------------ host pipeline
def test_host_helpers():
    assert D.revcomp("AACGTN") == "NACGTT"
    assert D.runs("==XII=") == [("=", 2), ("X", 1), ("I", 2), ("=", 1)] and D.runs("") == []
    assert D.splice([("=", 2), ("I", 1)], [("I", 2), ("=", 3)], []) == [("=", 2), ("I", 3), ("=", 3)]
    rs = [("I", 2), ("=", 11), ("X", 1), ("=", 12), ("D", 3)]
    assert D.first_long(rs) == 1 and D.last_long(rs) == 1
    assert D.trim(rs) == ([("=", 11), ("X", 1), ("=", 12)], 2, 0, 0, 3)
    assert D.trim([("=", 10)])[0] == []
    q = D.adjust_qscores(np.array([10, 20, 30, 40, 50, 60], np.uint8), "ACGTTT", shift=1)
    assert q.dtype == np.float32 and q.tolist() == [10, 10, 10, 20, 20, 20]     # shifted, pooled, TTT averaged
    q = D.adjust_qscores(np.array([10, 20, 30, 40, 50, 60], np.uint8), "ACGTAC", shift=-1)
    assert q.tolist() == [20, 20, 20, 30, 40, 50]


def test_consensus_picks_the_better_strand_and_sums_agreement():
    tq = np.array([10, 10, 30, 10], np.float32)
    cq = np.array([20, 10, 5, 10], np.float32)
    seq, qs = D.consensus([("=", 1), ("X", 1), ("X", 1), ("I", 1)], "AGTC", tq, "ACA", cq)
    # col 0 agree: 10 + 20; col 1 tie 10 / 10 -> template G; col 2 template 30 beats 5; col 3 I: template C (q 10 vs 5)
    assert seq == "AGTC" and [ord(c) - 33 for c in qs] == [30, 10, 30, 10]


def test_golden_fixture_matches_the_cpu_pipeline():
    for tid, cid, t, tq, c, cq, seq, qs in load_golden():
        assert _cpu_call(t, tq, c, cq) == (seq, qs), (tid, cid)


@pytest.mark.skipif(not __import__("_reference_duplex").available(), reason="reference checkout absent")
def test_host_functions_and_pipeline_match_the_reference():
    import _reference_duplex as R
    ref = R.load_duplex()
    rng = random.Random(5)
    for alphabet in ("AACCGT", "AAAAAAAAC"):        # short runs, and runs of 10 to 40
        n = rng.randint(1, 300)
        seq = "".join(rng.choice(alphabet) for _ in range(n))
        q = np.array([rng.randint(0, 50) for _ in range(n)], np.uint8)
        for shift in (1, -1):
            assert np.array_equal(ref.adj_qscores(q, seq, qshift=shift), D.adjust_qscores(q, seq, shift))
    for tid, cid, t, tq, c, cq, seq, qs in load_golden():
        assert ref.call_basespace_duplex(t, tq, c, cq) == (seq, qs) == _cpu_call(t, tq, c, cq)


# ------------------------------------------------------------------------------------------------ readers, CLI
def _write_inputs(tmp_path, pairs, fmt, extra_records=True):
    path = tmp_path / f"reads.{fmt}"
    lines = []
    if fmt == "sam":
        lines.append("@HD\tVN:1.5\tSO:unknown")
    for tid, cid, t, tq, c, cq, *_ in pairs:
        for rid, s, q in ((tid, t, tq), (cid, c, cq)):
            qual = (np.asarray(q, np.uint8) + 33).tobytes().decode()
            if fmt == "sam":
                if extra_records:      # a secondary and a supplementary record of the same id come first
                    lines.append(f"{rid}\t256\t*\t0\t0\t*\t*\t0\t0\tACGT\t!!!!")
                    lines.append(f"{rid}\t2048\t*\t0\t0\t*\t*\t0\t0\tACGT\t!!!!")
                lines.append(f"{rid}\t4\t*\t0\t0\t*\t*\t0\t0\t{s}\t{qual}\tqs:i:20")
                if extra_records:      # a later duplicate primary record is ignored
                    lines.append(f"{rid}\t4\t*\t0\t0\t*\t*\t0\t0\tACGT\t!!!!")
            else:
                lines.append(f"@{rid} qs:i:20\n{s}\n+\n{qual}")
                if extra_records:
                    lines.append(f"@{rid}\nACGT\n+\n!!!!")
    path.write_text("\n".join(lines) + "\n")
    return path


def test_readers_take_the_first_primary_record(tmp_path):
    pairs = [("a", "b", "ACGTT", [1, 2, 3, 4, 5], "GGC", [9, 9, 9], "", "")]
    for fmt in ("sam", "fastq"):
        reads = cli.read_records(str(_write_inputs(tmp_path, pairs, fmt)))
        assert reads["a"][0] == "ACGTT" and reads["a"][1].tolist() == [1, 2, 3, 4, 5] and reads["b"][0] == "GGC"
    sam = tmp_path / "star.sam"
    sam.write_text("x\t0\t*\t0\t0\t*\t*\t0\t0\tACGT\t*\ny\t16\t*\t0\t0\t*\t*\t0\t0\tACGT\t++++\n")
    reads = cli.read_records(str(sam))
    assert reads["x"] == ("ACGT", None) and reads["y"][1].tolist() == [10] * 4
    assert cli.pair_input(reads, ("x", "y")) is None and cli.pair_input(reads, ("y", "missing")) is None
    assert cli.read_records(str(sam), wanted={"y"}).keys() == {"y"}


def test_pairs_file_with_and_without_header(tmp_path):
    p = tmp_path / "pairs.txt"
    p.write_text("temp comp\nr1 r2\nr3\tr4\n")
    assert cli.read_pairs(str(p)) == [("r1", "r2"), ("r3", "r4")]
    assert cli.read_pairs(str(p), header=False) == [("temp", "comp"), ("r1", "r2"), ("r3", "r4")]


def _run(args, cwd=ROOT, stdout=None, env=None):
    return subprocess.run([sys.executable, "-m", "bonito_b200", "duplex", *args], cwd=cwd, capture_output=stdout is None,
                          stdout=stdout, stderr=subprocess.PIPE if stdout is not None else None, text=True, env=env)


def test_duplex_help_lists_the_reference_flags():
    out = _run(["-h"]).stdout
    for flag in ("in_bam", "duplex_pairs_file", "--reference", "--min-qscore", "--no-header", "--threads",
                 "--alignment-threads", "--mm2-preset"):
        assert flag in out, flag
    args = cli.argparser().parse_args(["r.sam", "p.txt"])
    assert (args.min_qscore, args.threads, args.alignment_threads, args.mm2_preset, args.no_header) == (0, 8, 8, "lr:hq", False)


def test_duplex_refusals_come_before_any_cuda_use(tmp_path):
    pairs = tmp_path / "pairs.txt"
    pairs.write_text("a b\n")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    for name in ("reads.bam", "reads.cram"):
        (tmp_path / name).write_bytes(b"")
        res = _run([str(tmp_path / name), str(pairs)], env=env)
        assert res.returncode == 1 and "htslib" in res.stderr and len(res.stderr.strip().splitlines()) == 1
    (tmp_path / "reads.sam").write_text("")
    res = _run([str(tmp_path / "reads.sam"), str(pairs), "--reference", "ref.fa"], env=env)
    assert res.returncode == 1 and "minimap2" in res.stderr


# ------------------------------------------------------------------------------------------------ GPU
def _mutate(rng, s, rate):
    out = []
    for ch in s:
        x = rng.random()
        if x < rate / 2:
            out.append(rng.choice([b for b in "ACGT" if b != ch]))
        elif x < 3 * rate / 4:
            out.append(ch)
            out.append(rng.choice("ACGT"))
        elif x >= rate:
            out.append(ch)
    return "".join(out)


def _gpu_batch(seed=7, n=36):
    rng = random.Random(seed)
    qs, rs = ["", "", "A", "ACGT"], ["", "ACGTA", "", "TGCA"]
    while len(qs) < n:
        base = "".join(rng.choice("ACGT") for _ in range(rng.choice([5, 40, 300, 1200, 2500])))
        rate = rng.choice([0.0, 0.05, 0.15, 0.3])
        q, r = _mutate(rng, base, rate), _mutate(rng, base, rate)
        if rng.random() < 0.25:
            r = r[: len(r) // 3]                        # a large length difference
        qs.append(q)
        rs.append(r)
    return qs, rs


@pytest.mark.gpu
def test_gpu_pair_align_matches_the_oracle_alone_and_banded():
    """Both modes bit for bit against the CPU oracle on a seeded batch (band doubled from 8, so long divergent pairs take
    several passes); every pair again alone; the banded GLOBAL_EDIT against the full band."""
    from bonito_b200 import native
    from bonito_b200.align import PairAligner
    qs, rs = _gpu_batch()
    al = PairAligner(qs, rs)
    idx = np.arange(len(qs))
    dist, ops, passes = al.global_edit(idx, k0=8)
    assert passes.max() >= 3
    full_d, full_ops = al._launch(native.PAIR_GLOBAL_EDIT, idx, np.maximum([len(q) for q in qs], [len(r) for r in rs]), True)
    score, aops = al.semiglobal_affine(idx)
    for p, (q, r) in enumerate(zip(qs, rs)):
        assert (dist[p], ops[p]) == O.global_edit(q, r), p
        assert (full_d[p], full_ops[p]) == (dist[p], ops[p]), p
        assert (score[p], aops[p]) == O.semiglobal_affine(q, r), p
    for p in range(0, len(qs), 5):
        alone = PairAligner([qs[p]], [rs[p]])
        d1, o1, _ = alone.global_edit([0], k0=8)
        s1, a1 = alone.semiglobal_affine([0])
        assert (d1[0], o1[0], s1[0], a1[0]) == (dist[p], ops[p], score[p], aops[p]), p


@pytest.mark.gpu
def test_gpu_over_budget_pair_gets_an_empty_consensus():
    from bonito_b200 import native
    from bonito_b200.align import EDIT_BAND0
    rng = random.Random(2)
    big = "".join(rng.choice("ACGT") for _ in range(3000))
    small = "".join(rng.choice("ACGT") for _ in range(200))
    t_big, c_big = big, D.revcomp(_mutate(rng, big, 0.05))
    t_small, c_small = small, D.revcomp(_mutate(rng, small, 0.02))
    pairs = [(t_big, np.full(len(t_big), 20, np.uint8), c_big, np.full(len(c_big), 20, np.uint8)),
             (t_small, np.full(len(t_small), 20, np.uint8), c_small, np.full(len(c_small), 20, np.uint8))]
    prepared = [D.prepare(*p) for p in pairs]
    budget = native.pair_align_trace_bytes(native.PAIR_GLOBAL_EDIT, len(t_small), len(c_small), 256) + 16
    # the first band of the big pair already needs more than the budget
    assert native.pair_align_trace_bytes(native.PAIR_GLOBAL_EDIT, len(t_big), len(c_big), EDIT_BAND0) > budget
    rs = D.align_pairs(prepared, budget=budget)
    assert rs[0] is None and rs[1] is not None
    assert D.finish(rs[1], *prepared[1]) == _cpu_call(*pairs[1])


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["sam", "fastq"])
def test_gpu_duplex_end_to_end_equals_the_golden_fixture(tmp_path, fmt):
    pairs = load_golden()
    reads = _write_inputs(tmp_path, pairs, fmt)
    pairs_file = tmp_path / "pairs.txt"
    lines = [f"{p[0]} {p[1]}" for p in pairs] + ["read000 missing_id"]
    pairs_file.write_text("template_id complement_id\n" + "\n".join(lines) + "\n")
    out_path = tmp_path / "out.fastq"
    with open(out_path, "w") as fh:
        res = _run([str(reads), str(pairs_file), "--threads", "3"], stdout=fh)
    assert res.returncode == 0, res.stderr
    assert "> completed reads: %d" % (len(pairs) + 1) in res.stderr and "bases per second" in res.stderr
    text = out_path.read_text().splitlines()
    got = {text[i][1:].split("\t")[0].split(" ")[0]: (text[i + 1], text[i + 3]) for i in range(0, len(text), 4)}
    want = {f"{p[0]};{p[1]}": (p[6], p[7]) for p in pairs if p[6]}
    assert got == want
    from bonito_b200.util import mean_qscore_from_qstring
    for i in range(0, len(text), 4):
        assert text[i].endswith(f"qs:i:{round(mean_qscore_from_qstring(text[i + 3]))}")

    sam_path = tmp_path / "out.sam"
    with open(sam_path, "w") as fh:
        res = _run([str(reads), str(pairs_file), "--min-qscore", "200"], stdout=fh)
    assert res.returncode == 0, res.stderr
    lines = sam_path.read_text().splitlines()
    assert [line.split("\t")[0] for line in lines] == ["@HD", "@PG"]
