"""GPU mapping (bonito_b200/csrc/map.cu through bonito_b200.aligner) against the CPU oracle tests/_oracle_map.py, byte for
byte, then end to end on a simulated genome with known read origins, and `basecaller --reference` on the CLI."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import _oracle_map as O
from _map_helpers import _fasta, _mutate, _rand, _rc
from bonito_b200 import aligner as A
from bonito_b200 import native

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_minimizer_kernel_equals_oracle():
    rng = np.random.default_rng(1)
    seqs = [_rand(rng, n) for n in (0, 5, 36, 37, 1000, 20000, 0, 3)]
    seqs[5][100:400] = ord("N")
    seqs[4][500:501] = ord("N")
    for k, w in A.PRESETS.values():
        data = np.concatenate(seqs)
        off = np.concatenate(([0], np.cumsum([len(s) for s in seqs]))).astype(np.int64)
        seq, seq_off = torch.from_numpy(data).cuda(), torch.from_numpy(off).cuda()
        kmer, mm = torch.empty(len(data), dtype=torch.int64, device="cuda"), torch.empty(len(data), dtype=torch.int64,
                                                                                          device="cuda")
        native.map_minimizers(seq, seq_off, k, w, kmer, mm)
        got = mm.cpu().numpy()
        want = np.full(len(data), -1, dtype=np.int64)
        for s, o in zip(seqs, off[:-1]):
            for p, key in O.minimizers(s.tobytes(), k, w):
                want[o + p] = key
        assert np.array_equal(got, want), (k, w)
        for s, o in zip(seqs, off[:-1]):
            if len(s) < k + w - 1:                     # shorter than one window: no minimizer
                assert (got[o:o + len(s)] < 0).all()


def _small_genome(rng):
    contigs = [("chrA", _rand(rng, 40000)), ("chrB", _rand(rng, 8000)), ("tiny", _rand(rng, 20)), ("chrC", _rand(rng, 3000))]
    contigs[0][1][30000:30300] = ord("N")
    return contigs


def _planted_reads(rng, contigs, n):
    reads = []
    for t in range(n):
        c = [0, 1, 3][t % 3]
        seq = contigs[c][1]
        L = int(rng.integers(200, 1500))
        st = [0, len(seq) - L, int(rng.integers(0, len(seq) - L))][t % 3] if L < len(seq) else 0
        r = _mutate(rng, seq[st:st + L], 0.03, 0.02, 0.02)
        if t % 2:
            r = _rc(r)
        if t % 7 == 0:
            r = r.copy()
            r[len(r) // 3:len(r) // 3 + 40] = ord("N")
        reads.append(r.tobytes())
    reads += [_rand(rng, 700).tobytes(), _rand(rng, 30).tobytes(), b"", contigs[0][1][29900:30500].tobytes()]
    return reads


@pytest.mark.parametrize("preset", ["lr:hq", "map-ont"])
def test_map_batch_equals_oracle(tmp_path, preset):
    """Reads near contig ends and N runs, reads shorter than a window, a contig shorter than a window, random reads."""
    rng = np.random.default_rng(2 if preset == "lr:hq" else 3)
    contigs = _small_genome(rng)
    _fasta(tmp_path / "ref.fa", contigs)
    al = A.Aligner(str(tmp_path / "ref.fa"), preset=preset)
    index = O.Index([(n, s.tobytes()) for n, s in contigs], *A.PRESETS[preset])
    reads = _planted_reads(rng, contigs, 24)
    res, _, _, lens = al.chains(reads)
    got = al.map_batch(reads)
    n_mapped = 0
    for t, read in enumerate(reads):
        anc = O.anchors(index, read, index.k)
        f, pred = O.chain_dp(anc, index.off, index.k)
        ch = O.extract(anc, f, pred, len(read), index.k)
        if ch is None:
            assert res[t, 0] == 0, t
        else:
            want = [ch["n"], ch["f1"], ch["f2"], ch["strand"], ch["W"], *ch["chain"][0], *ch["chain"][-1]]
            assert res[t].tolist() == want, t
        m = O.map_read(index, read)
        assert (None if got[t] is None else tuple(vars(got[t]).values())) == m, t
        n_mapped += m is not None
    assert n_mapped >= 20


def test_more_reads_than_warps_and_any_batching(tmp_path):
    rng = np.random.default_rng(4)
    contigs = _small_genome(rng)
    _fasta(tmp_path / "ref.fa", contigs)
    al = A.Aligner(str(tmp_path / "ref.fa"), preset="map-ont")
    reads = []
    for _ in range(5000):
        c = contigs[int(rng.integers(0, 2))][1]
        st = int(rng.integers(0, len(c) - 400))
        r = _mutate(rng, c[st:st + int(rng.integers(200, 400))], 0.02, 0.01, 0.01)
        reads.append((_rc(r) if rng.random() < 0.5 else r).tobytes())
    whole = al.map_batch(reads)
    assert sum(m is not None for m in whole) > 4096          # more alignments than the align kernel's grid has warps
    parts = [m for i in range(0, len(reads), 700) for m in al.map_batch(reads[i:i + 700])]
    assert whole == parts
    index = O.Index([(n, s.tobytes()) for n, s in contigs], 15, 10)
    for t in range(0, 5000, 500):
        assert (None if whole[t] is None else tuple(vars(whole[t]).values())) == O.map_read(index, reads[t]), t


def _check_record(m, read, contigs_by_name):
    """CIGAR consumption and NM / MD recomputed from the CIGAR, the read and the contig."""
    import re
    q = read if m.strand == 1 else _rc(np.frombuffer(read, np.uint8)).tobytes()
    lo, hi = (m.q_st, m.q_en) if m.strand == 1 else (len(read) - m.q_en, len(read) - m.q_st)
    ops = re.findall(r"(\d+)([MID])", m.cigar_str)
    assert sum(int(n) for n, op in ops if op in "MI") == m.q_en - m.q_st
    assert sum(int(n) for n, op in ops if op in "MD") == m.r_en - m.r_st
    nm, md = O.nm_md_from_cigar(m.cigar_str, q[lo:hi], contigs_by_name[m.ctg][m.r_st:m.r_en])
    assert (nm, md) == (m.NM, m.MD)


def test_simulated_genome_end_to_end(tmp_path):
    rng = np.random.default_rng(5)
    contigs = [("chr1", _rand(rng, 1_000_000)), ("chr2", _rand(rng, 400_000)), ("chr3", _rand(rng, 50_000))]
    dup_src, dup_dst, DUP = 200_000, 150_000, 20_000
    contigs[1][1][dup_dst:dup_dst + DUP] = contigs[0][1][dup_src:dup_src + DUP]
    _fasta(tmp_path / "ref.fa", contigs)
    by_name = {n: s.tobytes() for n, s in contigs}
    al = A.Aligner(str(tmp_path / "ref.fa"))
    reads, truth = [], []
    for t in range(240):
        c = int(rng.choice(3, p=[0.6, 0.3, 0.1]))
        seq = contigs[c][1]
        L = int(min(np.exp(rng.uniform(np.log(1000), np.log(30000))), len(seq) - 1))
        st = int(rng.integers(0, len(seq) - L))
        rates = (0.02, 0.01, 0.01) if t % 2 else (0.05, 0.03, 0.03)
        r = _mutate(rng, seq[st:st + L], *rates)
        strand = -1 if t % 4 >= 2 else 1
        inside_dup = (c == 0 and st < dup_src + DUP and st + L > dup_src) or (c == 1 and st < dup_dst + DUP and st + L > dup_dst)
        reads.append((_rc(r) if strand < 0 else r).tobytes())
        truth.append(None if inside_dup else (contigs[c][0], st, strand))
    dup_reads = []
    for t in range(20):
        L = int(rng.integers(1000, 15000))
        st = dup_src + 100 + int(rng.integers(0, DUP - 200 - L))
        r = _mutate(rng, contigs[0][1][st:st + L], 0.02, 0.01, 0.01)
        dup_reads.append(len(reads))
        reads.append((_rc(r) if t % 2 else r).tobytes())
        truth.append(None)
    random_reads = list(range(len(reads), len(reads) + 100))
    reads += [_rand(rng, int(rng.integers(1000, 30000))).tobytes() for _ in random_reads]
    truth += [None] * len(random_reads)

    got = al.map_batch(reads)
    assert got == al.map_batch(reads)                        # two runs are identical
    good = total = 0
    for t, want in enumerate(truth):
        m = got[t]
        if m is not None:
            _check_record(m, reads[t], by_name)
        if want is None:
            continue
        total += 1
        if m is None:
            continue
        lead = m.q_st if m.strand == 1 else len(reads[t]) - m.q_en
        good += (m.ctg, m.strand) == (want[0], want[2]) and abs(m.r_st - lead - want[1]) <= 50
    assert good >= 0.99 * total, (good, total)
    assert all(got[t] is not None and got[t].mapq == 0 for t in dup_reads), [got[t] for t in dup_reads]
    assert sum(got[t] is None for t in random_reads) >= 0.99 * len(random_reads)


def test_cli_basecaller_reference(tmp_path):
    """Basecall seeded reads, write the calls (some reverse-complemented) as the reference, run `--reference` on the same
    reads: every read maps to its own contig on the planted strand, full length, NM 0."""
    from oracle import synth
    spec = synth.model_spec("fast", n_lstm=3)
    weights = synth.make_weights(spec, seed=4)
    mdir = synth.write_model_dir(str(tmp_path / "model"), spec, weights, batchsize=8, chunksize=2000, overlap=120)
    rdir = tmp_path / "reads"
    rdir.mkdir()
    for i in range(6):
        np.save(rdir / f"read{i}.npy", 93.7 + 23.5 * synth.squiggle(1, 24000 + 1000 * i, seed=40 + i)[0, 0].numpy())
    base = [sys.executable, "-m", "bonito_b200", "basecaller", mdir, str(rdir), "--no-trim"]
    with open(tmp_path / "calls.fastq", "w") as fh:
        p = subprocess.run(base, cwd=ROOT, stdout=fh, stderr=subprocess.PIPE, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    lines = (tmp_path / "calls.fastq").read_text().split("\n")
    calls = {lines[i][1:].split()[0]: lines[i + 1] for i in range(0, len(lines) - 1, 4)}
    assert len(calls) == 6
    planted = {rid: (16 if i % 2 else 0) for i, rid in enumerate(sorted(calls))}
    _fasta(tmp_path / "ref.fa", [(f"ctg_{rid}", np.frombuffer((A.revcomp(s) if planted[rid] else s).encode(), np.uint8))
                                 for rid, s in sorted(calls.items())])
    with open(tmp_path / "out.sam", "w") as fh:
        p = subprocess.run(base + ["--reference", str(tmp_path / "ref.fa"), "--alignment-threads", "3"], cwd=ROOT,
                           stdout=fh, stderr=subprocess.PIPE, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    assert "> loading reference" in p.stderr and "> outputting aligned sam" in p.stderr
    text = (tmp_path / "out.sam").read_text().splitlines()
    header = [l for l in text if l.startswith("@")]
    assert [l.split("\t")[1] for l in header if l.startswith("@SQ")] == [f"SN:ctg_{r}" for r in sorted(calls)]
    assert any(l.startswith("@PG\tID:aligner") for l in header)
    for rec in (l.split("\t") for l in text if not l.startswith("@")):
        rid, seq = rec[0], calls[rec[0]]
        assert rec[2] == f"ctg_{rid}" and int(rec[1]) == planted[rid] and rec[3] == "1", rec[:6]
        assert rec[5] == f"{len(seq)}M" and "NM:i:0" in rec and f"MD:Z:{len(seq)}" in rec
        assert rec[9] == (A.revcomp(seq) if planted[rid] else seq)
    with open(tmp_path / "out.fastq", "w") as fh:
        p = subprocess.run(base + ["--reference", str(tmp_path / "ref.fa")], cwd=ROOT, stdout=fh, stderr=subprocess.PIPE,
                           text=True, timeout=600)
    assert p.returncode == 0 and "did you really want aligned fastq?" in p.stderr
    assert (tmp_path / "out.fastq").read_text() == (tmp_path / "calls.fastq").read_text()
    for args, msg in ((["--reference", str(tmp_path / "ref.fa"), "--mm2-preset", "sr"], "mm2-preset"),
                      (["--reference", str(tmp_path / "missing.fa")], "> failed to load/build index"),
                      (["--save-ctc"], "--save-ctc")):
        p = subprocess.run(base + args, cwd=ROOT, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, text=True, timeout=600)
        assert p.returncode == 1 and msg in p.stderr, p.stderr[-1000:]
