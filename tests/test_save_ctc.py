"""
CTC training-data export (`basecaller --reference --save-ctc`) on the CPU: chunking, the per-chunk filters and their order,
targets, row selection, file locations and the writer's outputs, with fake mappings and a fake aligner.
"""
import io
import os
import pty
import subprocess
import sys

import numpy as np
import pytest
import torch

from bonito_b200.aligner import Mapping, revcomp
from bonito_b200.io import (CtcDataError, CtcWriter, alignment_lengths, ctc_output_paths, ctc_reject, ctc_target,
                            sam_header, sam_record, summary_field_names, typical_indices)
from bonito_b200.reader import Read, ReadChunk, read_chunks

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class FakeAligner:
    def __init__(self, contigs):
        self._seqs = dict(contigs)

    @property
    def contigs(self):
        return [(name, len(s)) for name, s in self._seqs.items()]

    def seq(self, name, start=0, end=None):
        return self._seqs[name][start:end]


def _read(read_id="r", n=1000, seed=0):
    rng = np.random.default_rng(seed)
    return Read(read_id, 90 + 20 * rng.standard_normal(n), filename="reads.npy", do_trim=False,
                meta={"run_id": "run0", "channel": 7, "mux": 2, "start_time": "12.5", "duration": 0.2})


def _reference_chunks(signal, chunksize, overlap):
    """The reference's rule, restated with torch.unfold."""
    if len(signal) < chunksize:
        return []
    _, offset = divmod(len(signal) - chunksize, chunksize - overlap)
    return [b.numpy() for b in torch.from_numpy(signal[offset:]).unfold(0, chunksize, chunksize - overlap)]


@pytest.mark.parametrize("length", [399, 400, 400 + 3 * 360, 400 + 3 * 360 + 17, 1999])
def test_read_chunks_reference_formula(length):
    read = _read(n=length)
    got = list(read_chunks(read, chunksize=400, overlap=40))
    want = _reference_chunks(read.signal, 400, 40)
    assert len(got) == len(want)
    assert len(got) == {399: 0, 400: 1, 1480: 4, 1497: 4, 1999: 5}[length]
    for i, (c, w) in enumerate(zip(got, want)):
        assert c.read_id == f"r:{i + 1}:{len(want)}"
        assert c.signal.dtype == np.float32 and c.signal.shape == (400,)
        np.testing.assert_array_equal(c.signal, w)
    if got:
        np.testing.assert_array_equal(got[-1].signal, read.signal[-400:])     # the last window ends at the read's end


def test_read_chunk_metadata():
    read = _read(n=800)
    c = next(read_chunks(read, chunksize=400, overlap=40))
    assert isinstance(c, ReadChunk)
    assert (c.filename, c.run_id, c.channel, c.mux) == ("reads.npy", "run0", 7, 2)
    assert (c.start, c.duration, c.template_start, c.template_duration) == ("12.5", 0.2, "12.5", 0.2)


def _mapping(ctg="c", r_st=0, r_en=100, q_st=0, q_en=100, strand=1, cigar="100M", nm=0, mapq=60):
    return Mapping(ctg, r_st, r_en, q_st, q_en, strand, mapq, cigar, nm, "")


def test_alignment_lengths():
    assert alignment_lengths(_mapping(cigar="50M2I10M3D38M", nm=7)) == (96, 103)


def test_reject_reasons_and_order():
    good = _mapping()
    seq = "A" * 100
    assert ctc_reject(seq, 20.0, good, "ACGT") is None
    # each reason alone
    assert ctc_reject(seq, 4.9, good, "ACGT", min_qscore=5) == "low_qscore"
    assert ctc_reject("", 20.0, good, "ACGT") == "zerolen_sequence"
    assert ctc_reject(seq, 20.0, None, "") == "no_mapping"
    assert ctc_reject(seq, 20.0, _mapping(nm=2), "ACGT") == "low_accuracy0.99"
    assert ctc_reject(seq, 20.0, _mapping(nm=2), "ACGT", min_accuracy=0.95) is None
    assert ctc_reject(seq, 20.0, _mapping(nm=2), "ACGT", min_accuracy=0.985) == "low_accuracy0.98"   # name uses :.2f
    assert ctc_reject(seq, 20.0, _mapping(q_st=11, cigar="89M", r_en=89), "ACGT") == "low_coverage0.90"
    assert ctc_reject(seq, 20.0, _mapping(q_st=10, cigar="90M", r_en=90), "ACGT") is None          # 0.90 is kept
    assert ctc_reject(seq, 20.0, good, "ACNGT") == "N_in_sequence"
    # the first reason that holds wins
    bad_all = _mapping(q_st=50, cigar="50M", nm=5)
    assert ctc_reject("", 1.0, None, "N", min_qscore=5) == "low_qscore"
    assert ctc_reject("", 20.0, None, "N") == "zerolen_sequence"
    assert ctc_reject(seq, 20.0, bad_all, "N") == "low_accuracy0.99"
    assert ctc_reject(seq, 20.0, _mapping(q_st=50, cigar="50M"), "N") == "low_coverage0.90"


@pytest.mark.parametrize("rna", [False, True])
@pytest.mark.parametrize("strand", [1, -1])
def test_targets(strand, rna):
    ref = "ACGGTTA"
    target = ctc_target(ref, strand, rna)
    oriented = ref if strand == 1 else revcomp(ref)
    want = np.array(["_ACGT".index(b) for b in oriented], dtype=np.uint8)
    np.testing.assert_array_equal(target, want[::-1] if rna else want)
    assert target.dtype == np.uint8


def test_typical_indices():
    x = np.array([100, 101, 99, 100, 102, 98, 100, 100, 101, 99, 100, 400], dtype=np.uint16)
    mu, sd = x.mean(), x.std()
    want = [i for i, v in enumerate(x) if mu - 2.5 * sd < v < mu + 2.5 * sd]
    assert typical_indices(x).tolist() == want and 11 not in want
    assert typical_indices(np.full(5, 37, dtype=np.uint16)).tolist() == [0, 1, 2, 3, 4]      # sd = 0 keeps all rows


def _items(n=12, chunksize=64, seed=3):
    """(chunk, result) pairs over one contig; chunk k carries the constant signal k, and its reference span has 20 + k
    bases, on alternate strands, so a row's chunk, target and summary line can be matched up."""
    rng = np.random.default_rng(seed)
    genome = "".join(rng.choice(list("ACGT"), 4000))
    parent = _read("p", n=chunksize * n)
    items, pos = [], 0
    for k in range(n):
        length = 20 + k
        chunk = ReadChunk(parent, np.full(chunksize, k, dtype=np.float32), k + 1, n)
        ref = genome[pos:pos + length]
        strand = 1 if k % 2 == 0 else -1
        seq = ref if strand == 1 else revcomp(ref)
        m = _mapping(r_st=pos, r_en=pos + length, q_en=length, strand=strand, cigar=f"{length}M")
        items.append((chunk, {"sequence": seq, "qstring": "5" * length, "mapping": m}))
        pos += length
    return genome, items


def _run(tmp_path, items, aligner, mode="w", seed=7, **kwargs):
    out, err = io.StringIO(), io.StringIO()
    np.random.seed(seed)
    w = CtcWriter(iter(items), aligner, fd=out, mode=mode, directory=str(tmp_path),
                  summary=str(tmp_path / "out_summary.tsv"), stderr=err, **kwargs)
    w.run()
    if w.error is not None:
        raise w.error
    return w, out.getvalue(), err.getvalue()


def _arrays(d):
    return [np.load(os.path.join(d, f)) for f in ("chunks.npy", "references.npy", "reference_lengths.npy")]


def _summary(path):
    lines = open(path).read().splitlines()
    assert lines[0].split("\t") == summary_field_names
    return [dict(zip(summary_field_names, line.split("\t"))) for line in lines[1:]]


def test_writer_rows_summary_and_records(tmp_path):
    genome, items = _items()
    aligner = FakeAligner([("c", genome)])
    w, out, err = _run(tmp_path, items, aligner)
    chunks, refs, lengths = _arrays(tmp_path)
    n = len(items)
    assert chunks.dtype == np.float16 and chunks.shape == (n, 64)
    assert refs.dtype == np.uint8 and refs.shape == (n, 20 + n - 1)
    assert lengths.dtype == np.uint16
    rows = _summary(tmp_path / "out_summary.tsv")
    assert len(rows) == n
    order = chunks[:, 0].astype(int)
    assert sorted(order.tolist()) == list(range(n)) and order.tolist() != list(range(n))       # permuted
    for i, k in enumerate(order):
        assert (chunks[i] == k).all() and lengths[i] == 20 + k
        chunk, res = items[k]
        m = res["mapping"]
        want = ctc_target(genome[m.r_st:m.r_en], m.strand)
        np.testing.assert_array_equal(refs[i, :lengths[i]], want)
        assert not refs[i, lengths[i]:].any()
        row = rows[i]
        assert row["read_id"] == chunk.read_id == f"p:{k + 1}:{n}"
        assert int(row["sequence_length_template"]) == 20 + k and int(row["alignment_genome_start"]) == m.r_st
        assert row["alignment_direction"] == ("+" if m.strand == 1 else "-")
        assert float(row["alignment_accuracy"]) == 1.0 and float(row["alignment_strand_coverage"]) == 1.0
        assert row["template_start"] == row["start_time"] == "12.5"
    # one SAM record per kept chunk, in input order, no tags
    lines = out.splitlines()
    header = sam_header(contigs=aligner.contigs).splitlines()
    assert lines[:len(header)] == header
    assert lines[len(header):] == [sam_record(c.read_id, r["sequence"], r["qstring"], r["mapping"]) for c, r in items]
    assert w.log == [(c.read_id, 64) for c, _ in items]
    assert f"> written ctc training data to {tmp_path}\n" in err
    assert f"  - chunks.npy with shape ({n},64)\n" in err
    assert f"  - references.npy with shape ({n},{20 + n - 1})\n" in err
    assert f"  - reference_lengths.npy shape ({n})\n" in err


def test_writer_rejects_and_typical_filter(tmp_path):
    genome, items = _items(n=14)
    aligner = FakeAligner([("c", genome[:300] + "N" + genome[301:])])
    # chunk 0 low qscore, 1 empty, 2 unmapped, 3 inaccurate, 4 low coverage, 5 over the N; the rest are kept
    items[0][1]["qstring"] = "!" * 20
    items[1][1].update(sequence="", qstring="", mean_qscore=20.0)     # an empty qstring alone would be low_qscore
    items[2][1]["mapping"] = None
    m = items[3][1]["mapping"]
    items[3][1]["mapping"] = Mapping(m.ctg, m.r_st, m.r_en, m.q_st, m.q_en, m.strand, m.mapq, m.cigar_str, 2, "")
    items[4][1]["mapping"] = Mapping(m.ctg, m.r_st, m.r_st + 10, m.q_st, 10, m.strand, m.mapq, "10M", 0, "")
    k_n = max(k for k in range(6, 14) if items[k][1]["mapping"].r_st <= 300)
    assert k_n > 5
    items[5], items[k_n] = items[k_n], items[5]      # the chunk over the N goes to position 5
    w, out, err = _run(tmp_path, items, aligner, min_qscore=5)
    assert w.rejected == {"low_qscore": 1, "zerolen_sequence": 1, "no_mapping": 1, "low_accuracy0.99": 1,
                          "low_coverage0.90": 1, "N_in_sequence": 1}
    assert list(w.rejected) == ["low_qscore", "zerolen_sequence", "no_mapping", "low_accuracy0.99",
                                "low_coverage0.90", "N_in_sequence"]
    assert err.startswith("> Chunks rejected from training data:\n - low_qscore: 1\n - zerolen_sequence: 1\n")
    kept = [c.read_id for c, _ in items[6:]]
    assert [l.split("\t")[0] for l in out.splitlines() if not l.startswith("@")] == kept
    chunks, refs, lengths = _arrays(tmp_path)
    want = typical_indices(np.array([20 + int(c.signal[0]) for c, _ in items[6:]], dtype=np.uint16))
    assert sorted(chunks[:, 0].astype(int).tolist()) == sorted(int(items[6 + i][0].signal[0]) for i in want)


def test_writer_outlier_dropped(tmp_path):
    genome, items = _items(n=12)
    chunk, res = items[11]
    long_ref = genome[3000:3300]
    m = _mapping(r_st=3000, r_en=3300, q_en=300, cigar="300M")
    items[11] = (chunk, {"sequence": long_ref, "qstring": "5" * 300, "mapping": m})
    w, out, err = _run(tmp_path, items, FakeAligner([("c", genome)]))
    chunks, refs, lengths = _arrays(tmp_path)
    assert 11 not in chunks[:, 0].astype(int).tolist() and len(chunks) == 11
    assert refs.shape[1] == 300 and lengths.max() == 30        # padded to the longest accepted target, as the reference
    assert len([l for l in out.splitlines() if not l.startswith("@")]) == 12    # its record is still written


def test_seeded_determinism(tmp_path):
    genome, items = _items(n=20)
    aligner = FakeAligner([("c", genome)])
    files = ("chunks.npy", "references.npy", "reference_lengths.npy", "out_summary.tsv")
    got = []
    for run, seed in (("a", 7), ("b", 7), ("c", 8)):
        d = tmp_path / run
        d.mkdir()
        _run(d, items, aligner, seed=seed)
        got.append([(d / f).read_bytes() for f in files])
    assert got[0] == got[1]
    assert got[0][0] != got[2][0]


def test_fastq_mode_headerless_sam(tmp_path):
    genome, items = _items(n=4)
    _, out, _ = _run(tmp_path, items, FakeAligner([("c", genome)]), mode="wfq")
    assert out.splitlines() == [sam_record(c.read_id, r["sequence"], r["qstring"], r["mapping"]) for c, r in items]


def test_no_data(tmp_path):
    genome, items = _items(n=3)
    for _, res in items:
        res["mapping"] = None
    w, out, err = _run(tmp_path, items, FakeAligner([("c", genome)]))
    assert err == "> no suitable ctc data to write\n"
    assert not any(f.endswith(".npy") for f in os.listdir(tmp_path))
    assert w.rejected == {"no_mapping": 3} and len(w.log) == 3


def test_target_over_uint16(tmp_path):
    n = 65_536
    genome = "ACGT" * (n // 4)
    chunk = ReadChunk(_read("p", n=64), np.zeros(64, dtype=np.float32), 1, 1)
    items = [(chunk, {"sequence": genome, "qstring": "5" * n,
                      "mapping": _mapping(r_en=n, q_en=n, cigar=f"{n}M")})]
    with pytest.raises(CtcDataError, match="65535"):
        _run(tmp_path, items, FakeAligner([("c", genome)]))
    assert not (tmp_path / "chunks.npy").exists()
    items[0][1]["mapping"] = _mapping(r_en=n - 1, q_en=n - 1, cigar=f"{n - 1}M")
    _run(tmp_path, items, FakeAligner([("c", genome)]))                 # 65 535 bases still fit
    assert np.load(tmp_path / "reference_lengths.npy").tolist() == [n - 1]


def test_output_paths_redirected_file(tmp_path):
    path = tmp_path / "calls.sam"
    with open(path, "w") as fh:
        assert ctc_output_paths(fh.fileno()) == (str(tmp_path), str(tmp_path / "calls_summary.tsv"))


def test_output_paths_pipe_and_terminal():
    r, w = os.pipe()
    try:
        assert ctc_output_paths(w) == (".", "summary.tsv")
    finally:
        os.close(r)
        os.close(w)
    master, slave = pty.openpty()
    try:
        assert ctc_output_paths(slave) == (".", "summary.tsv")
    finally:
        os.close(master)
        os.close(slave)
    with open(os.devnull, "w") as fh:
        assert ctc_output_paths(fh.fileno()) == (".", "summary.tsv")


def test_output_paths_of_stdout_in_a_child(tmp_path):
    """The default location comes from the process's own stdout: a file beside it, the working directory for a pipe."""
    code = "from bonito_b200.io import ctc_output_paths; import sys; sys.stderr.write(repr(ctc_output_paths()))"
    env = {**os.environ, "PYTHONPATH": ROOT}
    with open(tmp_path / "x.bam", "w") as fh:
        p = subprocess.run([sys.executable, "-c", code], stdout=fh, stderr=subprocess.PIPE, text=True, env=env)
    assert p.stderr == repr((str(tmp_path), str(tmp_path / "x_summary.tsv")))
    p = subprocess.run([sys.executable, "-c", code], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, env=env)
    assert p.stderr == repr((".", "summary.tsv"))


def test_cli_save_ctc_needs_reference(tmp_path):
    np.save(tmp_path / "read0.npy", np.zeros(100, dtype=np.float32))
    p = subprocess.run([sys.executable, "-m", "bonito_b200", "basecaller", str(tmp_path / "no_model"), str(tmp_path),
                        "--save-ctc", "--device", "cpu"], cwd=ROOT, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE,
                       text=True, timeout=300)
    assert p.returncode == 1
    assert "> error: --save-ctc needs --reference" in p.stderr
