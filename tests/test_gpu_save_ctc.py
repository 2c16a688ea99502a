"""
`basecaller --reference --save-ctc` end to end on the GPU: the reference is built from the chunk calls themselves (as they
are, reverse-complemented, with ~3 % substitutions, with an N, or left out), and the CLI's rows, reject counts and
records must be exactly what `Aligner.map_batch` of the same calls and the reference's filter rules, restated here, give.
"""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import _oracle_bam as B
from _map_helpers import _fasta
from bonito_b200 import synth
from bonito_b200.aligner import Aligner, revcomp
from bonito_b200.io import sam_record
from bonito_b200.nn import fuse_bn_
from bonito_b200.reader import Reader, read_chunks
from bonito_b200.util import load_model, load_symbol

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FILES = ("chunks.npy", "references.npy", "reference_lengths.npy")


def _chunk_calls(mdir, rdir):
    """(chunk reads, results) of the chunks the CLI makes, basecalled in the CLI's batches."""
    model = load_model(mdir, "cuda", use_koi=True).apply(fuse_bn_)
    scaling = model.config.get("scaling")
    pa = bool(scaling) and scaling.get("strategy") == "pa"
    reads = Reader(rdir).get_reads(rdir, do_trim=False, scaling_strategy=scaling,
                                   norm_params=model.config.get("standardisation") if pa else model.config.get("normalisation"))
    p = model.config["basecaller"]
    chunks = [c for r in reads for c in read_chunks(r, p["chunksize"], p["overlap"])]
    results = list(load_symbol(mdir, "basecall")(model, iter(chunks), batchsize=p["batchsize"], chunksize=p["chunksize"],
                                                   overlap=p["overlap"]))
    assert [r.read_id for r, _ in results] == [c.read_id for c in chunks]
    return chunks, [res for _, res in results]


def _plant(tmp_path, chunks, results, plan, seed=0):
    """A FASTA of one contig per chunk call, placed per parent read by `plan` ("as_is", "revcomp", "subs", "n", "absent")."""
    rng = np.random.default_rng(seed)
    contigs = []
    for c, res in zip(chunks, results):
        seq = res["sequence"]
        kind = plan[int(c.read_id.split(":")[0][len("read"):])]
        if not seq or kind == "absent":
            continue
        if kind == "revcomp":
            seq = revcomp(seq)
        elif kind == "subs":
            s = bytearray(seq.encode())
            for pos in rng.choice(len(s), max(1, round(0.03 * len(s))), replace=False):
                s[pos] = ord("ACGT".replace(chr(s[pos]), "")[rng.integers(3)])
            seq = s.decode()
        elif kind == "n":
            mid = len(seq) // 2
            seq = seq[:mid] + "N" + seq[mid + 1:]
        contigs.append((f"ctg_{c.read_id}", np.frombuffer(seq.encode(), np.uint8)))
    path = tmp_path / "ref.fa"
    _fasta(path, contigs)
    return str(path)


def _reason(seq, m, refspan, min_accuracy=0.99, min_coverage=0.90):
    """The reference's per-chunk filters in their order (mean qscore >= 0 always passes the default --min-qscore 0)."""
    if not seq:
        return "zerolen_sequence"
    if m is None:
        return "no_mapping"
    ops = {"M": 0, "I": 0, "D": 0}
    for n, op in re.findall(r"(\d+)([MID])", m.cigar_str):
        ops[op] += int(n)
    blen = sum(ops.values())
    if (blen - m.NM) / blen < min_accuracy:
        return f"low_accuracy{min_accuracy:.2f}"
    if (m.q_en - m.q_st) / len(seq) < min_coverage:
        return f"low_coverage{min_coverage:.2f}"
    if "N" in refspan:
        return "N_in_sequence"
    return None


def _expected(ref, chunks, results):
    """(kept (chunk index, mapping) in input order, reject counts, expected row set after the typical-length filter,
    the reason of every chunk)."""
    al = Aligner(ref)
    maps = al.map_batch([res["sequence"] for res in results])
    kept, rejected, rows, reasons = [], {}, [], []
    for k, (c, res, m) in enumerate(zip(chunks, results, maps)):
        span = al.seq(m.ctg, m.r_st, m.r_en) if m is not None else ""
        why = _reason(res["sequence"], m, span)
        reasons.append(why)
        if why is not None:
            rejected[why] = rejected.get(why, 0) + 1
            continue
        oriented = span if m.strand == 1 else revcomp(span)
        target = np.array(["_ACGT".index(b) for b in oriented], dtype=np.uint8)
        kept.append((k, m))
        rows.append((c.signal.astype(np.float16).tobytes(), target.tobytes()))
    lengths = np.array([len(t) for _, t in rows], dtype=np.float64)
    mu, sd = lengths.mean(), lengths.std()
    typical = [r for r, n in zip(rows, lengths) if sd == 0 or mu - 2.5 * sd < n < mu + 2.5 * sd]
    return kept, rejected, typical, reasons


def _basecaller(mdir, rdir, out, ref):
    """`basecaller --reference ref --save-ctc > out` -> its stderr."""
    cmd = [sys.executable, "-m", "bonito_b200", "basecaller", mdir, rdir, "--no-trim", "--reference", ref, "--save-ctc"]
    os.makedirs(os.path.dirname(out), exist_ok=True)
    with open(out, "w") as fh:
        p = subprocess.run(cmd, cwd=ROOT, stdout=fh, stderr=subprocess.PIPE, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-3000:]
    return p.stderr


def _rows(directory):
    chunks, refs, lengths = (np.load(os.path.join(directory, f)) for f in FILES)
    assert chunks.dtype == np.float16 and refs.dtype == np.uint8 and lengths.dtype == np.uint16
    return [(c.tobytes(), r[:n].tobytes()) for c, r, n in zip(chunks, refs, lengths)]


def _rejects(stderr):
    return {m.group(1): int(m.group(2)) for m in re.finditer(r"^ - (\S+): (\d+)$", stderr, re.M)}


def _records(path):
    return [l for l in open(path).read().splitlines() if not l.startswith("@")]


def test_save_ctc_lstm_crf(tmp_path):
    spec = synth.model_spec("fast", n_lstm=3)
    mdir = synth.write_model_dir(str(tmp_path / "model"), spec, synth.make_weights(spec, seed=4), batchsize=8,
                                 chunksize=2000, overlap=120)
    rdir = tmp_path / "reads"
    rdir.mkdir()
    for i in range(6):
        np.save(rdir / f"read{i}.npy", 93.7 + 23.5 * synth.squiggle(1, 25000 + 137 * i, seed=40 + i)[0, 0].numpy())
    chunks, results = _chunk_calls(mdir, str(rdir))
    plan = ["as_is", "as_is", "revcomp", "subs", "n", "absent"]
    ref = _plant(tmp_path, chunks, results, plan)
    kept, rejected, typical, reasons = _expected(ref, chunks, results)

    sam = tmp_path / "sam" / "out.sam"
    err = _basecaller(mdir, str(rdir), str(sam), ref)
    assert f"> written ctc training data to {sam.parent}" in err, err[-3000:]
    assert sorted(_rows(sam.parent)) == sorted(typical)
    assert _rejects(err) == rejected
    assert f"> completed reads: {len(chunks)}" in err
    want = [sam_record(chunks[k].read_id, results[k]["sequence"], results[k]["qstring"], m) for k, m in kept]
    assert _records(sam) == want
    header = [l for l in open(sam).read().splitlines() if l.startswith("@")]
    assert sum(l.startswith("@SQ") for l in header) == len(Aligner(ref).contigs)
    summary = open(sam.parent / "out_summary.tsv").read().splitlines()
    assert len(summary) == 1 + len(typical)

    # every planted category shows up
    parent = {k: int(chunks[k].read_id.split(":")[0][len("read"):]) for k in range(len(chunks))}
    accepted = {parent[k] for k, m in kept if m.NM == 0}
    assert {0, 1, 2} <= accepted
    assert any(parent[k] == 2 and m.strand == -1 for k, m in kept)
    assert not any(parent[k] in (3, 4, 5) for k, _ in kept)
    assert "low_accuracy0.99" in [reasons[k] for k in parent if parent[k] == 3]
    assert "N_in_sequence" in [reasons[k] for k in parent if parent[k] == 4]

    # the same seed writes the same files; BAM and FASTQ runs write the same arrays and records
    again = tmp_path / "again" / "out.sam"
    _basecaller(mdir, str(rdir), str(again), ref)
    for f in (*FILES, "out_summary.tsv"):
        assert (again.parent / f).read_bytes() == (sam.parent / f).read_bytes(), f
    bam = tmp_path / "bam" / "out.bam"
    _basecaller(mdir, str(rdir), str(bam), ref)
    _, refs, lines, _ = B.decode_bam(B.bgzf_decompress(bam.read_bytes()))
    assert refs == Aligner(ref).contigs
    assert len(lines) == len(want) and all(B.same_sam_line(a, b) for a, b in zip(lines, want))
    fq = tmp_path / "fq" / "out.fastq"
    err = _basecaller(mdir, str(rdir), str(fq), ref)
    assert "did you really want aligned fastq?" in err
    assert fq.read_text().splitlines() == want
    for d in (bam.parent, fq.parent):
        for f in FILES:
            assert (d / f).read_bytes() == (sam.parent / f).read_bytes(), (d, f)

    p = subprocess.run([sys.executable, "-m", "bonito_b200", "basecaller", mdir, str(rdir), "--save-ctc"], cwd=ROOT,
                       stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, text=True, timeout=600)
    assert p.returncode == 1 and "--save-ctc" in p.stderr

    # evaluate reads the dataset back: the targets are the model's own calls of the same fp16 chunks
    n = len(typical)
    p = subprocess.run([sys.executable, "-m", "bonito_b200", "evaluate", mdir, "--directory", str(sam.parent),
                        "--chunks", str(n), "--weights", "1"], cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                       text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-3000:]
    out = p.stdout + p.stderr
    assert re.search(rf"\* num_chunks\s+{n}\b", out), out[-2000:]
    assert re.search(r"\* accuracy\s+100\.00%", out), out[-2000:]


def test_save_ctc_quartznet(tmp_path):
    spec = synth.quartznet_spec("v1", max_repeat=2)
    mdir = synth.write_quartznet_dir(str(tmp_path / "ctc"), spec, synth.make_quartznet_weights(spec, seed=11),
                                     batchsize=16, chunksize=2000, overlap=200)
    rdir = tmp_path / "reads"
    rdir.mkdir()
    for i in range(3):
        np.save(rdir / f"read{i}.npy", 93.7 + 23.5 * synth.squiggle(1, 9000 + 311 * i, seed=70 + i)[0, 0].numpy())
    chunks, results = _chunk_calls(mdir, str(rdir))
    ref = _plant(tmp_path, chunks, results, ["as_is", "revcomp", "absent"])
    kept, rejected, typical, reasons = _expected(ref, chunks, results)
    sam = tmp_path / "sam" / "out.sam"
    err = _basecaller(mdir, str(rdir), str(sam), ref)
    assert typical and f"> written ctc training data to {sam.parent}" in err, err[-3000:]
    assert sorted(_rows(sam.parent)) == sorted(typical)
    assert _rejects(err) == rejected
    want = [sam_record(chunks[k].read_id, results[k]["sequence"], results[k]["qstring"], m) for k, m in kept]
    assert _records(sam) == want
