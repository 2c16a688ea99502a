"""
pysam-free output for `bonito_b200 basecaller` and `duplex`: FASTQ, SAM text (unaligned, or aligned by
bonito_b200.aligner) and BAM, with the reference's header, record and tag layout (`bonito/io.py:41-166,400-469`,
`documentation/SAM.md`), including the sequence-to-signal move table `mv:B:c,<stride>,<moves...>` (`io.py:57-70,455-456`).
The reference writes through pysam / htslib.  Here BAM records are the binary encoding of the SAM lines this module
builds (bonito_b200.bam), BGZF-compressed on the GPU; CRAM needs htslib, which this build does not bundle, so it is refused
with an explanation instead of being approximated.
Deviation: on the reverse strand QUAL is reversed along with SEQ, as the SAM specification requires; the reference
reverse-complements SEQ and leaves QUAL as called.

`CtcWriter` writes the CTC training data of `basecaller --reference --save-ctc` (reference: `CTCWriter`,
bonito/io.py:513-619): every mapped chunk call that passes the reference's filters becomes a row of `chunks.npy`,
`references.npy` and `reference_lengths.npy`, and a record on stdout.  Deviations from the reference:
  * when every target has the same length (sd = 0) `typical_indices` keeps all rows; the reference's strict
    `mu - 2.5 sd < x < mu + 2.5 sd` keeps none and then reports success with empty arrays.
  * a Mapping has no `mlen` / `blen`: they come from its CIGAR (M / I / D) and NM, `blen = M + I + D`, `mlen = blen - NM`,
    so N columns count in both (mappy leaves ambiguous bases out).  A chunk over an N is rejected either way; only the
    reject name can differ.
  * the summary TSV is overwritten; the reference's CSVLogger appends to an existing file and then rewrites it.
  * a target over 65 535 bases stops the run with an error instead of wrapping in uint16 (only a very large
    `--chunksize` can produce one).
  * the arrays and summary go next to the file stdout is redirected to, or to the working directory when stdout is not a
    regular file (a terminal, a pipe, /dev/null); the reference's `dirname(realpath('/dev/fd/1'))` points into /proc for
    a pipe.
"""

import os
import re
import sys
from collections import namedtuple
from os.path import realpath
from threading import Thread

import numpy as np

from bonito_b200.aligner import revcomp
from bonito_b200.bam import BamOutput
from bonito_b200.util import mean_qscore_from_qstring

__ont_bam_spec__ = "0.0.2"
__version__ = "0.2.0"

Format = namedtuple("Format", "aligned name mode")


def biofmt(aligned=False):
    """Output format from the file extension stdout is redirected to (reference: bonito/io.py:35-54)."""
    mode, name = ("w", "sam") if aligned else ("wfq", "fastq")
    aligned = "aligned" if aligned else "unaligned"
    try:
        stdout = realpath("/dev/fd/1")
    except OSError:
        stdout = ""
    if sys.stdout.isatty() or stdout.startswith("/proc") or not stdout:
        return Format(aligned, name, mode)
    ext = stdout.split(os.extsep)[-1]
    if ext in ("fq", "fastq"):
        return Format(aligned, "fastq", "wfq")
    if ext == "bam":
        return Format(aligned, "bam", "wb")
    if ext == "cram":
        return Format(aligned, "cram", "wc")
    if ext == "sam":
        return Format(aligned, "sam", "w")
    return Format(aligned, name, mode)


def encode_moves(moves, stride, sep=","):
    """
    `stride` followed by the single-digit moves, comma separated (reference: bonito/io.py:57-70).

    >>> encode_moves(np.array([0, 1, 0, 1, 1], dtype=np.int8), 5)
    '5,0,1,0,1,1'
    """
    moves = np.asarray(moves)
    out = np.full(2 * moves.size, ord(sep), dtype=np.uint8)
    out[1::2] = moves.astype(np.uint8) + ord("0")
    return f"{stride}{out.tobytes().decode('ascii')}"


def write_fastq(header, sequence, qstring, fd=sys.stdout, tags=None, sep="\t"):
    """FASTQ record; tags (if any) follow the read id on the header line (reference: bonito/io.py:97-106)."""
    if tags is not None:
        fd.write(f"@{header} {sep.join(tags)}\n")
    else:
        fd.write(f"@{header}\n")
    fd.write(f"{sequence}\n+\n{qstring}\n")


def sam_header(groups=(), sep="\t", argv=None, contigs=None):
    """@HD (+ @SQ per contig) + @PG basecaller (+ @PG aligner when `contigs`, [(name, length)], is given) + read groups
    (reference: io.py:109-133)."""
    argv = sys.argv[1:] if argv is None else argv
    lines = [sep.join(["@HD", "VN:1.5", "SO:unknown", "ob:%s" % __ont_bam_spec__])]
    lines += [sep.join(["@SQ", f"SN:{name}", f"LN:{length}"]) for name, length in contigs or ()]
    lines.append(sep.join(["@PG", "ID:basecaller", "PN:bonito_b200", "VN:%s" % __version__,
                           "CL:bonito_b200 %s" % " ".join(argv)]))
    if contigs:
        lines.append(sep.join(["@PG", "ID:aligner", "PN:bonito_b200", "VN:%s" % __version__,
                               "DS:GPU minimizer chaining and banded local alignment"]))
    return "%s\n" % "\n".join([*lines, *groups])


def sam_record(read_id, sequence, qstring, mapping=None, tags=None, sep="\t"):
    """SAM record in the layout of the reference's `sam_record` (io.py:136-166): flag 4 without a mapping; with one (a
    bonito_b200.aligner.Mapping) flag 0 / 16, soft clips in reference orientation, SEQ and QUAL reversed on strand -."""
    if mapping:
        fwd = mapping.strand == +1
        right = len(sequence) - mapping.q_en
        clips = ["%dS" % mapping.q_st if mapping.q_st else "", mapping.cigar_str, "%dS" % right if right else ""]
        record = [read_id, 0 if fwd else 16, mapping.ctg, mapping.r_st + 1, mapping.mapq,
                  "".join(clips if fwd else clips[::-1]), "*", 0, 0, sequence if fwd else revcomp(sequence),
                  qstring if fwd else qstring[::-1], "NM:i:%d" % mapping.NM, "MD:Z:%s" % mapping.MD]
    else:
        record = [read_id, 4, "*", 0, 0, "*", "*", 0, 0, sequence, qstring, "NM:i:0"]
    if tags is not None:
        record.extend(tags)
    return sep.join(map(str, record))


def read_tags(read, res, group_key=None, with_moves=True):
    """RG / qs / ns / ts + the read's own tag data + the move table (reference: bonito/io.py:441-456)."""
    qstring = res.get("qstring", "*")
    mean_q = res.get("mean_qscore", mean_qscore_from_qstring(qstring))
    tags = []
    run_id = getattr(read, "run_id", None)
    if run_id is not None:
        tags.append(f"RG:Z:{run_id}_{group_key}")
    tags += [f"qs:i:{round(mean_q)}", f"ns:i:{getattr(read, 'num_samples', len(read.signal))}",
             f"ts:i:{getattr(read, 'trimmed_samples', 0)}"]
    if hasattr(read, "tagdata"):
        tags += list(read.tagdata())
    if with_moves and res.get("moves") is not None:
        tags.append(f"mv:B:c,{encode_moves(res['moves'], res['stride'])}")
    return tags


class DuplexWriter(Thread):
    """
    Writes `duplex` consensus reads, named `<template id>;<complement id>` with a `qs:i:` tag (reference: bonito/io.py:472-502):
    `iterator` yields ((template id, complement id), {"sequence", "qstring"}).  `.log` holds (read name, bases) of every
    pair, written or not, as the reference counts them; empty and below-`min_qscore` consensuses are not written.
    """

    def __init__(self, iterator, fd=sys.stdout, min_qscore=0, mode="wfq"):
        super().__init__(daemon=True)
        if mode not in ("wfq", "w"):
            raise ValueError(f"output mode {mode!r} needs htslib (BAM / CRAM), which this build does not bundle: "
                             "redirect to a .sam or .fastq file")
        self.iterator, self.fd, self.min_qscore, self.mode = iterator, fd, min_qscore, mode
        self.log, self.error = [], None

    def run(self):
        try:
            self.begin()
            for (temp_id, comp_id), res in self.iterator:
                read_id = f"{temp_id};{comp_id}"
                seq, qstring = res["sequence"], res["qstring"]
                mean_q = mean_qscore_from_qstring(qstring)
                self.log.append((read_id, len(seq)))
                if mean_q < self.min_qscore or not len(seq):
                    continue
                self.write_read(read_id, seq, qstring, [f"qs:i:{round(mean_q)}"])
            self.end()
        except BaseException as err:   # surfaced by the CLI after join()
            self.error = err

    def begin(self):
        if self.mode == "w":
            self.fd.write(sam_header())

    def write_read(self, read_id, seq, qstring, tags):
        if self.mode == "w":
            self.fd.write(sam_record(read_id, seq, qstring, tags=tags) + "\n")
        else:
            write_fastq(read_id, seq, qstring, fd=self.fd, tags=tags)

    def end(self):
        self.fd.flush()


class DuplexBamWriter(DuplexWriter):
    """DuplexWriter to BAM: the records of its SAM mode, encoded by bonito_b200.bam onto the binary file `fd`."""

    def __init__(self, iterator, fd=None, min_qscore=0, device="cuda", members_per_launch=256):
        super().__init__(iterator, fd=fd if fd is not None else sys.stdout.buffer, min_qscore=min_qscore, mode="w")
        self.device, self.members_per_launch = device, members_per_launch

    def begin(self):
        self.bam = BamOutput(self.fd, sam_header(), device=self.device, members_per_launch=self.members_per_launch)

    def write_read(self, read_id, seq, qstring, tags):
        self.bam.write_sam(sam_record(read_id, seq, qstring, tags=tags))

    def end(self):
        self.bam.close()


class Writer(Thread):
    """
    Drains the basecall iterator on its own thread; `.log` holds (read_id, num_samples) of the reads written.
    mode "wfq": FASTQ (`tags=True` puts the SAM tags on the header line as the reference does); mode "w": SAM text, aligned
    where a result carries a `mapping` (with `contigs` [(name, length)] for the @SQ header lines).
    """

    def __init__(self, iterator, fd=sys.stdout, min_qscore=0, mode="wfq", groups=(), group_key=None, tags=False,
                 contigs=None):
        super().__init__(daemon=True)
        if mode not in ("wfq", "w"):
            raise ValueError(f"output mode {mode!r} needs htslib (BAM / CRAM), which this build does not bundle: "
                             "redirect to a .sam or .fastq file")
        self.iterator, self.fd, self.min_qscore, self.mode = iterator, fd, min_qscore, mode
        self.groups, self.group_key, self.tags, self.contigs = list(groups), group_key, tags, contigs
        self.log, self.error = [], None

    def run(self):
        try:
            self.begin()
            for read, res in self.iterator:
                seq, qstring = res["sequence"], res["qstring"]
                samples = len(read.signal) + getattr(read, "trimmed_samples", 0)
                if len(seq) and mean_qscore_from_qstring(qstring) >= self.min_qscore:
                    self.write_read(read, res, seq, qstring)
                    self.log.append((read.read_id, samples))
                else:
                    sys.stderr.write(f"> skipping empty / low quality sequence {read.read_id}\n")
            self.end()
        except BaseException as err:   # surfaced by the CLI after join()
            self.error = err

    def begin(self):
        if self.mode == "w":
            self.fd.write(sam_header(self.groups, contigs=self.contigs))

    def sam_line(self, read, res, seq, qstring):
        return sam_record(read.read_id, seq, qstring, mapping=res.get("mapping"), tags=read_tags(read, res, self.group_key))

    def write_read(self, read, res, seq, qstring):
        if self.mode == "w":
            self.fd.write(self.sam_line(read, res, seq, qstring) + "\n")
        else:
            write_fastq(read.read_id, seq, qstring, fd=self.fd,
                        tags=read_tags(read, res, self.group_key, with_moves=False) if self.tags else None)

    def end(self):
        self.fd.flush()


class BamWriter(Writer):
    """Writer to BAM: the header and records of its SAM mode, encoded by bonito_b200.bam onto the binary file `fd` (the
    BGZF compression runs on `device`)."""

    def __init__(self, iterator, fd=None, device="cuda", members_per_launch=256, **kwargs):
        super().__init__(iterator, fd=fd if fd is not None else sys.stdout.buffer, mode="w", **kwargs)
        self.device, self.members_per_launch = device, members_per_launch

    def begin(self):
        self.bam = BamOutput(self.fd, sam_header(self.groups, contigs=self.contigs), self.contigs, device=self.device,
                             members_per_launch=self.members_per_launch)

    def write_read(self, read, res, seq, qstring):
        self.bam.write_sam(self.sam_line(read, res, seq, qstring))

    def end(self):
        self.bam.close()


summary_field_names = [
    "filename", "read_id", "run_id", "channel", "mux", "start_time", "duration", "template_start", "template_duration",
    "sequence_length_template", "mean_qscore_template",
    "alignment_genome", "alignment_genome_start", "alignment_genome_end", "alignment_strand_start",
    "alignment_strand_end", "alignment_direction", "alignment_length", "alignment_num_aligned", "alignment_num_correct",
    "alignment_num_insertions", "alignment_num_deletions", "alignment_num_substitutions", "alignment_mapq",
    "alignment_strand_coverage", "alignment_identity", "alignment_accuracy",
]

_CIGAR_OP = re.compile(r"(\d+)([MID])")
_TARGET_CODE = np.zeros(256, dtype=np.uint8)
_TARGET_CODE[np.frombuffer(b"ACGT", dtype=np.uint8)] = np.arange(1, 5, dtype=np.uint8)
MAX_TARGET = np.iinfo(np.uint16).max


class CtcDataError(ValueError):
    """CTC training data that cannot be written as the reference's dtypes (a target longer than uint16 counts)."""


def cigar_counts(cigar_str):
    """(M, I, D) base counts of an M / I / D CIGAR string."""
    counts = {"M": 0, "I": 0, "D": 0}
    for n, op in _CIGAR_OP.findall(cigar_str):
        counts[op] += int(n)
    return counts["M"], counts["I"], counts["D"]


def alignment_lengths(mapping):
    """(mlen, blen) of a Mapping as mappy defines them, from its CIGAR and NM: blen = M + I + D, mlen = blen - NM."""
    blen = sum(cigar_counts(mapping.cigar_str))
    return blen - mapping.NM, blen


def summary_row(read, seqlen, qscore, mapping):
    """One row of the summary TSV, a dict keyed by `summary_field_names` (reference: bonito/io.py:211-258)."""
    fields = [read.filename, read.read_id, read.run_id, read.channel, read.mux, read.start, read.duration,
              read.template_start, read.template_duration, seqlen, float(qscore)]
    if mapping is None:
        fields += ["*", -1, -1, -1, -1, "*", 0, 0, 0, 0, 0, 0, 0, 0.0, 0.0, 0.0]
    else:
        _, ins, dels = cigar_counts(mapping.cigar_str)
        correct, length = alignment_lengths(mapping)
        matches = length - ins - dels
        fwd = mapping.strand == +1
        fields += [mapping.ctg, mapping.r_st, mapping.r_en,
                   mapping.q_st if fwd else seqlen - mapping.q_en, mapping.q_en if fwd else seqlen - mapping.q_st,
                   "+" if fwd else "-", length, matches, correct, ins, dels, mapping.NM - ins - dels, mapping.mapq,
                   (mapping.q_en - mapping.q_st) / seqlen, correct / matches if matches else 0.0,
                   correct / length if length else 0.0]
    return dict(zip(summary_field_names, fields))


def typical_indices(x, n=2.5):
    """Indices of the values strictly within n standard deviations of the mean (reference: bonito/io.py:29-32).
    Deviation: when every value is the same (sd = 0) all indices are kept; the reference's strict test keeps none."""
    x = np.asarray(x)
    mu, sd = np.mean(x), np.std(x)
    if sd == 0:
        return np.arange(x.size)
    idx, = np.where((mu - n * sd < x) & (x < mu + n * sd))
    return idx


def ctc_target(refseq, strand, rna=False):
    """uint8 target of a reference span: reverse-complemented on strand -1, A C G T -> 1 2 3 4, reversed back to signal
    orientation for RNA (whose calls are reversed)."""
    if strand == -1:
        refseq = revcomp(refseq)
    target = _TARGET_CODE[np.frombuffer(refseq.encode(), dtype=np.uint8)]
    return target[::-1].copy() if rna else target


def ctc_reject(seq, mean_qscore, mapping, refseq, min_qscore=0, min_accuracy=0.99, min_coverage=0.90):
    """The reject name of a chunk call, the first of the reference's filters that holds in its order, or None when the
    chunk is kept.  `refseq` is the mapped reference span (unused when `mapping` is None)."""
    if mean_qscore < min_qscore:
        return "low_qscore"
    if not len(seq):
        return "zerolen_sequence"
    if mapping is None:
        return "no_mapping"
    mlen, blen = alignment_lengths(mapping)
    if (mlen / blen if blen else 0.0) < min_accuracy:
        return f"low_accuracy{min_accuracy:.2f}"
    if (mapping.q_en - mapping.q_st) / len(seq) < min_coverage:
        return f"low_coverage{min_coverage:.2f}"
    if "N" in refseq:
        return "N_in_sequence"
    return None


def ctc_output_paths(fd=1):
    """(directory, summary file) of the CTC training data: beside the regular file `fd` is redirected to, as
    `<stem>_summary.tsv`; otherwise (a terminal, a pipe, a device) the working directory and `summary.tsv`."""
    path = ""
    if not os.isatty(fd):
        try:
            path = realpath(f"/dev/fd/{fd}")
        except OSError:
            path = ""
    if path and not path.startswith("/proc") and os.path.isfile(path):
        return os.path.dirname(path), "%s_summary.tsv" % os.path.splitext(path)[0]
    return ".", "summary.tsv"


def _tsv_value(v):
    return repr(v) if isinstance(v, float) else str(v)


def write_summary(path, rows):
    """The summary TSV: a header line of `summary_field_names`, then one line per row dict."""
    with open(path, "w") as fh:
        fh.write("\t".join(summary_field_names) + "\n")
        for row in rows:
            fh.write("\t".join(_tsv_value(row[k]) for k in summary_field_names) + "\n")


class CtcWriter(Thread):
    """
    Writes the CTC training data of `basecaller --save-ctc` from (chunk read, result with `mapping`) pairs.  `aligner` is
    any object with `seq(name, start, end)` and `contigs` [(name, length)].  Chunks are filtered by `ctc_reject`; every
    kept chunk is written to `fd` in input order as a record without tags: SAM text with the header in mode "w", BAM
    (BGZF on `device`) in mode "wb", SAM lines without a header in mode "wfq" (the reference's pysam output with
    `add_sam_header=False`).  At the end the rows within `typical_indices` of the target lengths are saved in the order of
    `np.random.permutation` (numpy's global state, seeded by `init`) to `chunks.npy` (float16 [n, chunksize]),
    `references.npy` (uint8 [n, max length], zero-padded) and `reference_lengths.npy` (uint16 [n]) in `directory`, with
    the summary TSV `summary` filtered and permuted in step.  `.log` holds (chunk id, samples) of every chunk; `.rejected`
    the reject counts in order of first occurrence.
    """

    def __init__(self, iterator, aligner, fd=None, mode="w", min_qscore=0, min_accuracy=0.99, min_coverage=0.90,
                 rna=False, directory=None, summary=None, device="cuda", stderr=None):
        super().__init__(daemon=True)
        if mode not in ("wfq", "w", "wb"):
            raise ValueError(f"output mode {mode!r} needs htslib (CRAM), which this build does not bundle: "
                             "redirect to a .bam, .sam or .fastq file")
        if fd is None:
            fd = sys.stdout.buffer if mode == "wb" else sys.stdout
        if directory is None or summary is None:
            default_dir, default_summary = ctc_output_paths()
            directory = default_dir if directory is None else directory
            summary = default_summary if summary is None else summary
        self.iterator, self.aligner, self.fd, self.mode = iterator, aligner, fd, mode
        self.min_qscore, self.min_accuracy, self.min_coverage, self.rna = min_qscore, min_accuracy, min_coverage, rna
        self.directory, self.summary = directory, summary
        self.device = device
        self.stderr = stderr if stderr is not None else sys.stderr
        self.log, self.rejected, self.error = [], {}, None

    def run(self):
        try:
            self.begin()
            chunks, targets, rows = [], [], []
            for read, res in self.iterator:
                seq, qstring = res["sequence"], res["qstring"]
                mean_qscore = res.get("mean_qscore", mean_qscore_from_qstring(qstring))
                mapping = res.get("mapping")
                self.log.append((read.read_id, len(read.signal)))
                refseq = self.aligner.seq(mapping.ctg, mapping.r_st, mapping.r_en) if mapping and len(seq) else ""
                reason = ctc_reject(seq, mean_qscore, mapping, refseq, self.min_qscore, self.min_accuracy,
                                    self.min_coverage)
                if reason is not None:
                    self.rejected[reason] = self.rejected.get(reason, 0) + 1
                    continue
                target = ctc_target(refseq, mapping.strand, self.rna)
                if target.size > MAX_TARGET:
                    raise CtcDataError(f"chunk {read.read_id} has a {target.size}-base reference, over the {MAX_TARGET} "
                                       "that reference_lengths.npy (uint16) holds: use a smaller --chunksize")
                self.write_record(sam_record(read.read_id, seq, qstring, mapping))
                rows.append(summary_row(read, len(seq), mean_qscore, mapping))
                targets.append(target)
                chunks.append(np.asarray(read.signal, dtype=np.float16))
            self.end()
            self.save(chunks, targets, rows)
        except BaseException as err:   # surfaced by the CLI after join()
            self.error = err

    def begin(self):
        header = sam_header(contigs=self.aligner.contigs)
        if self.mode == "wb":
            self.bam = BamOutput(self.fd, header, self.aligner.contigs, device=self.device)
        elif self.mode == "w":
            self.fd.write(header)

    def write_record(self, line):
        if self.mode == "wb":
            self.bam.write_sam(line)
        else:
            self.fd.write(line + "\n")

    def end(self):
        if self.mode == "wb":
            self.bam.close()
        else:
            self.fd.flush()

    def save(self, chunks, targets, rows):
        if not chunks:
            self.stderr.write("> no suitable ctc data to write\n")
            return
        chunks = np.stack(chunks)
        lengths = np.array([t.size for t in targets], dtype=np.uint16)
        references = np.zeros((len(targets), int(lengths.max())), dtype=np.uint8)
        for row, target in zip(references, targets):
            row[:target.size] = target
        indices = np.random.permutation(typical_indices(lengths))
        chunks, references, lengths = chunks[indices], references[indices], lengths[indices]
        write_summary(self.summary, [rows[i] for i in indices])
        np.save(os.path.join(self.directory, "chunks.npy"), chunks)
        np.save(os.path.join(self.directory, "references.npy"), references)
        np.save(os.path.join(self.directory, "reference_lengths.npy"), lengths)
        self.stderr.write("> Chunks rejected from training data:\n")
        for name, count in self.rejected.items():
            self.stderr.write(f" - {name}: {count}\n")
        self.stderr.write(f"> written ctc training data to {self.directory}\n")
        self.stderr.write("  - chunks.npy with shape (%s)\n" % ",".join(map(str, chunks.shape)))
        self.stderr.write("  - references.npy with shape (%s)\n" % ",".join(map(str, references.shape)))
        self.stderr.write("  - reference_lengths.npy shape (%s)\n" % ",".join(map(str, lengths.shape)))
