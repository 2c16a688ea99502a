"""
pysam-free output for `bonito_b200 basecaller` and `duplex`: FASTQ, SAM text (unaligned, or aligned by
bonito_b200.aligner) and BAM, with the reference's header, record and tag layout (`bonito/io.py:41-166,400-469`,
`documentation/SAM.md`), including the sequence-to-signal move table `mv:B:c,<stride>,<moves...>` (`io.py:57-70,455-456`).
The reference writes through pysam / htslib.  Here BAM records are the binary encoding of the SAM lines this module
builds (bonito_b200.bam), BGZF-compressed on the GPU; CRAM needs htslib, which this build does not bundle, so it is refused
with an explanation instead of being approximated.
Deviation: on the reverse strand QUAL is reversed along with SEQ, as the SAM specification requires; the reference
reverse-complements SEQ and leaves QUAL as called.
"""

import os
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
