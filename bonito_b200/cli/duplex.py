"""
`bonito_b200 duplex <reads> <pairs_file>` -- base-space duplex consensus of (template, complement) read pairs, with the
flag surface and the printed summary of the reference's `bonito duplex` (bonito/cli/duplex.py).  The per-pair logic is in
bonito_b200/duplex.py; the alignments of a batch of pairs run as GPU launches (b200_pair_align) on a background thread
while a pool of `--threads` host threads builds the consensus of the previous batch.

Output: FASTQ, SAM text or BAM (BGZF-compressed on the GPU), chosen by the extension stdout is redirected to; CRAM is
refused.
Input: SAM text (`.sam`), BAM (`.bam`, what `basecaller` writes when redirected to a .bam file, or any BGZF-compressed
BAM such as htslib writes; inflated on the GPU by bonito_b200.bam) or FASTQ (`.fastq` / `.fq`), chosen by the
extension.  For each read id the first record that is neither secondary (0x100) nor supplementary (0x800) is used, SEQ
and QUAL as stored (reverse-strand records included, as pysam's query_sequence gives them).  A `.bam` that is empty or
lacks the BGZF EOF marker is refused before any GPU work.  CRAM input and `--reference` (minimap2) are refused: htslib
and mappy are not bundled.  `--alignment-threads` and `--mm2-preset` only matter with `--reference` and are accepted
for compatibility.
"""

import os
import sys
from argparse import ArgumentDefaultsHelpFormatter, ArgumentParser
from concurrent.futures import ThreadPoolExecutor
from datetime import timedelta
from time import perf_counter

import numpy as np

from bonito_b200 import bam, duplex, native
from bonito_b200.io import DuplexBamWriter, DuplexWriter, biofmt
from bonito_b200.multiprocessing import thread_iter

BATCH_PAIRS = 1024               # pairs per GPU batch
BATCH_BASES = 64 << 20           # template + complement bases per GPU batch


def _fail(msg):
    sys.stderr.write(f"> error: {msg}\n")
    exit(1)


def read_format(path):
    """"sam" / "bam" / "fastq" from the extension; CRAM and anything else are refused."""
    ext = path.lower().rsplit(".", 1)[-1] if "." in os.path.basename(path) else ""
    if ext == "cram":
        raise ValueError("CRAM input needs htslib, which this build does not bundle; convert to .sam or .fastq")
    if ext in ("sam", "bam"):
        return ext
    if ext in ("fastq", "fq"):
        return "fastq"
    raise ValueError(f"cannot tell the format of {path}: expected a .sam, .bam, .fastq or .fq file")


def read_pairs(path, header=True):
    """[(template id, complement id)] of a pairs file: whitespace-separated ids, the first line a header unless header=False."""
    pairs = []
    with open(path) as fh:
        if header:
            fh.readline()
        for line in fh:
            if not line.strip():
                continue
            temp_id, comp_id = line.split()
            pairs.append((temp_id, comp_id))
    return pairs


def _sam_records(fh):
    for line in fh:
        if line.startswith("@") or not line.strip():
            continue
        f = line.rstrip("\n").split("\t")
        if int(f[1]) & 0x900:
            continue
        yield f[0], f[9], f[10]


def _fastq_records(fh):
    while True:
        head = fh.readline()
        if not head:
            return
        seq, _, qual = fh.readline().rstrip("\n"), fh.readline(), fh.readline().rstrip("\n")
        if not head.startswith("@"):
            raise ValueError(f"malformed FASTQ record header {head.strip()!r}")
        yield head[1:].split(maxsplit=1)[0] if head[1:].strip() else "", seq, qual


def read_records(path, wanted=None):
    """{read id: (sequence, qualities as uint8 Q values, or None for a QUAL of '*')} of the first primary record of each
    id (restricted to `wanted` ids when given).  BAM is inflated on the GPU."""
    fmt = read_format(path)
    if fmt == "bam":
        return bam.read_records(path, wanted)
    reads = {}
    with open(path) as fh:
        for read_id, seq, qual in (_sam_records(fh) if fmt == "sam" else _fastq_records(fh)):
            if read_id in reads or (wanted is not None and read_id not in wanted):
                continue
            if qual == "*" or seq == "*" or len(qual) != len(seq):
                reads[read_id] = (seq, None)
            else:
                reads[read_id] = (seq, np.frombuffer(qual.encode("ascii"), dtype=np.uint8) - np.uint8(33))
    return reads


def pair_input(reads, pair):
    """(temp_seq, temp_q, comp_seq, comp_q) of a pair, or None when a read is missing or has no qualities."""
    temp, comp = reads.get(pair[0]), reads.get(pair[1])
    if temp is None or comp is None or temp[1] is None or comp[1] is None:
        return None
    return temp[0], temp[1], comp[0], comp[1]


def batches(pairs, reads):
    batch, bases = [], 0
    for pair in pairs:
        inp = pair_input(reads, pair)
        size = 0 if inp is None else len(inp[0]) + len(inp[2])
        if batch and (len(batch) >= BATCH_PAIRS or bases + size > BATCH_BASES):
            yield batch
            batch, bases = [], 0
        batch.append((pair, inp))
        bases += size
    if batch:
        yield batch


def call(pairs, reads, pool, device="cuda", counts=None):
    """Yields (pair, {"sequence", "qstring"}) in input order: batches aligned on the GPU on a background thread, the
    consensus of each pair on `pool`."""
    counts = counts if counts is not None else {}

    def aligned():
        for batch in batches(pairs, reads):
            prepared = list(pool.map(duplex.prepare_pair, [inp for _, inp in batch]))
            ok = [i for i, p in enumerate(prepared) if p is not None]
            rs = duplex.align_pairs([prepared[i] for i in ok], device)
            per_pair = [None] * len(batch)
            for i, r in zip(ok, rs):
                per_pair[i] = r
                if r is None:
                    counts["over_budget"] = counts.get("over_budget", 0) + 1
            yield batch, prepared, per_pair

    def finish(args):
        prep, rs = args
        if prep is None or rs is None:
            return "", ""
        return duplex.finish(rs, *prep)

    for batch, prepared, per_pair in thread_iter(aligned()):
        for (pair, _), (seq, qstring) in zip(batch, pool.map(finish, zip(prepared, per_pair))):
            yield pair, {"sequence": seq, "qstring": qstring}


def main(args):
    if args.reference:
        _fail("--reference needs minimap2 (mappy), which this build does not bundle")
    try:
        if read_format(args.in_bam) == "bam":
            bam.check_bgzf_file(args.in_bam)
    except ValueError as err:
        _fail(str(err))
    fmt = biofmt(aligned=False)
    if fmt.mode not in ("wfq", "w", "wb"):
        _fail(f"{fmt.name} output needs htslib, which this build does not bundle; redirect to .bam, .sam or .fastq")
    sys.stderr.write(f"> outputting {fmt.aligned} {fmt.name}\n")

    pairs = read_pairs(args.duplex_pairs_file, header=not args.no_header)
    try:
        native.require()
    except native.NativeError as err:
        _fail(str(err))
    try:
        reads = read_records(args.in_bam, wanted={rid for pair in pairs for rid in pair})
    except ValueError as err:
        _fail(str(err))

    counts = {}
    t0 = perf_counter()
    with ThreadPoolExecutor(max(1, args.threads)) as pool:
        results = call(pairs, reads, pool, counts=counts)
        if fmt.mode == "wb":
            writer = DuplexBamWriter(results, min_qscore=args.min_qscore)
        else:
            writer = DuplexWriter(results, mode=fmt.mode, min_qscore=args.min_qscore)
        writer.start()
        writer.join()
    duration = perf_counter() - t0
    if writer.error is not None:
        raise writer.error
    if counts.get("over_budget"):
        sys.stderr.write(f"> {counts['over_budget']} pairs not aligned: traceback over "
                         f"{duplex.TRACE_BUDGET >> 30} GiB (empty consensus)\n")

    num_bases = sum(n for _, n in writer.log)
    sys.stderr.write("> completed reads: %s\n" % len(writer.log))
    sys.stderr.write("> duration: %s\n" % timedelta(seconds=np.round(duration)))
    sys.stderr.write("> bases per second %.1E\n" % (num_bases / duration if duration > 0 else 0.0))
    sys.stderr.write("> done\n")


def argparser():
    parser = ArgumentParser(formatter_class=ArgumentDefaultsHelpFormatter, add_help=False)
    parser.add_argument("in_bam")
    parser.add_argument("duplex_pairs_file")
    parser.add_argument("--reference")
    parser.add_argument("--min-qscore", default=0, type=int)
    parser.add_argument("--no-header", action="store_true")
    parser.add_argument("--threads", default=8, type=int)
    parser.add_argument("--alignment-threads", default=8, type=int)
    parser.add_argument("--mm2-preset", default="lr:hq", type=str)
    return parser
