"""
`bonito_b200 basecaller <model_directory> <reads_directory>` -- the flag surface of the reference's
`bonito basecaller` (`bonito/cli/basecaller.py:168-199`) over the native engine.
Output is FASTQ, or SAM text with the `mv:B:c` move table when stdout is redirected to a `.sam` file, or BAM with the same
records when it is redirected to a `.bam` file, BGZF-compressed on the GPU (the reference's `biofmt` rule,
bonito/io.py:35-54); CRAM is refused.  `--reference <fasta>` maps the calls on the GPU (bonito_b200.aligner, this
project's rules in place of minimap2's) and writes aligned SAM or BAM; `--alignment-threads` is accepted and has no effect.  CTC
training-data export (`--save-ctc`) exits with an explanation.
`B200_CTC_BEAMSIZE=W` in the environment (1..32, unset = 1, the greedy decode) decodes the QuartzNet CTC models with the
prefix beam search of width W; the flag surface itself is the reference's and has no beam option.
"""

import os
import sys
from argparse import ArgumentParser, ArgumentDefaultsHelpFormatter
from datetime import timedelta
from itertools import islice
from time import perf_counter

import numpy as np

from bonito_b200.aligner import PRESETS, Aligner, IndexBuildError, align_map
from bonito_b200.ctc.model import MAX_BEAMSIZE, Model as CtcModel
from bonito_b200.io import BamWriter, Writer, biofmt
from bonito_b200.nn import fuse_bn_
from bonito_b200.reader import Reader
from bonito_b200.util import init, load_model, load_symbol


def _column_to_set(filename, idx=0):
    if not filename:
        return None
    with open(filename) as fh:
        return {line.split()[idx] for line in fh if line.strip()}


def main(args):
    init(args.seed, args.device)
    if args.save_ctc:
        sys.stderr.write("> error: --save-ctc (CTC training data) is not supported by this build\n")
        exit(1)
    if args.reference and args.mm2_preset not in PRESETS:
        sys.stderr.write(f"> error: unknown --mm2-preset '{args.mm2_preset}', choose one of {', '.join(PRESETS)}\n")
        exit(1)
    try:
        reader = Reader(args.reads_directory, args.recursive)
        sys.stderr.write("> reading %s\n" % reader.fmt)
    except FileNotFoundError:
        sys.stderr.write("> error: no suitable files found in %s\n" % args.reads_directory)
        exit(1)
    fmt = biofmt(aligned=args.reference is not None)
    if fmt.mode not in ("wfq", "w", "wb"):
        sys.stderr.write(f"> error: {fmt.name} output needs htslib, which this build does not bundle; "
                         "redirect to .bam, .sam or .fastq\n")
        exit(1)
    if args.reference and fmt.name == "fastq":
        sys.stderr.write(f"> warning: did you really want {fmt.aligned} {fmt.name}?\n")
    else:
        sys.stderr.write(f"> outputting {fmt.aligned} {fmt.name}\n")
    sys.stderr.write(f"> loading model {args.model_directory}\n")
    try:
        model = load_model(args.model_directory, args.device, weights=args.weights if args.weights > 0 else None,
                           chunksize=args.chunksize, overlap=args.overlap, batchsize=args.batchsize,
                           quantize=args.quantize, use_koi=True)
        model = model.apply(fuse_bn_)
    except FileNotFoundError:
        sys.stderr.write(f"> error: failed to load {args.model_directory}\n")
        exit(1)
    except ImportError as err:                  # a model package this build does not have
        sys.stderr.write(f"> error: no native path for this model (there is no eager fallback): {err}\n")
        exit(1)
    if args.revcomp and isinstance(model, CtcModel):
        sys.stderr.write("> error: --revcomp is not supported for the QuartzNet CTC models (dna_r9.4.1@v1, @v2)\n")
        exit(1)
    decode_args = {}
    if isinstance(model, CtcModel):
        width = os.environ.get("B200_CTC_BEAMSIZE", "1")
        if not width.isdigit() or not 1 <= int(width) <= MAX_BEAMSIZE:
            sys.stderr.write(f"> error: B200_CTC_BEAMSIZE must be an integer in 1..{MAX_BEAMSIZE}, got '{width}'\n")
            exit(1)
        decode_args["beamsize"] = int(width)
    try:
        # build the native plan now: a layer stack without a native kernel is reported here, not from the writer thread
        model.native_plan()
    except NotImplementedError as err:          # engine.UnsupportedModel
        sys.stderr.write(f"> error: no native path for this model (there is no eager fallback): {err}\n")
        exit(1)
    if args.verbose:
        sys.stderr.write(f"> model basecaller params: {model.config['basecaller']}\n")

    basecall = load_symbol(args.model_directory, "basecall")
    aligner = None
    if args.reference and fmt.name != "fastq":       # FASTQ has no alignment fields: the mapping is skipped
        sys.stderr.write("> loading reference\n")
        try:
            aligner = Aligner(args.reference, preset=args.mm2_preset, device=args.device)
        except IndexBuildError:
            sys.stderr.write("> failed to load/build index\n")
            exit(1)
    scaling = model.config.get("scaling")
    pa = bool(scaling) and scaling.get("strategy") == "pa"
    reads = reader.get_reads(
        args.reads_directory, recursive=args.recursive, read_ids=_column_to_set(args.read_ids), skip=args.skip,
        do_trim=not args.no_trim, scaling_strategy=scaling,
        norm_params=model.config.get("standardisation") if pa else model.config.get("normalisation"))
    if args.max_reads:
        reads = islice(reads, args.max_reads)

    params = model.config["basecaller"]
    results = basecall(model, reads, reverse=args.revcomp, rna=args.rna, batchsize=params["batchsize"],
                       chunksize=params["chunksize"], overlap=params["overlap"], **decode_args)
    if aligner:
        results = align_map(aligner, results, n_thread=args.alignment_threads)
    writer_args = dict(min_qscore=args.min_qscore, group_key=os.path.basename(os.path.normpath(args.model_directory)),
                       contigs=aligner.contigs if aligner else None)
    if fmt.mode == "wb":
        writer = BamWriter(results, device=args.device, **writer_args)
    else:
        writer = Writer(results, mode=fmt.mode, **writer_args)
    t0 = perf_counter()
    writer.start()
    writer.join()
    duration = perf_counter() - t0
    if writer.error is not None:
        raise writer.error
    num_samples = sum(n for _, n in writer.log)
    sys.stderr.write("> completed reads: %s\n" % len(writer.log))
    sys.stderr.write("> duration: %s\n" % timedelta(seconds=np.round(duration)))
    sys.stderr.write("> samples per second %.1E\n" % (num_samples / max(duration, 1e-9)))
    sys.stderr.write("> done\n")


def argparser():
    parser = ArgumentParser(formatter_class=ArgumentDefaultsHelpFormatter, add_help=False)
    parser.add_argument("model_directory")
    parser.add_argument("reads_directory")
    parser.add_argument("--reference")
    parser.add_argument("--read-ids")
    parser.add_argument("--device", default="cuda")
    parser.add_argument("--seed", default=25, type=int)
    parser.add_argument("--weights", default=0, type=int)
    parser.add_argument("--skip", action="store_true", default=False)
    parser.add_argument("--no-trim", action="store_true", default=False)
    parser.add_argument("--save-ctc", action="store_true", default=False)
    parser.add_argument("--revcomp", action="store_true", default=False)
    parser.add_argument("--rna", action="store_true", default=False)
    parser.add_argument("--recursive", action="store_true", default=False)
    quant = parser.add_mutually_exclusive_group(required=False)
    quant.add_argument("--quantize", dest="quantize", action="store_true")
    quant.add_argument("--no-quantize", dest="quantize", action="store_false")
    parser.set_defaults(quantize=None)
    parser.add_argument("--overlap", default=None, type=int)
    parser.add_argument("--chunksize", default=None, type=int)
    parser.add_argument("--batchsize", default=None, type=int)
    parser.add_argument("--max-reads", default=0, type=int)
    parser.add_argument("--min-qscore", default=0, type=int)
    parser.add_argument("--min-accuracy-save-ctc", default=0.99, type=float)
    parser.add_argument("--alignment-threads", default=8, type=int)
    parser.add_argument("--mm2-preset", default="lr:hq", type=str)
    parser.add_argument("-v", "--verbose", action="count", default=0)
    return parser
