"""
`bonito_b200 evaluate <model_directory> --directory <training data>` -- the accuracy of a model on a chunk dataset, with the
flag surface and the printed summary of the reference's `bonito evaluate` (bonito/cli/evaluate.py).

Each batch of chunks runs the native forward and decode; the calls are aligned to their references by one batched
Smith-Waterman launch on the GPU (`bonito_b200.align`; the scoring and tie rules are in bonito_b200/csrc/align.cu).
Deviations from the reference:
  * CTC models (QuartzNet) are decoded greedily, so their accuracies here are greedy accuracies; the reference decodes
    them with a width-5 beam search.  The package has a CTC beam search (`bonito_b200.ctc.model.beam_search`, `basecall(...,
    beamsize=W)`), but `evaluate` does not use it: its flags and outputs are the reference's and have no decode switch.
  * a chunk whose call shares no base with its reference reports accuracy 0 (the reference raises ZeroDivisionError).
  * alignment ties follow this project's rules, not parasail's (which nothing pins); among co-optimal alignments the
    counts almost never differ.
"""

import dataclasses
import os
import sys
import textwrap
import warnings
from argparse import ArgumentDefaultsHelpFormatter, ArgumentParser
from pathlib import Path

import numpy as np
import torch

from bonito_b200 import native
from bonito_b200.align import AlignResult, align_batch
from bonito_b200.ctc.model import Model as CtcModel, greedy_collapse
from bonito_b200.data import ComputeSettings, DataSettings, ModelSetup, load_data
from bonito_b200.nn import fuse_bn_
from bonito_b200.util import init, load_model

FIELDS = [f.name for f in dataclasses.fields(AlignResult)]


def _fail(msg):
    sys.stderr.write(f"> error: {msg}\n")
    exit(1)


def chunk_length(directory, dataset):
    """Sample length of the chunks `evaluate` will read from a chunks.npy directory (None for a dataset.py directory)."""
    if directory is None:
        return None
    for sub in (("validation",) if dataset == "valid" else ()) + ("",):
        path = os.path.join(directory, sub, "chunks.npy")
        if os.path.exists(path):
            return int(np.load(path, mmap_mode="r").shape[-1])
    return None


def decode_refs(targets, alphabet):
    """Label rows (1..4 index the alphabet, 0 is padding) -> reference strings, zeros dropped."""
    letters = np.frombuffer("".join(alphabet).encode(), dtype=np.uint8)
    return [letters[t[t != 0]].tobytes().decode() for t in targets]


def call_batch(model, x):
    """Native forward + decode of one batch [N, 1, L] fp16 on the device -> N strings."""
    if isinstance(model, CtcModel):
        labels, probs = model.native_plan(x.device).greedy(x)
        out = []
        for lab, prob in zip(labels.cpu().numpy(), probs.cpu().numpy()):
            seq, _, _ = greedy_collapse(lab, prob, model.alphabet)
            out.append(seq[seq != 0].tobytes().decode())
        return out
    # batch-first native scores [N, T, C]: decode_batch takes them as they are
    return model.decode_batch(model(x))


def call_chunks(model, dataloader, device):
    """(seqs, refs) of every chunk the loader yields."""
    seqs, refs = [], []
    with torch.inference_mode():
        for data, target, *_ in dataloader:
            seqs.extend(call_batch(model, data.to(torch.float16).to(device)))
            refs.extend(decode_refs(target.numpy(), model.alphabet))
    return seqs, refs


def _column(results, name):
    return np.array([getattr(r, name) for r in results], dtype=np.float64)


def _mean(values):
    """pandas' Series.mean(): NaN skipped, NaN when nothing is left; an inf stays inf."""
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        return float(np.nanmean(values)) if len(values) else float("nan")


def _ratio(a, b):
    with np.errstate(divide="ignore", invalid="ignore"):
        return a / b


def summary(results):
    """The reference's printed block, `* num_chunks` through `* ref_rclip` (rates are per-chunk ratios averaged)."""
    c = {name: _column(results, name) for name in FIELDS}
    return textwrap.dedent(f"""
        * num_chunks      {len(results)}
        * accuracy        {_mean(c['accuracy']):.2%}
        * sub-rate        {_mean(_ratio(c['num_mismatches'], c['num_correct'])):.2%}
        * ins-rate        {_mean(_ratio(c['num_insertions'], c['num_correct'])):.2%}
        * del-rate        {_mean(_ratio(c['num_deletions'], c['num_correct'])):.2%}
        * seq_len         {_mean(c['seq_len']):.1f}
        * seq_lclip       {_mean(c['align_seq_start']):.1f}
        * seq_rclip       {_mean(c['seq_len'] - c['align_seq_end'] - 1):.1f}
        * ref_len         {_mean(c['ref_len']):.1f}
        * ref_lclip       {_mean(c['align_ref_start']):.1f}
        * ref_rclip       {_mean(c['ref_len'] - c['align_ref_end'] - 1):.1f}
        """)


def summary_table(results):
    """The results as `pandas.DataFrame(results).to_csv(sep="\\t")` writes them: an index column, a header row that starts
    with a tab, and a column written as floats when any of its values is a float (pandas' dtype inference)."""
    as_float = {name: any(isinstance(getattr(r, name), float) for r in results) for name in FIELDS}
    lines = ["\t" + "\t".join(FIELDS)]
    for i, r in enumerate(results):
        values = (repr(float(getattr(r, name))) if as_float[name] else str(int(getattr(r, name))) for name in FIELDS)
        lines.append(f"{i}\t" + "\t".join(values))
    return "\n".join(lines) + "\n"


def write_outputs(output_dir, seqs, refs, results):
    output_dir.mkdir(exist_ok=True, parents=True)
    with (output_dir / "seqs.fasta").open("w") as fh:
        fh.write("".join(f">chunk_{i}\n{s}\n" for i, s in enumerate(seqs)))
    with (output_dir / "refs.fasta").open("w") as fh:
        fh.write("".join(f">chunk_{i}\n{s}\n" for i, s in enumerate(refs)))
    with (output_dir / "summ.txt").open("w") as fh:
        fh.write(summary_table(results))


def main(args):
    init(args.seed, args.device)
    print(f"* loading model from: {args.model_directory}/weights_{args.weights}.tar")
    try:
        model = load_model(args.model_directory, args.device, weights=args.weights, batchsize=args.batchsize,
                           chunksize=chunk_length(args.directory, args.dataset), use_koi=True)
        model = model.apply(fuse_bn_)
        # build the native plan now: a layer stack without a native kernel is reported here
        model.native_plan()
    except FileNotFoundError as err:
        _fail(f"failed to load {args.model_directory}: {err}")
    except (ImportError, NotImplementedError, native.NativeError) as err:
        _fail(f"no native path for this model (there is no eager fallback): {err}")

    standardisation = model.config.get("standardisation", {}) if args.standardise else {}
    model_setup = ModelSetup(n_pre_context_bases=getattr(model, "n_pre_context_bases", 0),
                             n_post_context_bases=getattr(model, "n_post_context_bases", 0),
                             standardisation=standardisation)
    print(f"* * applying standardisation params: mean={standardisation.get('mean', 0.0)}, "
          f"stdev={standardisation.get('stdev', 1.0)}")

    print("* loading data")
    # no worker processes: the parent already holds a CUDA context, and the chunks are in memory
    compute = ComputeSettings(batch_size=args.batchsize, num_workers=0, seed=args.seed)
    if args.dataset == "valid":
        # the validation set may be a subset of the training set: ask for enough training chunks to take it from
        _, valid_loader = load_data(DataSettings(args.directory, args.chunks * 100, args.chunks, None),
                                    model_setup, compute)
        dataloader = valid_loader
    else:
        dataloader, _ = load_data(DataSettings(args.directory, args.chunks, args.chunks, None), model_setup, compute)

    print("* calling")
    try:
        seqs, refs = call_chunks(model, dataloader, args.device)
    except (NotImplementedError, native.NativeError) as err:
        _fail(f"no native path for these chunks (there is no eager fallback): {err}")
    results = align_batch(refs, seqs, args.device)

    print("* aligning")
    print(summary(results))

    if args.output_dir:
        write_outputs(args.output_dir, seqs, refs, results)


def argparser():
    parser = ArgumentParser(formatter_class=ArgumentDefaultsHelpFormatter, add_help=False)
    parser.add_argument("model_directory")
    parser.add_argument("--output_dir", type=Path)
    parser.add_argument("--directory", type=Path)
    parser.add_argument("--dataset", choices=["train", "valid"], default="valid")
    parser.add_argument("--device", default="cuda")
    parser.add_argument("--seed", default=9, type=int)
    parser.add_argument("--weights", default=0, type=None)
    parser.add_argument("--chunks", default=512, type=int)
    parser.add_argument("--batchsize", default=256, type=int)
    parser.add_argument("--standardise", action="store_true", default=False)
    return parser
