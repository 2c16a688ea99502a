"""
Chunked basecalling of the QuartzNet CTC models: chunk -> batchify -> native forward + per-frame greedy step -> D2H of the
labels and probabilities -> unbatchify -> stitch per read -> greedy collapse per read -> format.

It yields the `{'stride', 'moves', 'qstring', 'sequence'}` contract of the CRF path, so the FASTQ / SAM writers and the
`mv:B:c` move table work unchanged.  Deliberate deviations from the reference (bonito/ctc/basecall.py):
  * `beamsize` defaults to 1, the greedy decode; the CTC prefix beam search is not implemented and `beamsize > 1` raises
    NotImplementedError.  The reference defaults to a beam search of width 5.
  * Reads shorter than a chunk are cut to floor(length / stride) frames, as the CRF path's `stitch_results` does; the
    reference's CTC stitch keeps the tiled copies of the read and calls them.
  * `reverse=True` raises ValueError; the reference ignores it.
The collapse runs on the stitched per-frame arrays of the whole read, so it equals decoding the stitched log-probs: a run of
one label across a chunk join emits one base.
"""

import torch

from bonito_b200.crf.basecall import stitch_results
from bonito_b200.ctc.model import greedy_collapse
from bonito_b200.multiprocessing import thread_iter
from bonito_b200.util import batchify, chunk, unbatchify


def compute_greedy(model, batch):
    """One batch [N, 1, L] (host, float32) -> {'labels': uint8 [N, T], 'probs': float32 [N, T]} on the host."""
    with torch.inference_mode():
        device = next(model.parameters()).device
        plan = model.native_plan(device)
        labels, probs = plan.greedy(batch.to(torch.float16).to(device))
        return {"labels": labels.cpu(), "probs": probs.cpu()}


def fmt(model, attrs, rna=False):
    seq, qstring, moves = greedy_collapse(attrs["labels"].numpy(), attrs["probs"].numpy(), model.alphabet, model.qscale,
                                          model.qbias)
    seq, qstring = seq[seq != 0].tobytes().decode(), qstring[qstring != 0].tobytes().decode()
    if rna:
        seq, qstring = seq[::-1], qstring[::-1]
    return {"stride": model.stride, "moves": moves, "qstring": qstring, "sequence": seq}


def basecall(model, reads, beamsize=1, chunksize=4000, overlap=500, batchsize=64, qscores=False, reverse=False, rna=False):
    """Basecall an iterable of reads (objects with a float32 numpy `.signal`); yields (read, result) pairs in order."""
    if beamsize != 1:
        raise NotImplementedError("CTC beam search is not implemented; use beamsize=1")
    if reverse:
        raise ValueError("reverse-complement basecalling (--revcomp) is not supported for the QuartzNet CTC models")
    chunks = thread_iter(
        ((read, 0, read.signal.shape[-1]), chunk(torch.from_numpy(read.signal), chunksize, overlap)) for read in reads
    )
    batches = thread_iter(batchify(chunks, batchsize=batchsize))
    scores = thread_iter((keys, compute_greedy(model, batch)) for keys, batch in batches)
    results = thread_iter(
        (read, stitch_results(out, end - start, chunksize, overlap, model.stride))
        for ((read, start, end), out) in unbatchify(scores)
    )
    return thread_iter((read, fmt(model, attrs, rna)) for read, attrs in results)
