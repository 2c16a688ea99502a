"""
Chunked basecalling of the QuartzNet CTC models.  With `beamsize=1`: chunk -> batchify -> native forward + per-frame greedy
step -> D2H of the labels and probabilities -> unbatchify -> stitch per read -> greedy collapse per read -> format.  With
`beamsize > 1`: the forward's `[N, T, 5]` fp16 log-probs stay on the device, are unbatchified and stitched there, and
consecutive reads are collected into groups (up to `group_frames` frames or `group_reads` reads, order kept); each group
is decoded by one launch of the prefix beam search (`bonito_b200.ctc.model.beam_search`) and copied back once.  The search
is sequential along a read, so its throughput comes from the reads a launch has in flight; the decode of a read does not
depend on the group it is in.

It yields the `{'stride', 'moves', 'qstring', 'sequence'}` contract of the CRF path, so the FASTQ / SAM writers and the
`mv:B:c` move table work unchanged.  Deliberate deviations from the reference (bonito/ctc/basecall.py):
  * `beamsize` defaults to 1, the greedy decode; the reference defaults to fast_ctc_decode's beam search of width 5.  The
    beam search here follows this project's rules (bonito_b200/csrc/ctc_beam.cu) and also yields qualities and moves,
    which the reference's has not.  It has no CPU path: a CPU model with `beamsize > 1` raises NotImplementedError.
  * Reads shorter than a chunk are cut to floor(length / stride) frames, as the CRF path's `stitch_results` does; the
    reference's CTC stitch keeps the tiled copies of the read and calls them.
  * `reverse=True` raises ValueError; the reference ignores it.
The collapse runs on the stitched per-frame arrays of the whole read, so it equals decoding the stitched log-probs: a run of
one label across a chunk join emits one base.
"""

import torch

from bonito_b200.crf.basecall import stitch_results
from bonito_b200.ctc.model import beam_search, check_alphabet, check_beamsize, greedy_collapse
from bonito_b200.multiprocessing import thread_iter
from bonito_b200.util import batchify, chunk, unbatchify


def compute_greedy(model, batch):
    """One batch [N, 1, L] (host, float32) -> {'labels': uint8 [N, T], 'probs': float32 [N, T]} on the host."""
    with torch.inference_mode():
        device = next(model.parameters()).device
        plan = model.native_plan(device)
        labels, probs = plan.greedy(batch.to(torch.float16).to(device))
        return {"labels": labels.cpu(), "probs": probs.cpu()}


def compute_logp(model, batch):
    """One batch [N, 1, L] (host, float32) -> [N, T, 5] fp16 log-probs on the device."""
    with torch.inference_mode():
        device = next(model.parameters()).device
        return model.native_plan(device).forward(batch.to(torch.float16).to(device))


# A group is decoded when the next read would take it past either budget.  One warp searches one read, so a launch lasts
# as long as its longest read and its frame rate grows with the reads in flight: scripts/bench_ctc_beam.py, width 5 on
# copies of one 20 000-frame read on an NVIDIA H100 80GB HBM3 (700 W limit), took 26.2 ms for 16 reads, 27.4 ms for 528,
# 29.8 ms for 1056 and 37.7 ms for 2112 (profiles/h100_ctc_beam_bench.json).  1024 reads is where a launch stops being
# free of charge for the reads added to it; the frame budget keeps the prefix arena (8 * beamsize bytes per frame) at
# 1 GiB for the widest beam.
GROUP_FRAMES = 4_000_000
GROUP_READS = 1024


def decode_groups(model, stitched, beamsize, threshold, group_frames, group_reads):
    """(read, [T, 5] device log-probs) pairs -> (read, {'sequence', 'qstring', 'moves'} uint8 [T] host arrays), in order."""
    def flush(group):
        with torch.inference_mode():
            offsets = [0]
            for _, logp in group:
                offsets.append(offsets[-1] + logp.shape[0])
            out = beam_search(torch.cat([logp for _, logp in group]), offsets, beamsize, threshold, model.qscale,
                              model.qbias).cpu().numpy()
        for (read, _), lo, hi in zip(group, offsets, offsets[1:]):
            yield read, {"sequence": out[0, lo:hi], "qstring": out[1, lo:hi], "moves": out[2, lo:hi]}

    group, frames = [], 0
    for read, logp in stitched:
        if group and (frames + logp.shape[0] > group_frames or len(group) >= group_reads):
            yield from flush(group)
            group, frames = [], 0
        group.append((read, logp))
        frames += logp.shape[0]
    if group:
        yield from flush(group)


def fmt(model, attrs, rna=False):
    if "labels" in attrs:
        seq, qstring, moves = greedy_collapse(attrs["labels"].numpy(), attrs["probs"].numpy(), model.alphabet, model.qscale,
                                              model.qbias)
    else:
        seq, qstring, moves = attrs["sequence"], attrs["qstring"], attrs["moves"]
    seq, qstring = seq[seq != 0].tobytes().decode(), qstring[qstring != 0].tobytes().decode()
    if rna:
        seq, qstring = seq[::-1], qstring[::-1]
    return {"stride": model.stride, "moves": moves, "qstring": qstring, "sequence": seq}


def basecall(model, reads, beamsize=1, chunksize=4000, overlap=500, batchsize=64, qscores=False, reverse=False, rna=False,
             threshold=1e-3, group_frames=GROUP_FRAMES, group_reads=GROUP_READS):
    """Basecall an iterable of reads (objects with a float32 numpy `.signal`); yields (read, result) pairs in order.
    `beamsize` in 2..32 decodes with the prefix beam search (probability cut `threshold`) in groups of reads."""
    check_beamsize(beamsize)
    if reverse:
        raise ValueError("reverse-complement basecalling (--revcomp) is not supported for the QuartzNet CTC models")
    if beamsize > 1:
        check_alphabet(model.alphabet)
        if next(model.parameters()).device.type != "cuda":
            raise NotImplementedError("CTC beam search has no CPU path: the model must be on a CUDA device (use beamsize=1 "
                                      "for the greedy decode)")
        if group_frames < 1 or group_reads < 1:
            raise ValueError("group_frames and group_reads must be at least 1")
    chunks = thread_iter(
        ((read, 0, read.signal.shape[-1]), chunk(torch.from_numpy(read.signal), chunksize, overlap)) for read in reads
    )
    batches = thread_iter(batchify(chunks, batchsize=batchsize))
    compute = compute_greedy if beamsize == 1 else compute_logp
    scores = thread_iter((keys, compute(model, batch)) for keys, batch in batches)
    results = thread_iter(
        (read, stitch_results(out, end - start, chunksize, overlap, model.stride))
        for ((read, start, end), out) in unbatchify(scores)
    )
    if beamsize > 1:
        results = thread_iter(decode_groups(model, results, beamsize, threshold, group_frames, group_reads))
    return thread_iter((read, fmt(model, attrs, rna)) for read, attrs in results)
