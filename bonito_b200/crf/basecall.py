"""
Chunked basecalling: chunk -> batch -> forward -> decode -> stitch -> format.

Same generator graph and result contract as `bonito/crf/basecall.py:13-82`; the
forward pass and the decoder are the sm_90a kernels behind `model(...)` and
`bonito_b200.decode.beam_search`.  Host staging differs from the reference in one respect that does not
change results: the fp16 cast happens into a pinned buffer and the copy is asynchronous.
"""

import numpy as np
import torch

from bonito_b200 import native
from bonito_b200.decode import beam_search, to_str
from bonito_b200.multiprocessing import thread_iter
from bonito_b200.util import chunk, stitch, batchify, unbatchify


def stitch_results(results, length, size, overlap, stride, reverse=False):
    """Stitch per-chunk results of one read (dicts are stitched key by key)."""
    if isinstance(results, dict):
        return {k: stitch_results(v, length, size, overlap, stride, reverse=reverse) for k, v in results.items()}
    if length < size:
        return results[0, :int(np.floor(length / stride))]
    return stitch(results, size, overlap, length, stride, reverse=reverse)


_PINNED = {}   # (shape) -> [buffers, next index]: cudaHostAlloc costs milliseconds, so staging buffers are reused


def _stage_to_device(batch, device):
    """fp16 cast into pinned memory + async H2D (reference: `batch.to(torch.float16).to(device)`)."""
    if torch.device(device).type != "cuda":
        return batch.to(torch.float16).to(device)
    key = tuple(batch.shape)
    if key not in _PINNED:
        if len(_PINNED) > 8:
            _PINNED.clear()
        _PINNED[key] = [[torch.empty(batch.shape, dtype=torch.float16, pin_memory=True) for _ in range(2)], 0]
    bufs, idx = _PINNED[key]
    _PINNED[key][1] = idx ^ 1          # two buffers: the copy of batch i may still be in flight while i+1 is cast
    pinned = bufs[idx]
    pinned.copy_(batch)
    return pinned.to(device, non_blocking=True)


def compute_scores(model, batch, beam_width=32, beam_cut=100.0, scale=1.0, offset=0.0, blank_score=2.0,
                   reverse=False):
    """Forward + decode of one batch -> {'moves','qstring','sequence'} (CPU uint8 [N, T] each)."""
    with torch.inference_mode():
        device = next(model.parameters()).device
        scores = model(_stage_to_device(batch, device))
        if reverse:
            # reverse_complement is defined on the blank-expanded [T, N, C] layout
            scores = _revcomp_native(model, scores, blank_score)
        with torch.cuda.device(scores.device):
            sequence, qstring, moves = beam_search(
                scores, beam_width=beam_width, beam_cut=beam_cut, scale=scale, offset=offset, blank_score=blank_score)
        return {"moves": moves, "qstring": qstring, "sequence": sequence}


_STREAMS = {}


def _own_stream(device, role):
    """One CUDA stream per (device, role) for the life of the process, created through the library (`native.new_stream`):
    the batches in flight and the copy engine need streams that are really distinct, which pooled torch streams are not."""
    key = (torch.device(device).index or 0, role)
    if key not in _STREAMS:
        _STREAMS[key] = native.new_stream(device)
    return _STREAMS[key]


class _Stage:
    """Pinned fp16 staging of one input batch and the event of the H2D copy that last read it."""

    def __init__(self, shape):
        self.buf = torch.empty(shape, dtype=torch.float16, pin_memory=True)
        self.copied = None


class _Slot:
    """One in-flight batch on the device: device input, device + pinned result arrays, two events, and the CUDA stream the
    batch's kernels are enqueued on (one per slot: consecutive batches overlap on the device)."""

    def __init__(self, shape, device, index=0):
        self.index = index
        self.stream = _own_stream(device, "slot%d" % index)
        self.dev_in = torch.empty(shape, dtype=torch.float16, device=device)
        self.dev_out = self.pinned_out = None          # uint8 [3, N, T] (moves, sequence, qstring), sized on first use
        self.in_ready, self.done = torch.cuda.Event(), torch.cuda.Event()
        self.key = None


def score_batches(model, batches, depth=2, beam_width=32, beam_cut=100.0, scale=1.0, offset=0.0, blank_score=2.0,
                  reverse=False):
    """
    `compute_scores` over an iterable of (key, float32 host batch), yielding (key, result) in order, as a `depth`-deep
    pipeline: the fp16 cast + H2D copy of batch k+1 (copy stream) and the D2H copy of batch k-1 overlap the kernels of
    batch k, the host does not wait for the GPU before the next batch is enqueued, and every slot runs on its own CUDA
    stream with its own buffer set of the native plan, so the kernels of consecutive batches overlap as well (the decode
    and the GEMMs of one batch fill the SMs the recurrent clusters of the other leave free).  This is the loop
    `basecall()` runs (the reference overlaps host stages with a background thread, bonito/crf/basecall.py:70-72);
    results are identical to calling `compute_scores` batch by batch.
    """
    from bonito_b200.decode import _decoder
    device = next(model.parameters()).device
    if device.type != "cuda":
        raise RuntimeError("bonito_b200 needs a CUDA device (there is no CPU path)")
    rings, pending = {}, []          # input shape -> [slots, next]; FIFO of slots whose results are not handed out yet
    copy_stream = _own_stream(device, "copy")
    # several batches in flight need one buffer set of the native plan per slot; plans without slots (the generic-layout
    # LSTM path of the narrow models) run their batches back to back on the slots' streams
    multi_slot = _supports_slots(model, device)

    def result_of(slot):
        slot.done.synchronize()
        moves, sequence, qstring = slot.pinned_out.clone().unbind(0)    # the pinned buffer is reused `depth` batches later
        return slot.key, {"moves": moves, "qstring": qstring, "sequence": sequence}

    def enqueue(slot, key, stage):
        with torch.inference_mode(), torch.cuda.device(device):
            slot.key = key
            with torch.cuda.stream(copy_stream):
                slot.dev_in.copy_(stage.buf, non_blocking=True)
                slot.in_ready.record(copy_stream)
                stage.copied = slot.in_ready
            with torch.cuda.stream(slot.stream):
                main = slot.stream
                main.wait_event(slot.in_ready)
                scores = model(slot.dev_in, slot=slot.index) if multi_slot else model(slot.dev_in)
                if reverse:
                    scores = _revcomp_native(model, scores, blank_score)
                n, t, c = scores.shape
                if slot.dev_out is None:
                    slot.dev_out = torch.empty(3, n, t, dtype=torch.uint8, device=device)
                    slot.pinned_out = torch.empty(3, n, t, dtype=torch.uint8, pin_memory=True)
                _decoder(scores, model.seqdist.state_len, blank_score=blank_score, qscale=scale, qbias=offset, out=slot.dev_out,
                         slot=slot.index)
                slot.pinned_out.copy_(slot.dev_out, non_blocking=True)
                slot.done.record(main)

    for key, batch in batches:
        shape = tuple(batch.shape)
        if shape not in rings:
            if len(rings) > 4:                       # many geometries seen: hand out what is in flight, drop old staging
                while pending:
                    yield result_of(pending.pop(0))
                rings.clear()
            # depth device slots, depth + 1 pinned input buffers: the host converts and stages batch k + depth while `depth`
            # batches are on the device, instead of starting on it only when a slot has drained
            rings[shape] = [[_Slot(shape, device, index=i) for i in range(depth)], 0, [_Stage(shape) for _ in range(depth + 1)], 0]
            if not multi_slot:                       # one shared stream: the batches serialise on the device
                for sl in rings[shape][0][1:]:
                    sl.stream = rings[shape][0][0].stream
            # the new device buffers may reuse memory that kernels already enqueued on the compute stream still touch (the
            # caching allocator only orders reuse on the allocating stream): the copy stream must not write them earlier
            with torch.cuda.device(device):
                copy_stream.wait_stream(torch.cuda.current_stream())
                for sl in rings[shape][0]:
                    sl.stream.wait_stream(torch.cuda.current_stream())
        ring = rings[shape]
        stage = ring[2][ring[3]]
        ring[3] = (ring[3] + 1) % (depth + 1)
        if stage.copied is not None:                 # its last H2D copy (depth + 1 batches ago) has long completed
            stage.copied.synchronize()
        stage.buf.copy_(batch)                       # fp32 -> fp16 on the host, as the reference does (batch.half())
        slot = ring[0][ring[1]]
        ring[1] = (ring[1] + 1) % depth
        while any(p is slot for p in pending):       # the slot's previous batch is handed out before the slot is reused
            yield result_of(pending.pop(0))
        enqueue(slot, key, stage)
        pending.append(slot)
    while pending:
        yield result_of(pending.pop(0))


def _supports_slots(model, device):
    """True when the model's native plan keeps independent buffer sets per slot (tile-layout LSTM path, transformer)."""
    try:
        plan = model.native_plan(device)
    except Exception:
        return False
    return bool(getattr(plan, "supports_slots", False))


def _revcomp_native(model, scores, blank_score):
    """[N,T,C] -> reverse-complemented [N,T,C] through the reference's [T,N,C+blanks] definition.  Fixed-blank scores (no
    blank column) are padded with `blank_score` and unpadded again; learned-blank scores already are that layout."""
    n, t, c = scores.shape
    nb = model.seqdist.n_base
    if c == model.seqdist.n_score():
        return model.seqdist.reverse_complement(scores.permute(1, 0, 2)).permute(1, 0, 2).contiguous()
    full = torch.nn.functional.pad(scores.permute(1, 0, 2).reshape(t, n, c // nb, nb), (1, 0), value=blank_score)
    rc = model.seqdist.reverse_complement(full.reshape(t, n, -1)).reshape(t, n, c // nb, nb + 1)
    return rc[..., 1:].reshape(t, n, c).permute(1, 0, 2).contiguous()


def fmt(stride, attrs, rna=False):
    flip = (lambda s: s[::-1]) if rna else (lambda s: s)
    return {
        "stride": stride,
        "moves": attrs["moves"].numpy(),
        "qstring": flip(to_str(attrs["qstring"])),
        "sequence": flip(to_str(attrs["sequence"])),
    }


def basecall(model, reads, chunksize=4000, overlap=100, batchsize=32, reverse=False, rna=False,
             qscore_calibration=False):
    """
    Basecall an iterable of reads (objects with a float32 numpy `.signal`).

    Like the reference (`bonito/crf/basecall.py:58-82`, which calls `compute_scores` with `reverse=` only) the quality
    strings use scale 1.0 / offset 0.0.  `qscore_calibration=True` is an opt-in DEVIATION: it applies the `[qscore]`
    scale / bias of the model config, which the reference's basecaller ignores.
    """
    qscale, qbias = 1.0, 0.0
    if qscore_calibration and hasattr(model, "config"):
        qscale = float(model.config.get("qscore", {}).get("scale", 1.0))
        qbias = float(model.config.get("qscore", {}).get("bias", 0.0))

    chunks = thread_iter(
        ((read, 0, read.signal.shape[-1]), chunk(torch.from_numpy(read.signal), chunksize, overlap))
        for read in reads
    )
    batches = thread_iter(batchify(chunks, batchsize=batchsize))
    scores = thread_iter(score_batches(model, batches, reverse=reverse, scale=qscale, offset=qbias))
    results = thread_iter(
        (read, stitch_results(out, end - start, chunksize, overlap, model.stride, reverse))
        for ((read, start, end), out) in unbatchify(scores)
    )
    return thread_iter((read, fmt(model.stride, attrs, rna)) for read, attrs in results)
