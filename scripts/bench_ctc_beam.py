"""
Time the CTC prefix beam search (b200_ctc_beam_search) and the whole `basecall` of the QuartzNet CTC models with it, beside
the greedy decode, on one GPU.  Seeded dna_r9.4.1@v1 and @v2 weights; --reads reads (default 64) of 30 000 to 300 000
samples, chunks of 3999 with overlap 498, batch 64.  Prints one JSON line:

  * per model and decode (greedy, beam width 5, beam width 32): `basecall` wall time (median of --steps runs after --warmup
    runs, the decodes alternating within every round) and samples/s;
  * per model and width: the beam search launch on the stitched log-probs of all the reads as one group (CUDA events around
    --steps launches after --warmup launches): ms per launch, frames/s, and that time as a share of the `basecall` run;
  * the agreement of the width-5 calls with the greedy calls (mean identity of `align_batch` over the first 50 000 bases);
  * a sweep of the reads in flight: width 5 on 16 .. 2048 copies of one 20 000-frame read, ms per launch and frames/s, which
    is what the group size of `bonito_b200.ctc.basecall` is chosen from;
  * the GPU name and power limit read in the same run.

    python scripts/bench_ctc_beam.py [--reads 64] [--steps 3] [--warmup 1] [--out profiles/h100_ctc_beam_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bonito_b200 import native, synth  # noqa: E402
from bonito_b200.align import align_batch  # noqa: E402
from bonito_b200.crf.basecall import stitch_results  # noqa: E402
from bonito_b200.ctc.basecall import basecall  # noqa: E402
from bonito_b200.ctc.model import Model  # noqa: E402
from bonito_b200.util import chunk  # noqa: E402

CHUNK, OVERLAP, BATCH = 3999, 498, 64
DECODES = (("greedy", 1), ("beam5", 5), ("beam32", 32))


class Read:
    def __init__(self, rid, signal):
        self.read_id, self.signal = rid, signal


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().split("\n")[0]
    name, power, clock = [v.strip() for v in q.split(",")]
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def make_reads(n):
    rng = np.random.default_rng(17)
    sig = synth.squiggle(8, 300_000, seed=33)[:, 0].numpy()
    return [Read(f"r{i}", sig[i % 8, :int(rng.integers(30_000, 300_001))].copy()) for i in range(n)]


def time_launches(logp, off, ln, width, steps, warmup):
    """ms per b200_ctc_beam_search launch over the packed reads (CUDA events)."""
    frames = logp.shape[0]
    ws = torch.empty(native.ctc_beam_workspace_bytes(len(ln), int(ln.sum()), width), dtype=torch.uint8, device="cuda")
    out = torch.empty(3, frames, dtype=torch.uint8, device="cuda")
    ms = []
    for i in range(warmup + steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        native.ctc_beam_search(logp, off, ln, width, 1e-3, 1.0, 0.0, ws, out[0], out[1], out[2])
        b.record()
        torch.cuda.synchronize()
        if i >= warmup:
            ms.append(a.elapsed_time(b))
    return sorted(ms)[len(ms) // 2]


def bench_model(version, reads, steps, warmup):
    spec = synth.quartznet_spec(version)
    m = Model(synth.quartznet_config(spec))
    m.load_state_dict(synth.make_quartznet_weights(spec, seed={"v1": 51, "v2": 52}[version]))
    m.use_koi(batchsize=BATCH, chunksize=CHUNK, quantize=False)
    m = m.half().eval().to("cuda")
    samples = sum(len(r.signal) for r in reads)
    times = {name: [] for name, _ in DECODES}
    calls = {}
    for rnd in range(warmup + steps):
        for name, width in DECODES:                      # the decodes alternate within every round
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = list(basecall(m, iter(reads), beamsize=width, chunksize=CHUNK, overlap=OVERLAP, batchsize=BATCH))
            torch.cuda.synchronize()
            if rnd >= warmup:
                times[name].append(time.perf_counter() - t0)
            calls[name] = [r["sequence"] for _, r in res]
    out = dict(model=f"dna_r9.4.1@{version}", reads=len(reads), samples=samples, bases_greedy=sum(map(len, calls["greedy"])))
    wall = {name: sorted(v)[len(v) // 2] for name, v in times.items()}
    for name, _ in DECODES:
        out[name] = dict(basecall_s=round(wall[name], 3), samples_per_s=round(samples / wall[name]))
    # the launch alone, on the stitched log-probs of every read as one group (what the default group budgets give here)
    plan = m.native_plan()
    stitched = []
    with torch.inference_mode():
        for r in reads:
            sig = torch.from_numpy(r.signal)
            logp = torch.cat([plan.forward(c.half().cuda()) for c in chunk(sig, CHUNK, OVERLAP).split(BATCH)])
            stitched.append(stitch_results(logp, len(r.signal), CHUNK, OVERLAP, m.stride))
        ln = np.array([s.shape[0] for s in stitched], dtype=np.int32)
        off = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.int64)
        packed = torch.cat(stitched).contiguous()
        del stitched
        for name, width in DECODES[1:]:
            ms = time_launches(packed, off, ln, width, steps, warmup)
            out[name].update(kernel_ms_per_launch=round(ms, 2), kernel_frames_per_s=round(int(ln.sum()) / (ms / 1e3)),
                             kernel_share_of_basecall=round(ms / 1e3 / wall[name], 3))
    ident = [a.accuracy for a in align_batch([g[:50_000] for g in calls["greedy"]], [b[:50_000] for b in calls["beam5"]])]
    out["beam5_identity_to_greedy"] = round(float(np.mean(ident)), 4)
    out["frames"] = int(ln.sum())
    return out, packed[:20_000].clone()


def sweep(read, steps, warmup):
    """Width 5 on R copies of one 20 000-frame read: the kernel's frame rate against the reads in flight."""
    rows = []
    T = read.shape[0]
    for R in (16, 64, 132, 264, 528, 1056, 2112):
        logp = read.repeat(R, 1).contiguous()
        ln = np.full(R, T, dtype=np.int32)
        off = (np.arange(R) * T).astype(np.int64)
        ms = time_launches(logp, off, ln, 5, steps, warmup)
        rows.append(dict(reads=R, ms_per_launch=round(ms, 2), frames_per_s=round(R * T / (ms / 1e3))))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=64)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ctc_beam.py needs a CUDA device")
    reads = make_reads(args.reads)
    results, one = [], None
    for version in ("v1", "v2"):
        res, one = bench_model(version, reads, args.steps, args.warmup)
        results.append(res)
    res = dict(gpu_info(), chunksize=CHUNK, overlap=OVERLAP, batchsize=BATCH, results=results,
               reads_in_flight_width5=sweep(one, args.steps, args.warmup))
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
