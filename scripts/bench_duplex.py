"""
Time `duplex` on one GPU and print one JSON line (written to --out as well):

  * pair sets: templates of 10 kb and 30 kb, each complement the reverse complement of an independently mutated copy of
    the same truth, at two edit profiles (2 / 1 / 1 % and 5 / 3 / 3 % substitution / insertion / deletion per strand);
    seeded, random qualities;
  * per set: GPU kernel milliseconds per mode (CUDA events around every b200_pair_align launch), the cells computed
    (GLOBAL_EDIT: band cells of every pass, the score-only doubling passes and the traceback pass; SEMIGLOBAL_AFFINE: m * n)
    and G cells/s over the kernel time, the histogram of GLOBAL_EDIT passes per pair (initial band EDIT_BAND0);
  * per set, steps run one after the other: host preparation, GPU alignment (uploads, launches, copies and the end
    re-alignment glue) and host consensus, in seconds; then the CLI's overlapped path (GPU batches on a background thread,
    consensus on an 8-thread pool): pairs/s and consensus bases/s;
  * the GPU name and power limit, read in the same run.

    python scripts/bench_duplex.py [--repeat 2] [--out profiles/h100_duplex_bench.json]
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bonito_b200 import duplex as D  # noqa: E402
from bonito_b200.align import EDIT_BAND0  # noqa: E402
from bonito_b200.cli import duplex as cli  # noqa: E402

SETS = [  # (name, template length, pairs, (sub, ins, del))
    ("10kb_2-1-1", 10_000, 128, (0.02, 0.01, 0.01)),
    ("10kb_5-3-3", 10_000, 128, (0.05, 0.03, 0.03)),
    ("30kb_2-1-1", 30_000, 32, (0.02, 0.01, 0.01)),
    ("30kb_5-3-3", 30_000, 32, (0.05, 0.03, 0.03)),
]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--id=%d" % torch.cuda.current_device(), "--query-gpu=name,power.limit",
                        "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().split("\n")[0]
    name, power = [v.strip() for v in q.split(",")]
    return dict(gpu=name, power_limit=power)


def mutate(rng, s, sub, ins, dele):
    a = np.frombuffer(s.encode(), dtype=np.uint8)
    x = rng.random(len(a))
    subs = np.frombuffer(b"ACGT", dtype=np.uint8)[(np.searchsorted(np.frombuffer(b"ACGT", dtype=np.uint8), a)
                                                     + rng.integers(1, 4, len(a))) % 4]
    out = np.where(x < sub, subs, a)
    keep = ~((x >= sub + ins) & (x < sub + ins + dele))
    extra = (x >= sub) & (x < sub + ins)
    reps = keep.astype(np.int64) + extra
    res = np.repeat(out, reps)
    ins_pos = np.cumsum(reps)[extra] - 1
    res[ins_pos] = np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, len(ins_pos))]
    return res.tobytes().decode()


def make_set(length, n, profile, seed):
    rng = np.random.default_rng(seed)
    pairs = []
    for _ in range(n):
        truth = np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, length)].tobytes().decode()
        t = mutate(rng, truth, *profile)
        c = D.revcomp(mutate(rng, truth, *profile))
        pairs.append((t, rng.integers(5, 40, len(t)).astype(np.uint8), c, rng.integers(5, 40, len(c)).astype(np.uint8)))
    return pairs


def run_set(pairs, repeat):
    best = None
    for _ in range(repeat):
        stats = {}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        prepared = [D.prepare_pair(p) for p in pairs]
        t1 = time.perf_counter()
        rs = D.align_pairs(prepared, stats=stats)
        t2 = time.perf_counter()
        calls = [D.finish(r, *p) for r, p in zip(rs, prepared)]
        t3 = time.perf_counter()
        if best is None or t3 - t0 < best[0]:
            best = (t3 - t0, t1 - t0, t2 - t1, t3 - t2, stats, calls)
    total, prep_s, align_s, cons_s, stats, calls = best
    bases = sum(len(s) for s, _ in calls)
    hist = {str(k): v for k, v in sorted(stats["pass_histogram"].items())}
    return dict(
        pairs=len(pairs), mean_template_len=round(float(np.mean([len(p[0]) for p in pairs])), 1),
        edit_kernel_ms=round(stats["edit_ms"], 2), edit_launches=stats["edit_passes"], edit_cells=int(stats["edit_cells"]),
        edit_gcells_per_s=round(stats["edit_cells"] / (stats["edit_ms"] / 1e3) / 1e9, 2) if stats["edit_ms"] else None,
        affine_kernel_ms=round(stats.get("affine_ms", 0.0), 2), affine_launches=stats.get("affine_launches", 0),
        affine_cells=int(stats.get("affine_cells", 0)),
        affine_gcells_per_s=(round(stats["affine_cells"] / (stats["affine_ms"] / 1e3) / 1e9, 2)
                             if stats.get("affine_ms") else None),
        edit_pass_histogram=hist,
        sequential_s=dict(prepare=round(prep_s, 3), gpu_alignment=round(align_s, 3), host_consensus=round(cons_s, 3),
                          total=round(total, 3)),
        consensus_bases=bases, empty_consensus=sum(1 for s, _ in calls if not s)), calls


def run_overlapped(pairs, calls_ref, threads=8):
    ids = [(f"t{i}", f"c{i}") for i in range(len(pairs))]
    reads = {}
    for (tid, cid), (t, tq, c, cq) in zip(ids, pairs):
        reads[tid], reads[cid] = (t, tq), (c, cq)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with ThreadPoolExecutor(threads) as pool:
        out = [(res["sequence"], res["qstring"]) for _, res in cli.call(ids, reads, pool)]
    dt = time.perf_counter() - t0
    assert out == calls_ref, "the overlapped path computed a different consensus"
    bases = sum(len(s) for s, _ in out)
    return dict(threads=threads, wall_s=round(dt, 3), pairs_per_s=round(len(pairs) / dt, 2),
                consensus_bases_per_s=round(bases / dt, 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_duplex.py needs a CUDA device")
    warm = make_set(2000, 8, (0.05, 0.03, 0.03), seed=1)
    run_set(warm, 1)                                       # module load, allocator
    res = dict(gpu_info(), edit_band0=EDIT_BAND0, trace_budget_bytes=D.TRACE_BUDGET, sets={})
    for n, (name, length, count, profile) in enumerate(SETS):
        pairs = make_set(length, count, profile, seed=100 + n)
        r, calls = run_set(pairs, args.repeat)
        r["overlapped"] = run_overlapped(pairs, calls)
        res["sets"][name] = r
        print(name, json.dumps(r), file=sys.stderr)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
