"""
Benchmark of GPU read mapping (bonito_b200.aligner) -> one JSON file (default profiles/h100_map_bench.json):

- the index build of a seeded 100 Mb reference (FASTA parse + minimizers + sort, seconds);
- map_batch throughput (reads/s, Mbases/s) for 10 kb and 30 kb reads at 2/1/1 % and 5/3/3 % sub/ins/del, half of them on
  the reverse strand, timed over a warmed-up batch with a device synchronise at the end;
- kernel milliseconds per stage of one such batch, from torch.profiler (a separate run);
- `basecaller` samples/s of a synthetic hac model on the same reads without and with `--reference` (the reference is
  built from the calls of the first run), alternated twice.

Usage: python scripts/bench_map.py [--out profiles/h100_map_bench.json] [--genome-mb 100]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bonito_b200 import aligner as A          # noqa: E402
from test_gpu_map import _fasta, _mutate, _rand, _rc  # noqa: E402


def _reads(rng, genome, n, length, rates):
    reads = []
    for t in range(n):
        st = int(rng.integers(0, len(genome) - length))
        r = _mutate(rng, genome[st:st + length], *rates)
        reads.append((_rc(r) if t % 2 else r).tobytes())
    return reads


def _kernel_ms(al, reads):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        al.map_batch(reads)
        torch.cuda.synchronize()
    stages = {}
    for ev in prof.key_averages():
        if ev.device_type.name != "CUDA":
            continue
        name = ev.key
        stage = next((s for s in ("kmer_kernel", "window_kernel", "anchor_kernel", "chain_kernel", "extract_kernel",
                                  "align_kernel") if s in name), "sort" if "Sort" in name or "sort" in name else "other")
        stages[stage] = stages.get(stage, 0.0) + ev.device_time_total / 1000.0
    return {k: round(v, 3) for k, v in sorted(stages.items())}


def _basecaller(tmp, mdir, rdir, ref=None):
    cmd = [sys.executable, "-m", "bonito_b200", "basecaller", mdir, rdir, "--no-trim"]
    if ref:
        cmd += ["--reference", ref]
    out = os.path.join(tmp, "ref.sam" if ref else "plain.sam")
    with open(out, "w") as fh:
        p = subprocess.run(cmd, cwd=ROOT, stdout=fh, stderr=subprocess.PIPE, text=True, check=True)
    rate = float(re.search(r"samples per second ([0-9.E+]+)", p.stderr).group(1))
    return rate, out


def main():
    parser = argparse.ArgumentParser()
    parser.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_map_bench.json"))
    parser.add_argument("--genome-mb", type=float, default=100)
    parser.add_argument("--bc-reads", type=int, default=400)
    parser.add_argument("--bc-samples", type=int, default=100_000)
    args = parser.parse_args()
    rng = np.random.default_rng(7)
    result = {"gpu": torch.cuda.get_device_name(0)}
    try:
        result["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                               capture_output=True, text=True).stdout.strip()
    except OSError:
        result["power_limit"] = "unknown"
    with tempfile.TemporaryDirectory() as tmp:
        n = int(args.genome_mb * 1e6)
        sizes = [n // 2, n // 4, n - n // 2 - n // 4]
        genome = [(f"chr{i + 1}", _rand(rng, s)) for i, s in enumerate(sizes)]
        _fasta(os.path.join(tmp, "genome.fa"), genome)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        al = A.Aligner(os.path.join(tmp, "genome.fa"))
        torch.cuda.synchronize()
        result["index_build_s"] = round(time.perf_counter() - t0, 3)
        result["genome_bases"] = n
        result["index_entries"] = int(al.idx_val.numel())
        result["map"] = []
        for length, count in ((10_000, 800), (30_000, 300)):
            for label, rates in (("2/1/1", (0.02, 0.01, 0.01)), ("5/3/3", (0.05, 0.03, 0.03))):
                reads = _reads(rng, genome[0][1], count, length, rates)
                al.map_batch(reads[:64])                       # warm-up
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                got = al.map_batch(reads)
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                bases = sum(len(r) for r in reads)
                result["map"].append({"read_length": length, "errors_sub_ins_del_pct": label, "reads": count,
                                      "seconds": round(dt, 4), "reads_per_s": round(count / dt, 1),
                                      "mbases_per_s": round(bases / dt / 1e6, 2),
                                      "mapped": sum(m is not None for m in got),
                                      "kernel_ms": _kernel_ms(al, reads)})
                print(json.dumps(result["map"][-1]), flush=True)
        del al
        torch.cuda.empty_cache()
        # basecaller with and without --reference
        from oracle import synth
        spec = synth.model_spec("hac")
        mdir = synth.write_model_dir(os.path.join(tmp, "model"), spec, synth.make_weights(spec, seed=3))
        rdir = os.path.join(tmp, "reads")
        os.makedirs(rdir)
        for i in range(args.bc_reads):
            np.save(os.path.join(rdir, f"read{i}.npy"),
                    (93.7 + 23.5 * synth.squiggle(1, args.bc_samples, seed=100 + i)[0, 0].numpy()).astype(np.float32))
        rate, sam = _basecaller(tmp, mdir, rdir)
        calls = [line.split("\t") for line in open(sam) if not line.startswith("@")]
        _fasta(os.path.join(tmp, "calls.fa"), [(r[0], np.frombuffer(r[9].encode(), np.uint8)) for r in calls])
        runs = {"plain": [], "reference": []}
        for _ in range(2):
            runs["plain"].append(_basecaller(tmp, mdir, rdir)[0])
            r, sam = _basecaller(tmp, mdir, rdir, os.path.join(tmp, "calls.fa"))
            runs["reference"].append(r)
        mapped = sum(1 for line in open(sam) if not line.startswith("@") and line.split("\t")[1] in ("0", "16"))
        result["basecaller"] = {"model": "synthetic hac", "reads": args.bc_reads, "samples_per_read": args.bc_samples,
                                "bases": sum(len(r[9]) for r in calls), "samples_per_s": runs,
                                "mapped_reads": mapped}
    with open(args.out, "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result["basecaller"]))


if __name__ == "__main__":
    main()
