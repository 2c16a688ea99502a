"""
Benchmark of BAM output (b200_bgzf_compress, bonito_b200.bam) -> one JSON file (default profiles/h100_bgzf_bench.json):

- `basecaller` samples/s of a seeded hac model on 400 reads x 100 000 samples to `.sam` and to `.bam`, three runs each,
  alternated (the rate the CLI prints, reads, basecalls and the writer together, and the seconds of the whole process);
- the kernel rate: CUDA events around repeated b200_bgzf_compress launches on >= 256 MB of BAM payload, the uncompressed
  BAM stream of those basecalls repeated (members are independent, so the repeats change nothing within a member), after
  a warm-up launch; input GB/s and the compressed size over the input size;
- zlib level 1 and level 6 on the same members of one copy of the stream: size ratio and MB/s on one host core.

Usage: python scripts/bench_bgzf.py [--out profiles/h100_bgzf_bench.json]
"""
import argparse
import gzip
import json
import os
import re
import statistics
import subprocess
import sys
import tempfile
import time
import zlib

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bonito_b200 import native   # noqa: E402

M = native.BGZF_MEMBER_INPUT


def _basecaller(mdir, rdir, out):
    """(samples/s the CLI prints, with two significant digits; seconds of the whole process)"""
    cmd = [sys.executable, "-m", "bonito_b200", "basecaller", mdir, rdir, "--no-trim"]
    t0 = time.perf_counter()
    with open(out, "wb") as fh:
        p = subprocess.run(cmd, cwd=ROOT, stdout=fh, stderr=subprocess.PIPE, text=True, check=True)
    wall = time.perf_counter() - t0
    return float(re.search(r"samples per second ([0-9.E+]+)", p.stderr).group(1)), round(wall, 3)


def _kernel(stream, target_bytes, reps):
    data = (stream * -(-target_bytes // len(stream)))[:target_bytes]
    inp = torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy()).cuda()
    n = native.bgzf_members(inp.numel())
    out = torch.empty(n * native.BGZF_MEMBER_MAX, dtype=torch.uint8, device="cuda")
    off = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    ws = torch.empty(native.bgzf_workspace_bytes(inp.numel()), dtype=torch.uint8, device="cuda")
    native.bgzf_compress(inp, out, off, ws)          # warm-up
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        native.bgzf_compress(inp, out, off, ws)
    stop.record()
    torch.cuda.synchronize()
    ms = start.elapsed_time(stop) / reps
    return {"input_bytes": len(data), "members": n, "launches": reps, "ms_per_launch": round(ms, 3),
            "input_gb_per_s": round(len(data) / ms / 1e6, 2), "ratio": round(int(off[-1]) / len(data), 4)}


def _gpu_size(data):
    inp = torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy()).cuda()
    n = native.bgzf_members(inp.numel())
    out = torch.empty(n * native.BGZF_MEMBER_MAX, dtype=torch.uint8, device="cuda")
    off = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    ws = torch.empty(native.bgzf_workspace_bytes(inp.numel()), dtype=torch.uint8, device="cuda")
    native.bgzf_compress(inp, out, off, ws)
    torch.cuda.synchronize()
    return int(off[-1])


def _zlib(data, level):
    """(BGZF-framed size, MB/s of input) of zlib raw DEFLATE on the same members, on this one thread."""
    t0 = time.perf_counter()
    size = 0
    for i in range(0, len(data), M):
        c = zlib.compressobj(level, zlib.DEFLATED, -15)
        size += len(c.compress(data[i:i + M]) + c.flush()) + 26
    return size, len(data) / (time.perf_counter() - t0) / 1e6


def main():
    parser = argparse.ArgumentParser()
    parser.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bgzf_bench.json"))
    parser.add_argument("--reads", type=int, default=400)
    parser.add_argument("--samples", type=int, default=100_000)
    parser.add_argument("--kernel-mb", type=int, default=256)
    parser.add_argument("--reps", type=int, default=10)
    args = parser.parse_args()
    result = {"gpu": torch.cuda.get_device_name(0)}
    try:
        result["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                               capture_output=True, text=True).stdout.strip()
    except OSError:
        result["power_limit"] = "unknown"
    from oracle import synth
    with tempfile.TemporaryDirectory() as tmp:
        spec = synth.model_spec("hac")
        mdir = synth.write_model_dir(os.path.join(tmp, "model"), spec, synth.make_weights(spec, seed=3))
        rdir = os.path.join(tmp, "reads")
        os.makedirs(rdir)
        for i in range(args.reads):
            np.save(os.path.join(rdir, f"read{i}.npy"),
                    (93.7 + 23.5 * synth.squiggle(1, args.samples, seed=100 + i)[0, 0].numpy()).astype(np.float32))
        runs, walls = {"sam": [], "bam": []}, {"sam": [], "bam": []}
        for _ in range(3):
            for fmt in ("sam", "bam"):
                rate, wall = _basecaller(mdir, rdir, os.path.join(tmp, f"out.{fmt}"))
                runs[fmt].append(rate)
                walls[fmt].append(wall)
        sam_bytes = os.path.getsize(os.path.join(tmp, "out.sam"))
        bam_bytes = os.path.getsize(os.path.join(tmp, "out.bam"))
        stream = gzip.decompress(open(os.path.join(tmp, "out.bam"), "rb").read())
    med = {k: statistics.median(v) for k, v in runs.items()}
    wall = {k: statistics.median(v) for k, v in walls.items()}
    result["basecaller"] = {"model": "synthetic hac (seed 3)", "reads": args.reads, "samples_per_read": args.samples,
                            "samples_per_s": runs, "median": med, "bam_over_sam": round(med["bam"] / med["sam"], 4),
                            "process_seconds": walls, "median_process_seconds": wall,
                            "sam_bytes": sam_bytes, "bam_bytes": bam_bytes, "bam_payload_bytes": len(stream)}
    print(json.dumps(result["basecaller"]), flush=True)
    result["kernel"] = _kernel(stream, args.kernel_mb << 20, args.reps)
    print(json.dumps(result["kernel"]), flush=True)
    gpu = _gpu_size(stream)
    z1, z1_rate = _zlib(stream, 1)
    z6, z6_rate = _zlib(stream, 6)
    result["same_members"] = {"input_bytes": len(stream), "gpu_bytes": gpu, "zlib1_bytes": z1, "zlib6_bytes": z6,
                              "gpu_over_zlib1": round(gpu / z1, 4), "gpu_over_zlib6": round(gpu / z6, 4),
                              "zlib1_mb_per_s_one_core": round(z1_rate, 1), "zlib6_mb_per_s_one_core": round(z6_rate, 1)}
    print(json.dumps(result["same_members"]), flush=True)
    with open(args.out, "w") as fh:
        json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
