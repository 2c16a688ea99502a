"""
Benchmark of BAM input (b200_bgzf_decompress, bonito_b200.bam) -> one JSON file (default
profiles/h100_bgzf_read_bench.json):

- payload: synthetic BAM records (uniform random bases, normally distributed qualities; --reads x --length), >= 256 MB
  uncompressed, written as BAM twice: members from b200_bgzf_compress (bam.BamOutput) and members from zlib level 6
  (htslib's default level, 65280 bytes each); the compression ratio of each;
- kernel: CUDA events around repeated b200_bgzf_decompress launches over all the members of each file at once, after a
  warm-up launch; output GB/s;
- host baseline: zlib inflating the same members on one thread and on 8 threads (zlib releases the GIL);
- end to end: seconds of `duplex.read_records` on the SAM text and on the BAM of the same reads, three alternated runs.

Usage: python scripts/bench_bgzf_read.py [--out profiles/h100_bgzf_read_bench.json]
"""
import argparse
import json
import os
import struct
import subprocess
import sys
import tempfile
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bonito_b200 import bam, native   # noqa: E402
from bonito_b200.cli import duplex     # noqa: E402

HEADER = "@HD\tVN:1.6\tSO:unknown\n"


def _write_inputs(tmp, reads, length, seed=0):
    """(SAM path, uncompressed BAM stream) of `reads` synthetic unaligned records."""
    rng = np.random.default_rng(seed)
    sam_path = os.path.join(tmp, "reads.sam")
    stream = [bam.encode_header(HEADER)]
    with open(sam_path, "w") as fh:
        fh.write(HEADER)
        for i in range(reads):
            seq = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, length)].tobytes().decode()
            qual = (np.clip(rng.normal(20, 6, length), 0, 60).astype(np.uint8) + 33).tobytes().decode()
            line = f"{i:08x}-read\t4\t*\t0\t0\t*\t*\t0\t0\t{seq}\t{qual}\tqs:i:20"
            fh.write(line + "\n")
            stream.append(bam.encode_record(line))
    return sam_path, b"".join(stream)


def _zlib_bgzf(stream, level=6):
    out = []
    for i in range(0, len(stream), native.BGZF_MEMBER_INPUT):
        d = stream[i:i + native.BGZF_MEMBER_INPUT]
        c = zlib.compressobj(level, zlib.DEFLATED, -15)
        raw = c.compress(d) + c.flush()
        bsize = 18 + len(raw) + 8
        out.append(b"\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\0BC\x02\0" + struct.pack("<H", bsize - 1) + raw +
                   struct.pack("<II", zlib.crc32(d), len(d)))
    return b"".join(out) + bam.EOF_MARKER


def _members(path):
    """[(raw DEFLATE bytes, ISIZE, CRC32)] of a BGZF file."""
    out, where = [], 0
    with open(path, "rb") as fh:
        while (m := bam.next_member(fh, where)) is not None:
            member, raw, n_raw, crc, isize = m
            out.append((member[raw:raw + n_raw], isize, crc))
            where += len(member)
    return out


def _kernel(members, reps):
    raws = b"".join(r for r, _, _ in members)
    sizes = np.array([len(r) for r, _, _ in members], np.int64)
    isizes = np.array([i for _, i, _ in members], np.int64)
    meta = np.stack([np.cumsum(sizes) - sizes, sizes, np.cumsum(isizes) - isizes, isizes,
                     np.array([c for _, _, c in members], np.int64)], 1)
    inp = torch.from_numpy(np.frombuffer(raws, np.uint8).copy()).cuda()
    d_meta = torch.from_numpy(meta).cuda()
    total = int(isizes.sum())
    out = torch.empty(total, dtype=torch.uint8, device="cuda")
    status = torch.empty(len(members), dtype=torch.int32, device="cuda")
    native.bgzf_decompress(inp, d_meta, out, status)              # warm-up
    torch.cuda.synchronize()
    assert int(status.abs().sum()) == 0
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        native.bgzf_decompress(inp, d_meta, out, status)
    stop.record()
    torch.cuda.synchronize()
    ms = start.elapsed_time(stop) / reps
    return {"members": len(members), "compressed_bytes": len(raws), "output_bytes": total, "launches": reps,
            "ms_per_launch": round(ms, 3), "output_gb_per_s": round(total / ms / 1e6, 2)}, out


def _host(members, threads):
    def one(m):
        return zlib.decompress(m[0], -15)
    t0 = time.perf_counter()
    if threads == 1:
        total = sum(len(one(m)) for m in members)
    else:
        with ThreadPoolExecutor(threads) as pool:
            total = sum(len(x) for x in pool.map(one, members, chunksize=16))
    s = time.perf_counter() - t0
    return {"threads": threads, "seconds": round(s, 3), "output_gb_per_s": round(total / s / 1e9, 3)}


def main():
    parser = argparse.ArgumentParser()
    parser.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bgzf_read_bench.json"))
    parser.add_argument("--reads", type=int, default=20_000)
    parser.add_argument("--length", type=int, default=10_000)
    parser.add_argument("--reps", type=int, default=10)
    args = parser.parse_args()
    result = {"gpu": torch.cuda.get_device_name(0)}
    try:
        result["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                               capture_output=True, text=True).stdout.strip()
    except OSError:
        result["power_limit"] = "unknown"
    result["host_cpus"] = os.cpu_count()
    with tempfile.TemporaryDirectory() as tmp:
        sam_path, stream = _write_inputs(tmp, args.reads, args.length)
        files = {"gpu": os.path.join(tmp, "gpu.bam"), "zlib6": os.path.join(tmp, "zlib6.bam")}
        with open(files["gpu"], "wb") as fh:
            w = bam.BgzfWriter(fh)
            w.write(stream)
            w.close()
        with open(files["zlib6"], "wb") as fh:
            fh.write(_zlib_bgzf(stream))
        result["payload"] = {"reads": args.reads, "read_length": args.length, "bam_payload_bytes": len(stream),
                             "sam_bytes": os.path.getsize(sam_path),
                             "ratio": {k: round(os.path.getsize(p) / len(stream), 4) for k, p in files.items()}}
        print(json.dumps(result["payload"]), flush=True)
        for name, path in files.items():
            members = _members(path)
            kern, out = _kernel(members, args.reps)
            assert out.cpu().numpy().tobytes() == stream
            del out
            kern["zlib_host"] = [_host(members, 1), _host(members, 8)]
            result[f"kernel_{name}_members"] = kern
            print(json.dumps({name: kern}), flush=True)
        runs = {"sam": [], "bam": []}
        for _ in range(3):
            for fmt, path in (("sam", sam_path), ("bam", files["zlib6"])):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                reads = duplex.read_records(path)
                runs[fmt].append(round(time.perf_counter() - t0, 3))
                assert len(reads) == args.reads
        result["read_records_seconds"] = {"bam_file": "zlib level 6 members", **runs}
        print(json.dumps(result["read_records_seconds"]), flush=True)
    with open(args.out, "w") as fh:
        json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
