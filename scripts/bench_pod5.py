"""
POD5 input on one GPU: the zstd and svb16 kernels against host libzstd plus the numpy svb16 decode, `Reader.get_reads` over
the same reads as POD5 and as `.npy`, and `basecaller` with a seeded hac model on both.  Needs the system libzstd.so.1 to
write its input.  Prints one JSON object (and writes it to --out).

    python scripts/bench_pod5.py --samples 200000000 --out profiles/h100_pod5_bench.json
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _pod5_writer as W  # noqa: E402
from bonito_b200 import native  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name(), "unknown"


def rows_of(samples, row=W.ROW_SAMPLES, seed=0):
    n = max(1, samples // row)
    sig = W.synthetic_reads(1, seed=seed, min_len=row * 8, max_len=row * 8 + 1)[0]["signal"]
    rows = [np.roll(sig, 977 * i)[:row] for i in range(n)]
    return rows


def bench_kernels(samples, reps):
    rows = rows_of(samples)
    blobs = [W.vbz_compress(r, level=1) for r in rows]
    counts = np.array([len(r) for r in rows], np.int64)
    caps = (counts + 7) // 8 + 2 * counts
    lens = np.array([len(b) for b in blobs], np.int64)
    zm = np.stack([np.concatenate([[0], np.cumsum(lens)[:-1]]), lens, np.concatenate([[0], np.cumsum(caps)[:-1]]), caps], 1)
    inp = torch.from_numpy(np.frombuffer(b"".join(blobs), np.uint8).copy()).cuda()
    zmeta = torch.from_numpy(zm).cuda()
    out = torch.empty(int(caps.sum()), dtype=torch.uint8, device="cuda")
    out_len = torch.empty(len(rows), dtype=torch.int64, device="cuda")
    st = torch.empty(len(rows), dtype=torch.int32, device="cuda")
    samples_d = torch.empty(int(counts.sum()), dtype=torch.int16, device="cuda")
    native.zstd_decompress(inp, zmeta, out, out_len, st)
    svb_len = out_len.cpu().numpy()
    smeta = torch.from_numpy(np.stack([zm[:, 2], svb_len, counts, np.concatenate([[0], np.cumsum(counts)[:-1]])], 1)).cuda()
    st2 = torch.empty_like(st)
    native.svb16_decode(out, smeta, samples_d, st2)
    torch.cuda.synchronize()
    assert not st.any() and not st2.any()
    assert np.array_equal(samples_d[:len(rows[0])].cpu().numpy(), rows[0])
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    tz, ts = [], []
    for _ in range(reps):
        ev[0].record()
        native.zstd_decompress(inp, zmeta, out, out_len, st)
        ev[1].record()
        native.svb16_decode(out, smeta, samples_d, st2)
        ev[2].record()
        torch.cuda.synchronize()
        tz.append(ev[0].elapsed_time(ev[1]) / 1e3)
        ts.append(ev[1].elapsed_time(ev[2]) / 1e3)
    zbytes, n = int(svb_len.sum()), int(counts.sum())
    res = dict(rows=len(rows), samples=n, compressed_bytes=int(lens.sum()), zstd_output_bytes=zbytes,
               zstd_s=float(np.median(tz)), svb16_s=float(np.median(ts)),
               zstd_GBps=zbytes / np.median(tz) / 1e9, svb16_Msamples_per_s=n / np.median(ts) / 1e6,
               gpu_Msamples_per_s=n / (np.median(tz) + np.median(ts)) / 1e6)

    def host_one(k):
        raw = W.zstd_decompress(blobs[k], int(caps[k]))
        return W.svb16_decode(raw, int(counts[k]))

    for threads in (1, 8):
        t0 = time.perf_counter()
        with ThreadPoolExecutor(threads) as ex:
            dec = list(ex.map(host_one, range(len(rows))))
        dt = time.perf_counter() - t0
        assert np.array_equal(dec[-1], rows[-1])
        res[f"host_{threads}t_s"] = dt
        res[f"host_{threads}t_Msamples_per_s"] = n / dt / 1e6
    return res


def make_reads_dirs(tmp, n_reads, seed=7):
    reads = W.synthetic_reads(n_reads, seed=seed, min_len=20000, max_len=60000)
    pod, npy = os.path.join(tmp, "pod5"), os.path.join(tmp, "npy")
    os.makedirs(pod)
    os.makedirs(npy)
    W.write_pod5(os.path.join(pod, "reads.pod5"), reads, vbz=True)
    for i, r in enumerate(reads):
        np.save(os.path.join(npy, f"{r['read_id']}.npy"), W.expected_pa(r, i))
    return pod, npy, sum(len(r["signal"]) for r in reads)


def bench_reader(pod, npy, reps=3):
    from bonito_b200.reader import Reader
    out = {}
    for name, d in (("pod5", pod), ("npy", npy)):
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            n = sum(len(r.signal) for r in Reader(d).get_reads(d))
            ts.append(time.perf_counter() - t0)
        out[f"get_reads_{name}_s"] = float(np.median(ts))
    return out


def bench_basecaller(tmp, pod, npy):
    from oracle import synth
    spec = synth.model_spec("hac")
    mdir = synth.write_model_dir(os.path.join(tmp, "model"), spec, synth.make_weights(spec, seed=3))
    out = {}
    for name, d in (("pod5", pod), ("npy", npy)):
        t0 = time.perf_counter()
        with open(os.path.join(tmp, f"{name}.fastq"), "wb") as fh:
            p = subprocess.run([sys.executable, "-m", "bonito_b200", "basecaller", mdir, d], cwd=ROOT, stdout=fh,
                               stderr=subprocess.PIPE, text=True, timeout=1800)
        assert p.returncode == 0, p.stderr[-2000:]
        out[f"basecaller_{name}_s"] = time.perf_counter() - t0
    records = []
    for n in ("pod5", "npy"):
        lines = open(os.path.join(tmp, f"{n}.fastq")).read().splitlines()
        records.append(sorted("\n".join(lines[i:i + 4]) for i in range(0, len(lines), 4)))
    out["basecaller_same_fastq_records"] = records[0] == records[1]  # in reads-table and file name order
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=200_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--reads", type=int, default=300)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    name, power = card()
    res = dict(card=name, power_limit=power, libzstd=W._zstd().ZSTD_versionNumber())
    res["kernels"] = bench_kernels(args.samples, args.reps)
    tmp = tempfile.mkdtemp()
    try:
        pod, npy, n = make_reads_dirs(tmp, args.reads)
        res["reads"] = dict(n_reads=args.reads, samples=n)
        res["reader"] = bench_reader(pod, npy)
        res["basecaller"] = bench_basecaller(tmp, pod, npy)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=2)


if __name__ == "__main__":
    main()
