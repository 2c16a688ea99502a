"""
Benchmark of CTC training-data export (`basecaller --reference --save-ctc`) -> one JSON file (default
profiles/h100_save_ctc_bench.json):

- a seeded hac model, `--bc-reads` reads of `--bc-samples` samples, and a reference made of the calls of a first plain
  `basecaller` pass (as scripts/bench_map.py builds it);
- `basecaller --reference` and `basecaller --reference --save-ctc` alternated `--repeats` times: the samples/s the CLI
  prints (two digits), chunks/s derived from it, the chunks written and rejected;
- one in-process run of the same `--save-ctc` pipeline (basecall -> align_map -> CtcWriter, with a device synchronise at
  the end) timed with a host clock: samples/s and chunks/s, the wall time of the mapping thread's `map_batch` batches
  (device and host work of the mapper), and the writer thread's busy time (its run time less the time it waited for
  the next mapped chunk), which is the per-chunk filtering, formatting and the final save.

Usage: python scripts/bench_save_ctc.py [--out profiles/h100_save_ctc_bench.json]
"""
import argparse
import io
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

from _map_helpers import _fasta                     # noqa: E402
from bonito_b200 import aligner as A                # noqa: E402
from bonito_b200 import synth                       # noqa: E402
from bonito_b200.io import CtcWriter                # noqa: E402
from bonito_b200.nn import fuse_bn_                 # noqa: E402
from bonito_b200.reader import Reader, read_chunks  # noqa: E402
from bonito_b200.util import init, load_model, load_symbol  # noqa: E402


def _basecaller(out, mdir, rdir, *args):
    os.makedirs(os.path.dirname(out), exist_ok=True)
    cmd = [sys.executable, "-m", "bonito_b200", "basecaller", mdir, rdir, "--no-trim", *args]
    with open(out, "w") as fh:
        p = subprocess.run(cmd, cwd=ROOT, stdout=fh, stderr=subprocess.PIPE, text=True, check=True)
    run = {"samples_per_s": float(re.search(r"samples per second ([0-9.E+]+)", p.stderr).group(1)),
           "completed": int(re.search(r"completed reads: (\d+)", p.stderr).group(1))}
    rejected = {m.group(1): int(m.group(2)) for m in re.finditer(r"^ - (\S+): (\d+)$", p.stderr, re.M)}
    if rejected or "--save-ctc" in args:
        shape = re.search(r"chunks\.npy with shape \((\d+),", p.stderr)
        run.update(rejected=rejected, written=int(shape.group(1)) if shape else 0)
    return run


def _in_process(tmp, mdir, rdir, ref):
    """The CLI's --save-ctc pipeline in this process, with the mapper's batches and the writer's waits timed."""
    init(25, "cuda")
    model = load_model(mdir, "cuda", use_koi=True).apply(fuse_bn_)
    model.native_plan()
    p = model.config["basecaller"]
    al = A.Aligner(ref)
    scaling = model.config.get("scaling")
    pa = bool(scaling) and scaling.get("strategy") == "pa"
    reads = Reader(rdir).get_reads(rdir, do_trim=False, scaling_strategy=scaling,
                                   norm_params=model.config.get("standardisation") if pa else model.config.get("normalisation"))
    chunks = (c for r in reads for c in read_chunks(r, p["chunksize"], p["overlap"]))
    results = load_symbol(mdir, "basecall")(model, chunks, batchsize=p["batchsize"], chunksize=p["chunksize"],
                                            overlap=p["overlap"])
    mapped_s, waited_s = [0.0], [0.0]
    original = A._mapped

    def timed_mapped(*args):
        t0 = time.perf_counter()
        out = original(*args)
        mapped_s[0] += time.perf_counter() - t0
        return out

    def timed_wait(it):
        while True:
            t0 = time.perf_counter()
            try:
                item = next(it)
            except StopIteration:
                return
            finally:
                waited_s[0] += time.perf_counter() - t0
            yield item

    A._mapped = timed_mapped
    try:
        d = os.path.join(tmp, "inproc")
        os.makedirs(d)
        with open(os.devnull, "w") as null:
            writer = CtcWriter(timed_wait(A.align_map(al, results)), al, fd=null, mode="w", directory=d,
                               summary=os.path.join(d, "summary.tsv"), stderr=io.StringIO())
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            writer.start()
            writer.join()
            torch.cuda.synchronize()
            total = time.perf_counter() - t0
    finally:
        A._mapped = original
    if writer.error is not None:
        raise writer.error
    n = len(writer.log)
    samples = sum(s for _, s in writer.log)
    lengths = os.path.join(d, "reference_lengths.npy")
    written = int(np.load(lengths).shape[0]) if os.path.exists(lengths) else 0
    return {"seconds": round(total, 3), "chunks": n, "samples_per_s": round(samples / total, 1),
            "chunks_per_s": round(n / total, 1), "map_batch_wall_s": round(mapped_s[0], 3),
            "writer_busy_s": round(total - waited_s[0], 3), "accepted": n - sum(writer.rejected.values()),
            "written": written, "rejected": writer.rejected}


def main():
    parser = argparse.ArgumentParser()
    parser.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_save_ctc_bench.json"))
    parser.add_argument("--bc-reads", type=int, default=400)
    parser.add_argument("--bc-samples", type=int, default=100_000)
    parser.add_argument("--repeats", type=int, default=2)
    args = parser.parse_args()
    result = {"gpu": torch.cuda.get_device_name(0)}
    try:
        result["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                               capture_output=True, text=True).stdout.strip()
    except OSError:
        result["power_limit"] = "unknown"
    with tempfile.TemporaryDirectory() as tmp:
        spec = synth.model_spec("hac")
        mdir = synth.write_model_dir(os.path.join(tmp, "model"), spec, synth.make_weights(spec, seed=3))
        rdir = os.path.join(tmp, "reads")
        os.makedirs(rdir)
        for i in range(args.bc_reads):
            np.save(os.path.join(rdir, f"read{i}.npy"),
                    (93.7 + 23.5 * synth.squiggle(1, args.bc_samples, seed=100 + i)[0, 0].numpy()).astype(np.float32))
        plain = os.path.join(tmp, "plain", "calls.sam")
        _basecaller(plain, mdir, rdir)
        calls = [line.split("\t") for line in open(plain) if not line.startswith("@")]
        ref = os.path.join(tmp, "calls.fa")
        _fasta(ref, [(r[0], np.frombuffer(r[9].encode(), np.uint8)) for r in calls])
        runs = {"reference": [], "reference_save_ctc": []}
        for k in range(args.repeats):
            runs["reference"].append(_basecaller(os.path.join(tmp, f"ref{k}", "out.sam"), mdir, rdir, "--reference", ref))
            runs["reference_save_ctc"].append(
                _basecaller(os.path.join(tmp, f"ctc{k}", "out.sam"), mdir, rdir, "--reference", ref, "--save-ctc"))
        chunksize = synth.model_config(spec)["basecaller"]["chunksize"]
        for run in runs["reference_save_ctc"]:
            run["chunks_per_s"] = round(run["samples_per_s"] / chunksize, 1)
            run["accepted_fraction"] = round((run["completed"] - sum(run["rejected"].values())) / run["completed"], 4)
        result["basecaller"] = {"model": "synthetic hac", "reads": args.bc_reads, "samples_per_read": args.bc_samples,
                                "chunksize": chunksize, "read_bases": sum(len(r[9]) for r in calls), "runs": runs}
        inproc = _in_process(tmp, mdir, rdir, ref)
        inproc["accepted_fraction"] = round(inproc["accepted"] / max(inproc["chunks"], 1), 4)
        result["save_ctc_in_process"] = inproc
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
