"""
Time the batched Smith-Waterman kernel (b200_sw_align) and one `evaluate` pass on one GPU.  Prints one JSON line:

  * kernel: 4096 seeded pairs, a ~1000-base core per pair with a 5 % substitution / 2 % insertion / 3 % deletion edit
    profile applied to the query, and 20 random flanking bases on each side of both query and reference.  Cells/s is
    sum(m * n) over the time of one b200_sw_align call (CUDA events around --steps calls after --warmup calls; a call
    includes the four small host-to-device copies of the per-pair offsets and lengths).
  * evaluate: 4096 chunks of 1998 samples through a seeded hac LSTM-CRF model (batch 256), references = the model's own
    calls with the same edit profile.  Wall time of data loading + forward + decode + alignment + summary, and the
    alignment's share of it (align_batch: packing, copies, the kernel and the result fields).
  * the GPU name and power limit, read in the same run.

    python scripts/bench_align.py [--steps 20] [--warmup 3] [--out profiles/h100_align_bench.json]
"""
import argparse
import json
import os
import random
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bonito_b200 import native, synth  # noqa: E402
from bonito_b200.align import align_batch, _pack  # noqa: E402
from bonito_b200.cli.evaluate import call_chunks, summary  # noqa: E402
from bonito_b200.data import ComputeSettings, DataSettings, ModelSetup, load_data  # noqa: E402
from bonito_b200.util import load_model  # noqa: E402

N_PAIRS, CORE, FLANK = 4096, 1000, 20


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--id=%d" % torch.cuda.current_device(), "--query-gpu=name,power.limit",
                        "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().split("\n")[0]
    name, power = [v.strip() for v in q.split(",")]
    return dict(gpu=name, power_limit=power)


def mutate(rng, s, sub=0.05, ins=0.02, dele=0.03):
    out = []
    for c in s:
        x = rng.random()
        if x < sub:
            out.append(rng.choice([b for b in "ACGT" if b != c]))
        elif x < sub + ins:
            out.append(c)
            out.append(rng.choice("ACGT"))
        elif x >= sub + ins + dele:
            out.append(c)
    return "".join(out)


def rand(rng, n):
    return "".join(rng.choice("ACGT") for _ in range(n))


def bench_kernel(steps, warmup):
    rng = random.Random(1)
    refs, seqs = [], []
    for _ in range(N_PAIRS):
        core = rand(rng, CORE)
        refs.append(rand(rng, FLANK) + core + rand(rng, FLANK))
        seqs.append(rand(rng, FLANK) + mutate(rng, core) + rand(rng, FLANK))
    q, q_off, q_len = _pack(seqs, "sequence")
    r, r_off, r_len = _pack(refs, "reference")
    pin = lambda a: torch.from_numpy(a).pin_memory()          # noqa: E731
    query, ref = pin(q).cuda(), pin(r).cuda()
    meta = [pin(a) for a in (q_off, q_len, r_off, r_len)]
    ws = torch.empty(native.sw_align_workspace_bytes(N_PAIRS, int(r_len.max())), dtype=torch.uint8, device="cuda")
    out = torch.empty(N_PAIRS, 7, dtype=torch.int32, device="cuda")

    def call():
        native.sw_align(query, meta[0], meta[1], ref, meta[2], meta[3], ws, out)

    for _ in range(warmup):
        call()
    torch.cuda.synchronize()
    times = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        call()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    ms = sorted(times)[len(times) // 2]
    cells = float(np.dot(q_len.astype(np.float64), r_len.astype(np.float64)))
    mean_score = float(out[:, 0].float().mean())
    return dict(pairs=N_PAIRS, mean_query_len=round(float(q_len.mean()), 1), mean_ref_len=round(float(r_len.mean()), 1),
                cells=int(cells), ms_per_call=round(ms, 3), gcups=round(cells / (ms / 1e3) / 1e9, 1),
                mean_score=round(mean_score, 1))


def bench_evaluate(n_chunks=4096, length=1998, batchsize=256):
    spec = synth.model_spec("hac")
    with tempfile.TemporaryDirectory() as tmp:
        mdir = synth.write_model_dir(os.path.join(tmp, "hac"), spec, synth.make_weights(spec, seed=3))
        model = load_model(mdir, "cuda", weights=1, batchsize=batchsize, chunksize=length, use_koi=True)
        chunks = synth.squiggle(n_chunks, length, seed=5)[:, 0].numpy()
        setup, compute = ModelSetup(3, 1, {}), ComputeSettings(batch_size=batchsize, num_workers=0, seed=9)

        def write(directory, refs):
            os.makedirs(directory)
            labels = np.zeros((n_chunks, max(1, max(map(len, refs)))), dtype=np.uint8)
            for i, s in enumerate(refs):
                labels[i, :len(s)] = ["NACGT".index(c) for c in s]
            np.save(os.path.join(directory, "chunks.npy"), chunks)
            np.save(os.path.join(directory, "references.npy"), labels)
            np.save(os.path.join(directory, "reference_lengths.npy"), np.array(list(map(len, refs)), dtype=np.uint16))

        write(os.path.join(tmp, "d0"), ["A"] * n_chunks)
        _, loader = load_data(DataSettings(os.path.join(tmp, "d0"), n_chunks * 100, n_chunks, None), setup, compute)
        calls, _ = call_chunks(model, loader, "cuda")                            # also the warm-up of every shape
        rng = random.Random(7)
        write(os.path.join(tmp, "d1"), [mutate(rng, c) or "A" for c in calls])
        align_batch(["ACGT"], ["ACGT"])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        _, loader = load_data(DataSettings(os.path.join(tmp, "d1"), n_chunks * 100, n_chunks, None), setup, compute)
        seqs, refs = call_chunks(model, loader, "cuda")
        t1 = time.perf_counter()
        results = align_batch(refs, seqs)
        t2 = time.perf_counter()
        text = summary(results)
        t3 = time.perf_counter()
    accuracy = [line for line in text.split("\n") if line.startswith("* accuracy")][0].split()[-1]
    return dict(chunks=n_chunks, chunk=length, batch=batchsize, mean_call_len=round(float(np.mean([len(s) for s in seqs])), 1),
                wall_s=round(t3 - t0, 3), load_forward_decode_s=round(t1 - t0, 3), align_s=round(t2 - t1, 3),
                align_share=round((t2 - t1) / (t3 - t0), 3), accuracy=accuracy)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_align.py needs a CUDA device")
    res = dict(gpu_info(), kernel=bench_kernel(args.steps, args.warmup), evaluate=bench_evaluate())
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
