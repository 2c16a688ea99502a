"""
Time the QuartzNet CTC models dna_r9.4.1@v1 and @v2 (seeded weights) at batch 512 x 3999 samples on one GPU, batches resident
in HBM.  A step is the native forward + per-frame greedy step (CtcPlan.greedy) + the D2H copy of the labels and probabilities;
the host-side collapse is not timed.  Prints one JSON line: samples/s and ms per step (median of --steps after --warmup steps
of the same shape), the per-stage split from the plan's CUDA events (a separate pass, summed over layers), the achieved
TFLOP/s of the GEMM stages (pointwise + dense) and of the depthwise stage from MACs computed from the shapes below, those
rates over the H100 SXM data-sheet rates (989 TFLOP/s dense FP16, 67 TFLOP/s FP32: data-sheet bounds, not measurements),
and the GPU name and power limit read in the same run.

    python scripts/bench_ctc.py [--batch 512] [--steps 20] [--warmup 3] [--out profiles/h100_ctc_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bonito_b200 import synth  # noqa: E402
from bonito_b200.ctc.model import Model  # noqa: E402

PEAK_FP16, PEAK_FP32 = 989e12, 67e12


def macs_per_frame(spec):
    """(depthwise, GEMM = pointwise + residual + dense after C1, first conv) multiply-accumulates per output frame."""
    dw = gemm = first = 0
    cin = 1
    for i, (f, r, k, s, res, sep) in enumerate(spec["blocks"]):
        for j in range(r):
            c = cin if j == 0 else f
            if sep:
                dw += c * k
                gemm += c * f
            elif i == 0:
                first += c * k * f
            else:
                gemm += c * k * f
        if res:
            gemm += cin * f
        cin = f
    gemm += cin * 5      # the head (runs on CUDA cores, counted with the GEMMs for the model total)
    return dw, gemm, first


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().split("\n")[0]
    name, power, clock = [v.strip() for v in q.split(",")]
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def bench(version, batch, chunk, steps, warmup):
    spec = synth.quartznet_spec(version)
    m = Model(synth.quartznet_config(spec))
    m.load_state_dict(synth.make_quartznet_weights(spec, seed=51))
    m.use_koi(batchsize=batch, chunksize=chunk, quantize=False)
    m = m.half().eval().to("cuda")
    plan = m.native_plan()
    x = synth.squiggle(batch, chunk, seed=5)[:, 0].half().cuda()
    T = plan.frames(chunk)
    labels_h = torch.empty(batch, T, dtype=torch.uint8, pin_memory=True)
    probs_h = torch.empty(batch, T, dtype=torch.float32, pin_memory=True)

    def step(events=None):
        labels, probs = plan.greedy(x, events=events)
        labels_h.copy_(labels, non_blocking=True)
        probs_h.copy_(probs, non_blocking=True)
        torch.cuda.synchronize()

    with torch.inference_mode():
        for _ in range(warmup):
            step()
        times = []
        for _ in range(steps):
            t0 = time.perf_counter()
            step()
            times.append(time.perf_counter() - t0)
        stages = {}
        for _ in range(3):
            ev = []
            step(ev)
            for name, a, b in ev:
                stages.setdefault(name, []).append(a.elapsed_time(b))
    split = {k: sum(v) / 3 for k, v in stages.items()}          # ms per step, summed over layers
    ms = sorted(times)[len(times) // 2] * 1e3
    dw, gemm, first = macs_per_frame(spec)
    frames = batch * T
    gemm_ms = split.get("pointwise", 0.0) + split.get("dense", 0.0)
    gemm_flop = 2.0 * frames * (gemm - spec["blocks"][-1][0] * 5)
    dw_flop = 2.0 * frames * dw
    return dict(model=f"dna_r9.4.1@{version}", batch=batch, chunk=chunk, frames_per_chunk=T, ms_per_step=round(ms, 3),
                samples_per_s=round(batch * chunk / (ms / 1e3)), stage_ms=split_round(split),
                gflop_per_chunk=round(2.0 * T * (dw + gemm + first) / 1e9, 2),
                gemm_tflops=round(gemm_flop / (gemm_ms / 1e3) / 1e12, 1),
                depthwise_tflops=round(dw_flop / (split["depthwise"] / 1e3) / 1e12, 1),
                gemm_over_datasheet_fp16=round(gemm_flop / (gemm_ms / 1e3) / PEAK_FP16, 3),
                depthwise_over_datasheet_fp32=round(dw_flop / (split["depthwise"] / 1e3) / PEAK_FP32, 3),
                depthwise_share_of_time=round(split["depthwise"] / sum(split.values()), 3),
                depthwise_share_of_macs=round(dw / (dw + gemm + first), 3))


def split_round(d):
    return {k: round(v, 3) for k, v in d.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--chunk", type=int, default=3999)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ctc.py needs a CUDA device")
    res = dict(gpu_info(), results=[bench(v, args.batch, args.chunk, args.steps, args.warmup) for v in ("v1", "v2")])
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
