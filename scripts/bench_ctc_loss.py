"""
Time the QuartzNet CTC loss on one GPU at training shapes: N = 128 chunks of T = 1334 frames (4000 samples at stride 3),
targets of 400-500 labels (about 450), C = 5 classes, reduction 'mean'.

Timed with CUDA events (median of --steps after --warmup), each against torch's CUDA F.ctc_loss on the same inputs:
  * fwd_bwd: the loss and its backward into the log-probs;
  * fwd:     the loss alone, no gradient.
The GPU name and power limit are read in the same run.  Prints one JSON line (and writes it to --out).

    python scripts/bench_ctc_loss.py [--steps 20] [--warmup 5] [--out profiles/h100_ctc_loss_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bonito_b200.ctc.loss import ctc_loss  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().split("\n")[0]
    name, power, clock = [v.strip() for v in q.split(",")]
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def inputs(N, T, C, device, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    log_probs = torch.randn(T, N, C, generator=g).mul(2).log_softmax(-1).to(device)
    lengths = torch.randint(400, 501, (N,), generator=g)
    targets = torch.randint(1, C, (N, int(lengths.max())), generator=g)
    return log_probs, targets.to(device), torch.full((N,), T, dtype=torch.int64), lengths


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    ms.sort()
    return round(ms[len(ms) // 2], 3), [round(ms[0], 3), round(ms[-1], 3)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--frames", type=int, default=1334)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ctc_loss.py needs a CUDA device")
    dev = torch.device("cuda:0")
    N, T, C = args.batch, args.frames, 5
    log_probs, targets, input_lengths, target_lengths = inputs(N, T, C, dev)
    x = log_probs.detach().requires_grad_()
    il_dev, tl_dev = input_lengths.to(dev), target_lengths.to(dev)

    def native_fwd_bwd():
        x.grad = None
        ctc_loss(x, targets, input_lengths, target_lengths).backward()

    def native_fwd():
        with torch.no_grad():
            ctc_loss(log_probs, targets, input_lengths, target_lengths)

    def torch_fwd_bwd():
        x.grad = None
        F.ctc_loss(x, targets, il_dev, tl_dev).backward()

    def torch_fwd():
        with torch.no_grad():
            F.ctc_loss(log_probs, targets, il_dev, tl_dev)

    res = {}
    for name, fn in (("native_fwd_bwd", native_fwd_bwd), ("torch_fwd_bwd", torch_fwd_bwd), ("native_fwd", native_fwd),
                     ("torch_fwd", torch_fwd)):
        res[name + "_ms"], res[name + "_ms_min_max"] = timed(fn, args.steps, args.warmup)
    with torch.no_grad():
        native_loss = float(ctc_loss(log_probs, targets, input_lengths, target_lengths))
        torch_loss = float(F.ctc_loss(log_probs, targets, il_dev, tl_dev))
    line = json.dumps(dict(gpu_info(), bench="ctc_loss", steps=args.steps, warmup=args.warmup, batch=N, frames=T,
                           classes=C, mean_target_labels=round(float(target_lengths.float().mean()), 1),
                           **res, fwd_bwd_speedup_over_torch=round(res["torch_fwd_bwd_ms"] / res["native_fwd_bwd_ms"], 2),
                           fwd_speedup_over_torch=round(res["torch_fwd_ms"] / res["native_fwd_ms"], 2),
                           loss=round(native_loss, 6), torch_loss=round(torch_loss, 6)))
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
