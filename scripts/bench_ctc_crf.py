"""
Time the CTC-CRF loss on one GPU at training shapes: N = 64 chunks of T = 2000 frames, targets of about 0.45 T bases,
state_len 4 (C = 1280 scores per frame) and 5 (C = 5120).

For each shape, timed with CUDA events (median of --steps after --warmup):
  * loss:  CTC_CRF.normalise + ctc_loss forward and backward (autograd over the sm_90a lattice kernels);
  * logz:  CTC_CRF.logZ alone, no gradient;
  * torch: the same loss with both lattices written as PyTorch ops on the GPU (fp32, autograd), for scale.
Achieved GB/s counts the bytes of the k-mer lattice on the training path: scores read twice (forward, gradient pass), the
gradient written, the alpha rows written and read (4 bytes each); logz counts one read of the scores.  Both are set against
the 3.35 TB/s HBM3 data-sheet bound of the H100 SXM (a bound, not a measurement).  The GPU name and power limit are read in
the same run.  Prints one JSON line.

    python scripts/bench_ctc_crf.py [--steps 10] [--warmup 3] [--out profiles/h100_ctc_crf_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bonito_b200.crf.model import CTC_CRF  # noqa: E402
from oracle.crf_oracle import crf_idx  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().split("\n")[0]
    name, power, clock = [v.strip() for v in q.split(",")]
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def inputs(state_len, N, T, device, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    scores = (5 * torch.tanh(torch.randn(T, N, 5 * 4 ** state_len, generator=g))).to(device)
    lengths = torch.randint(int(0.40 * T), int(0.50 * T), (N,), generator=g)
    targets = torch.zeros(N, int(lengths.max()), dtype=torch.long)
    for n in range(N):
        targets[n, :lengths[n]] = torch.randint(1, 5, (int(lengths[n]),), generator=g)
    return scores, targets.to(device), lengths.to(device)


def torch_loss(seqdist, scores, targets, target_lengths):
    """normalise + ctc_loss with both lattices as PyTorch ops (the scale reference, not the product path)."""
    T, N, _ = scores.shape
    idx = torch.as_tensor(crf_idx(seqdist.state_len), device=scores.device)
    Ms = scores.reshape(T, N, -1, 5)
    a = scores.new_zeros(N, idx.shape[0])
    for t in range(T):
        a = torch.logsumexp(Ms[t] + a[:, idx], -1)
    scores = scores - torch.logsumexp(a, -1)[:, None] / T
    stay, move = seqdist.prepare_ctc_scores(scores, targets)
    L = stay.shape[2]
    neg = torch.full((N, 1), -1e30, device=scores.device)
    a = torch.cat([scores.new_zeros(N, 1), neg.expand(N, L - 1)], 1)
    for t in range(T):
        a = torch.logaddexp(a + stay[t], torch.cat([neg, a[:, :-1] + move[t]], 1))
    logz = a.gather(1, (target_lengths - seqdist.state_len).clamp(min=0)[:, None])[:, 0]
    return (-(logz / target_lengths)).mean()


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
    return ms[len(ms) // 2], ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--torch-steps", type=int, default=2)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ctc_crf.py needs a CUDA device")
    dev = torch.device("cuda:0")
    N, T = args.batch, args.frames
    results = []
    for state_len in (4, 5):
        seqdist = CTC_CRF(state_len, "NACGT")
        scores, targets, lengths = inputs(state_len, N, T, dev)
        C = scores.shape[2]
        S = 4 ** state_len
        x = scores.detach().requires_grad_()

        def loss_step():
            x.grad = None
            seqdist.ctc_loss(x, targets, lengths).backward()

        def logz_step():
            with torch.no_grad():
                seqdist.logZ(scores)

        def torch_step():
            x.grad = None
            torch_loss(seqdist, x, targets, lengths).backward()

        loss_ms, loss_all = timed(loss_step, args.steps, args.warmup)
        logz_ms, logz_all = timed(logz_step, args.steps, args.warmup)
        torch_ms, torch_all = timed(torch_step, args.torch_steps, 1)
        with torch.no_grad():
            native_loss = float(seqdist.ctc_loss(scores, targets, lengths))
            ref_loss = float(torch_loss(seqdist, scores, targets, lengths))
        train_bytes = 3 * T * N * C * 4 + 2 * (T + 1) * N * S * 4
        logz_bytes = T * N * C * 4
        results.append(dict(
            state_len=state_len, n_score=C, batch=N, frames=T, mean_target_bases=round(float(lengths.float().mean()), 1),
            loss_fwd_bwd_ms=round(loss_ms, 3), logz_ms=round(logz_ms, 3), torch_ops_fwd_bwd_ms=round(torch_ms, 1),
            speedup_over_torch_ops=round(torch_ms / loss_ms, 1),
            loss_ms_min_max=[round(min(loss_all), 3), round(max(loss_all), 3)],
            logz_ms_min_max=[round(min(logz_all), 3), round(max(logz_all), 3)],
            train_lattice_gbytes=round(train_bytes / 1e9, 3), loss_gb_per_s=round(train_bytes / loss_ms / 1e6, 1),
            loss_over_hbm_datasheet=round(train_bytes / loss_ms / 1e-3 / HBM_BYTES_PER_S, 3),
            logz_gb_per_s=round(logz_bytes / logz_ms / 1e6, 1),
            logz_over_hbm_datasheet=round(logz_bytes / logz_ms / 1e-3 / HBM_BYTES_PER_S, 3),
            loss=round(native_loss, 6), torch_ops_loss=round(ref_loss, 6)))
        del scores, x
        torch.cuda.empty_cache()
    line = json.dumps(dict(gpu_info(), bench="ctc_crf_loss", steps=args.steps, warmup=args.warmup, results=results))
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
