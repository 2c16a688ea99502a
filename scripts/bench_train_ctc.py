"""
Time one full QuartzNet CTC training step on one GPU: dna_r9.4.1@v1 and @v2 shapes (v2 with dropout 0.05), batch 64 x
4000 samples, fp32 master weights, `Model.loss`, GradScaler and AdamW.

  * native: the train-mode forward on the native kernels (CtcTrainPlan), loss, backward, unscale + clip_grad_norm_(2.0),
    GradScaler step of AdamW;
  * torch:  the same module tree in eager torch under fp16 autocast (cuDNN convolutions and BatchNorm, torch's CUDA
    ctc_loss), the same loss, scaler, clip and optimizer.
The two alternate step by step, each timed with CUDA events (median of --steps after --warmup).  A separate profiled run of
the native step sums kernel times per stage (forward kernels, each weight-gradient kind, BatchNorm / activation, input
gradients, head, loss, optimizer) and gives the wgrad GEMM's achieved TFLOP/s (FLOPs counted from the shapes) against the
989 TFLOP/s dense FP16 data-sheet rate.  The GPU name and power limit are read in the same run.  Prints one JSON line (and
writes it to --out).

    python scripts/bench_train_ctc.py [--steps 10] [--warmup 3] [--out profiles/h100_train_ctc_bench.json]
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

from bonito_b200 import synth  # noqa: E402
from bonito_b200.ctc.model import Model  # noqa: E402

PEAK_FP16 = 989.0


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().split("\n")[0]
    name, power, clock = [v.strip() for v in q.split(",")]
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def build(name, dropout, device):
    spec = synth.quartznet_spec(name)
    cfg = synth.quartznet_config(spec)
    for b in cfg["block"]:
        b["dropout"] = dropout
    model = Model(cfg)
    model.load_state_dict(synth.make_quartznet_weights(spec, seed=25))
    return model.to(device).train()


def wgrad_flops(model, N, T):
    """2 * rows * Cout * K of every b200_wgrad_gemm call of one backward."""
    from bonito_b200.engine_ctc import _walk
    blocks, _ = _walk(model)
    M, total = N * T, 0
    for wb in blocks[1:]:
        if wb["separable"]:
            total += sum(2 * M * wb["cout"] * t.depthwise.in_channels for t, _ in wb["pairs"])
            if wb["residual"]:
                total += 2 * M * wb["cout"] * wb["cin"]
        else:
            total += 2 * M * wb["cout"] * wb["k"] * wb["cin"]
    return total


def stage(kernel):
    k = kernel.lower()
    for key, name in (("wgrad_gemm", "wgrad_gemm"), ("tap_wgrad_kernel<false", "wgrad_depthwise"),
                      ("tap_wgrad_kernel<true", "wgrad_first_conv"), ("sum_partials", "wgrad_reduce"),
                      ("bn_stats", "bn_stats"), ("bn_act_fwd", "bn_act_fwd"), ("bn_act_bwd", "bn_act_bwd"),
                      ("head", "head"), ("ctc_loss", "loss"), ("adam", "optimizer"), ("foreach", "optimizer"),
                      ("multi_tensor", "optimizer"), ("reduce_kernel", "other_reductions"),
                      ("elementwise", "other_elementwise"), ("copy", "other_elementwise"),
                      ("depthwise", "depthwise_conv"), ("gemm", "gemm_fwd_and_dx"), ("conv_first", "first_conv")):
        if key in k:
            return name
    return "other"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--chunk", type=int, default=4000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    N, L = args.batch, args.chunk
    result = dict(**gpu_info(), batch=N, chunk=L, steps=args.steps, warmup=args.warmup, models={})
    x = synth.squiggle(N, L, seed=1).to(dev)
    for name, dropout in (("v1", 0.0), ("v2", 0.05)):
        torch.manual_seed(0)
        native = build(name, dropout, dev)
        native.use_koi()
        ref = build(name, dropout, dev)
        T = (L - 1) // native.stride + 1
        g = torch.Generator().manual_seed(2)
        lengths = torch.full((N,), T // 6, dtype=torch.int64)
        targets = torch.randint(1, 5, (N, T // 6), generator=g)
        weights = torch.cat([torch.tensor([0.4]), (0.1 / 4) * torch.ones(4)]).to(dev)

        def torch_loss(lp):
            ctc = F.ctc_loss(lp.float(), targets.to(dev), torch.full((N,), T, dtype=torch.int64), lengths, reduction="mean")
            return ctc - (lp * weights).mean()

        def make_step(model, forward, loss_fn):
            opt = torch.optim.AdamW(model.parameters(), lr=1e-4)
            scaler = torch.amp.GradScaler("cuda")

            def step():
                opt.zero_grad()
                loss = loss_fn(forward(x))
                scaler.scale(loss).backward()
                scaler.unscale_(opt)
                torch.nn.utils.clip_grad_norm_(model.parameters(), max_norm=2.0)
                scaler.step(opt)
                scaler.update()
            return step

        def torch_forward(inp):
            with torch.autocast("cuda", dtype=torch.float16):
                return F.log_softmax(ref.decoder.layers(ref.encoder(inp)), dim=-1)     # [T, N, C]

        nat = make_step(native, native, lambda lp: native.loss(lp.permute(1, 0, 2), targets, lengths)["total_loss"])
        tor = make_step(ref, torch_forward, torch_loss)
        for _ in range(args.warmup):
            nat()
            tor()
        torch.cuda.synchronize()
        times = {"native": [], "torch": []}
        for _ in range(args.steps):
            for key, fn in (("native", nat), ("torch", tor)):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                fn()
                b.record()
                torch.cuda.synchronize()
                times[key].append(a.elapsed_time(b))
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        # per-stage kernel time of the native step, in a profiled run of its own
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                nat()
            torch.cuda.synchronize()
        stages = {}
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            if t > 0 and ev.key:
                s = stage(ev.key)
                stages[s] = stages.get(s, 0.0) + t / 1000.0 / 3
        flops = wgrad_flops(native, N, T)
        wg_ms = stages.get("wgrad_gemm", float("nan"))
        result["models"][name] = dict(
            dropout=dropout, frames=T,
            native_step_ms=round(med["native"], 2), torch_step_ms=round(med["torch"], 2),
            native_samples_per_s=round(N * L / med["native"] * 1e3), torch_samples_per_s=round(N * L / med["torch"] * 1e3),
            native_over_torch=round(med["native"] / med["torch"], 3),
            native_stage_ms={k: round(v, 2) for k, v in sorted(stages.items(), key=lambda kv: -kv[1])},
            wgrad_gemm_tflops=round(flops / (wg_ms * 1e-3) / 1e12, 1),
            wgrad_gemm_share_of_fp16_peak=round(flops / (wg_ms * 1e-3) / 1e12 / PEAK_FP16, 3))
        del native, ref, nat, tor
        torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
