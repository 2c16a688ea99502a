"""
Timing of the LSTM sup model (dna_r10.4.1@v4.3 shape: H = 1024, 5 LSTM layers, 4096 scores per frame) on the wide recurrent
kernel: seeded weights, 9996-sample chunks (T = 1666), resident forward + decode per step, at the config's batch size (96)
and at 512.  Prints one JSON line: ms per step, samples/s, per-stage event times, the recurrent kernel's time per time step
against its MMA-only lower bound, achieved TFLOP/s of the recurrence and of the whole step (algorithmic FLOPs), and the
device name and power limit read in the same run.

    python scripts/bench_lstm_wide.py [--batch 96 512] [--steps 3] [--warmup 1]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from bonito_b200 import synth  # noqa: E402
from bonito_b200.crf.model import Model  # noqa: E402
from bonito_b200.engine import CrfDecoder  # noqa: E402

DENSE_FP16_PEAK = 989e12   # H100 SXM5 dense fp16 tensor throughput (spec sheet, boost clock): the MMA-only bound's divisor


def device_info():
    try:
        out = subprocess.run(["nvidia-smi", "--id=%d" % torch.cuda.current_device(), "--query-gpu=name,power.limit",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(), None
    return name, power


def run(batch, L, steps, warmup, n_lstm):
    spec = synth.model_spec("sup_lstm", n_lstm=n_lstm)
    model = Model(synth.model_config(spec, batchsize=batch, chunksize=L))
    model.load_state_dict(synth.state_dict_from_weights(spec, synth.make_weights(spec, seed=25)))
    model.use_koi(batchsize=batch, chunksize=L, quantize=False)
    model = model.half().eval().to("cuda")
    plan = model.native_plan("cuda")
    x = synth.squiggle(32, L, seed=1).repeat(batch // 32 + 1, 1, 1)[:batch].half().cuda()
    decode = CrfDecoder()
    H, T = plan.hidden, plan.frames(L)
    with torch.inference_mode():
        out = None
        for _ in range(warmup):
            out = plan.forward(x, out=out)
            decode(out, spec["state_len"], 2.0)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            out = plan.forward(x, out=out)
            decode(out, spec["state_len"], 2.0)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / steps
        events = []                                  # one more step with per-kernel events (not part of the timed region)
        out = plan.forward(x, out=out, events=events)
        decode(out, spec["state_len"], 2.0, events=events)
        torch.cuda.synchronize()
    stages = {}
    for name, a, b in events:
        stages[name] = stages.get(name, 0.0) + a.elapsed_time(b)
    C = 4 ** (spec["state_len"] + 1)
    rec = n_lstm * 2.0 * batch * T * 4 * H * H
    step = rec + n_lstm * 2.0 * batch * T * 4 * H * H + 2.0 * batch * T * H * plan.k3 * plan.c2 + 2.0 * batch * T * C * H
    rec_us = stages["lstm_rec"] * 1e3 / (n_lstm * T)
    return {
        "batch": batch, "chunk": L, "frames": T, "ms_per_step": round(ms, 3),
        "samples_per_s": round(batch * L / (ms * 1e-3)), "stages_ms": {k: round(v, 3) for k, v in stages.items()},
        "lstm_rec_us_per_time_step": round(rec_us, 3),
        "lstm_rec_mma_bound_us_per_time_step": round(2.0 * batch * 4 * H * H / DENSE_FP16_PEAK * 1e6, 3),
        "lstm_rec_tflops": round(rec / (stages["lstm_rec"] * 1e-3) / 1e12, 2),
        "step_tflops": round(step / (ms * 1e-3) / 1e12, 2), "step_tflop": round(step / 1e12, 2),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[96, 512])
    ap.add_argument("--chunk", type=int, default=9996)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--n-lstm", type=int, default=5)
    args = ap.parse_args()
    name, power = device_info()
    results = [run(b, args.chunk, args.steps, args.warmup, args.n_lstm) for b in args.batch]
    print(json.dumps({"model": "sup_lstm (dna_r10.4.1@v4.3 shape, H = 1024, 5 LSTM layers)", "device": name,
                      "power_limit": power, "steps": args.steps, "warmup": args.warmup, "results": results}))


if __name__ == "__main__":
    main()
