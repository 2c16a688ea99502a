"""
Timing of dna_r10.4.1@v4.0 (H = 1024, per-conv clamps, Linear 1024 -> 256 in front of the head) and dna_r9.4.1@v3 (H = 768,
learned blank scores) on the wide recurrent kernel, and of the decode kernel with learned versus fixed blank scores.
Seeded weights; whole step = resident forward + exact decode, at each model's basecaller chunk size; the decode kernels on
the same random move scores at S = 1024 states, T = 2000 frames, N = 96 chunks, timed alternately with CUDA events.
Prints one JSON line with the device name and power limit read in the same run.

    python scripts/bench_v40_r9v3.py [--batch 96] [--steps 3] [--warmup 1] [--decode-reps 10]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from bonito_b200 import synth  # noqa: E402
from bonito_b200.crf.model import Model  # noqa: E402
from bonito_b200.engine import CrfDecoder  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_lstm_wide import device_info  # noqa: E402

MODELS = {
    # name: (spec, chunk size of the reference config)
    "dna_r10.4.1@v4.0": (synth.v40_spec, 10000),
    "dna_r9.4.1@v3": (lambda: synth.old_style_spec(blank_score=None), 4000),
}


def step(name, batch, steps, warmup):
    make_spec, L = MODELS[name]
    spec = make_spec()
    model = Model(synth.model_config(spec, batchsize=batch, chunksize=L))
    model.load_state_dict(synth.state_dict_from_weights(spec, synth.make_weights(spec, seed=25)))
    model.use_koi(batchsize=batch, chunksize=L, quantize=False)
    model = model.half().eval().to("cuda")
    plan = model.native_plan("cuda")
    x = synth.squiggle(32, L, seed=1).repeat(batch // 32 + 1, 1, 1)[:batch].half().cuda()
    decode = CrfDecoder()
    with torch.inference_mode():
        out = None
        for _ in range(warmup):
            out = plan.forward(x, out=out)
            decode(out, spec["state_len"])
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            out = plan.forward(x, out=out)
            decode(out, spec["state_len"])
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / steps
        events = []                                  # one more step with per-kernel events (not part of the timed region)
        out = plan.forward(x, out=out, events=events)
        decode(out, spec["state_len"], events=events)
        torch.cuda.synchronize()
    stages = {}
    for stage, a, b in events:
        stages[stage] = stages.get(stage, 0.0) + a.elapsed_time(b)
    return {"model": name, "batch": batch, "chunk": L, "frames": plan.frames(L), "scores": plan.n_scores,
            "ms_per_step": round(ms, 3), "samples_per_s": round(batch * L / (ms * 1e-3)),
            "stages_ms": {k: round(v, 3) for k, v in stages.items()}}


def decode_times(n, t, reps):
    """ms per call of the fixed-blank and the learned-blank decode on the same moves (learned blank column: random)."""
    g = torch.Generator().manual_seed(1)
    lb = (torch.randn(n, t, 1024, 5, generator=g) * 1.7).clamp(-5, 5).half().cuda()
    fixed = lb[..., 1:].reshape(n, t, -1).contiguous()
    lb = lb.reshape(n, t, -1).contiguous()
    dec = CrfDecoder()
    times = {"fixed_blank": [], "learned_blank": []}
    with torch.inference_mode():
        for _ in range(2):                           # warm-up: module load, workspace allocation
            dec(fixed, 5, 2.0)
            dec(lb, 5)
        torch.cuda.synchronize()
        for _ in range(reps):                        # alternate the two kernels
            for key, scores in (("fixed_blank", fixed), ("learned_blank", lb)):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                dec(scores, 5, 2.0) if key == "fixed_blank" else dec(scores, 5)
                b.record()
                b.synchronize()
                times[key].append(a.elapsed_time(b))
    out = {"n": n, "t": t, "states": 1024}
    for key, v in times.items():
        v = sorted(v)
        out[key + "_ms"] = {"median": round(v[len(v) // 2], 3), "min": round(v[0], 3), "max": round(v[-1], 3)}
    out["score_bytes"] = {"fixed_blank": n * t * 4096 * 2, "learned_blank": n * t * 5120 * 2}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=96)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--decode-reps", type=int, default=10)
    args = ap.parse_args()
    name, power = device_info()
    results = [step(m, args.batch, args.steps, args.warmup) for m in MODELS]
    print(json.dumps({"device": name, "power_limit": power, "steps": args.steps, "warmup": args.warmup,
                      "results": results, "decode": decode_times(args.batch, 2000, args.decode_reps)}))


if __name__ == "__main__":
    main()
