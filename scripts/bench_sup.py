"""Timing of benchmark config 3: sup v5.0-shaped transformer (18 layers, d=512), batch 256, 9996-sample chunks, 1 GPU."""
import os, sys, json
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from bonito_b200 import synth
from bonito_b200.transformer import Model
from bonito_b200.decode import _decoder
N = int(sys.argv[1]) if len(sys.argv) > 1 else 256
L = int(sys.argv[2]) if len(sys.argv) > 2 else 9996
spec = synth.sup_spec(depth=18)
model = Model(synth.sup_config(spec))
model.load_state_dict(synth.sup_state_dict(spec, synth.make_sup_weights(spec, seed=25)))
model.use_koi(batchsize=N, chunksize=L, quantize=False)
model = model.half().eval().to("cuda")
x = synth.squiggle(32, L, seed=1).repeat(N // 32 + 1, 1, 1)[:N].half().cuda()
plan = model.native_plan("cuda")
with torch.inference_mode():
    for _ in range(2):
        s = plan.forward(x); _decoder(s, 5, blank_score=2.0)
    torch.cuda.synchronize()
    ev = []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    steps = 3
    for _ in range(steps):
        s = plan.forward(x, events=ev); _decoder(s, 5, blank_score=2.0, events=ev)
    e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / steps
agg = {}
for n, a, b in ev: agg[n] = agg.get(n, 0) + a.elapsed_time(b) / steps
flops = 143.4e9 * N * (L / 9996)
print(json.dumps({"model": "sup-shaped transformer, 18 layers", "batch": N, "chunk": L, "ms_per_step": ms,
                  "samples_per_s": N * L / (ms * 1e-3), "model_tflops_per_s": flops / (ms * 1e-3) / 1e12,
                  "stages_ms": {k: round(v, 3) for k, v in agg.items()}}))
