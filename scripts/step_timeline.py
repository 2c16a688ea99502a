"""Launch-level timeline of the pipelined hac step (two batches in flight): start / end of every kernel of a few steady-state
steps, by stream, from the CUDA events the engine records per launch, and the time of the LSTM stack (`lstm_rec`: all
layers, in chains of tiles, when the input projection is fused in) per step and per time step and layer."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
from bonito_b200 import synth
from bonito_b200.decode import _decoder

dev = torch.device("cuda", 0)
N = int(os.environ.get("TL_BATCH", "512"))
SLOTS = int(os.environ.get("TL_SLOTS", "2"))
model, spec, weights, L = bench.build_hac(dev, 0, 1, batch=N)
x = synth.squiggle(64, L, seed=100).repeat(N // 64 + 1, 1, 1)[:N].contiguous().to(dev, torch.float16)
plan = model.native_plan(dev)
from bonito_b200 import native
streams = [native.new_stream(dev) for _ in range(SLOTS)]


def step(i, events):
    with torch.cuda.stream(streams[i % SLOTS]):
        scores = plan.forward(x, events=events, slot=i % SLOTS)
        _decoder(scores, spec["state_len"], blank_score=plan.blank_score, events=events, slot=i % SLOTS)


with torch.inference_mode():
    for i in range(4):
        step(i, None)
    torch.cuda.synchronize()
    t0 = torch.cuda.Event(enable_timing=True)
    t0.record()
    for st in streams:
        st.wait_event(t0)
    per_step = []
    for i in range(8):
        ev = []
        step(i, ev)
        per_step.append(ev)
    torch.cuda.synchronize()
rows = []
for i, ev in enumerate(per_step):
    for name, a, b in ev:
        rows.append((t0.elapsed_time(a), t0.elapsed_time(b), i, name))
end = max(r[1] for r in rows)
print(f"8 steps in {end:.2f} ms = {end / 8:.2f} ms/step ({SLOTS} in flight)")
lo = min(r[0] for r in rows if r[2] == 4)
for a, b, i, name in sorted(rows):
    if i in (4, 5, 6):
        print(f"step {i} (stream {i % SLOTS})  {name:14s} {a - lo:8.2f} -> {b - lo:8.2f}   {b - a:6.2f} ms")
T = plan.frames(L)
n_layers = len(plan.lstm)
rec = [sum(b - a for a, b, i, name in rows if i == s and name == "lstm_rec") for s in range(4, 8)]
print(f"lstm_rec (the {n_layers}-layer stack): {min(rec):6.2f} .. {max(rec):6.2f} ms per step over steps 4-7, "
      f"{1e3 * sum(rec) / len(rec) / T / n_layers:5.2f} us per time step and layer ({T} steps)")
