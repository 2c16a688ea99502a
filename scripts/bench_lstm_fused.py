"""Time per LSTM time step of the fused width-384 layer (b200_lstm_fused_tile_fwd) at the hac layer shape, alone on the GPU
and as two concurrent launches on two streams (the way the layers of the two batches in flight meet in the pipelined hac
step).

  python scripts/bench_lstm_fused.py [--lib PATH ...] [--n 512] [--t 1666] [--iters 5] [--warmup 2] [--rounds 3] [--out FILE]

Every launch goes through the C ABI of each `--lib` (default: the package's libbonito_b200.so), loaded with ctypes, so that
two builds of the library can be timed in one process: the libraries alternate round by round on the same inputs.  Both
directions are timed.  Per setup and library it prints the median over rounds of the mean wall time of `--iters` launches
(CUDA events, after `--warmup` launches) and that time per time step.  With two or more libraries the outputs are compared
byte for byte.  The card's name and power limit are read in the same run.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
from ctypes import c_int, c_size_t, c_void_p

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H, TB = 384, 64


class Lib:
    def __init__(self, path):
        self.path_arg = path
        self.lib = ctypes.CDLL(os.path.abspath(path))
        self.lib.b200_lstm_fused_tile_fwd.restype = c_int
        self.lib.b200_lstm_fused_tile_fwd.argtypes = [c_void_p] * 6 + [c_int] * 4 + [c_void_p]
        self.lib.b200_lstm_rec_tile_workspace_bytes.restype = c_size_t
        self.lib.b200_lstm_rec_tile_workspace_bytes.argtypes = [c_int]
        self.lib.b200_last_error.restype = ctypes.c_char_p

    def launch(self, x, wih, bias, whh, y, ws, t, n, reverse, stream):
        rc = self.lib.b200_lstm_fused_tile_fwd(x.data_ptr(), wih.data_ptr(), bias.data_ptr(), whh.data_ptr(), y.data_ptr(),
                                               ws.data_ptr(), t, n, H, int(reverse), stream.cuda_stream)
        if rc:
            raise RuntimeError(f"{self.path_arg}: {self.lib.b200_last_error().decode()}")


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable ({e})"
    return {"name": name, "power_limit_and_max_sm_clock": q}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--lib", action="append", default=None, help="libbonito_b200.so to time (repeatable)")
    ap.add_argument("--n", type=int, default=512, help="chunks per launch (hac batch)")
    ap.add_argument("--t", type=int, default=1666, help="time steps (hac: 9996 samples / stride 6)")
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_lstm_fused.py needs a CUDA device")
    from bonito_b200 import native
    paths = args.lib or [native.lib_path()]
    libs = [Lib(p) for p in paths]
    dev = torch.device("cuda:0")
    n, t = args.n, args.t
    nt = -(-n // TB)
    g = torch.Generator().manual_seed(11)
    x = (torch.randn(nt, t, TB, H, generator=g) * 0.5).half().to(dev)
    wih = (torch.randn(4 * H, H, generator=g) / H ** 0.5).half().to(dev)
    whh = (torch.randn(4 * H, H, generator=g) / H ** 0.5).half().to(dev)
    bias = (torch.randn(4 * H, generator=g) * 0.3).half().to(dev)
    ys = [torch.empty(nt, t, TB, H, dtype=torch.float16, device=dev) for _ in range(2)]
    wsb = libs[0].lib.b200_lstm_rec_tile_workspace_bytes(n)
    wss = [torch.empty(wsb, dtype=torch.uint8, device=dev) for _ in range(2)]
    streams = [torch.cuda.Stream(dev) for _ in range(2)]
    main_stream = torch.cuda.current_stream(dev)

    def run(lib, setup, reverse):
        k = 1 if setup == "alone" else 2
        for i in range(k):
            streams[i].wait_stream(main_stream)
            lib.launch(x, wih, bias, whh, ys[i], wss[i], t, n, reverse, streams[i])
        for i in range(k):
            main_stream.wait_stream(streams[i])

    result = {"card": card(), "libs": paths, "n": n, "t": t, "iters": args.iters, "rounds": args.rounds, "setups": {}}
    for reverse in (False, True):
        for setup in ("alone", "two_streams"):
            key = f"{setup}_{'reverse' if reverse else 'forward'}"
            times = {p: [] for p in paths}
            for lib in libs:
                for _ in range(args.warmup):
                    run(lib, setup, reverse)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for _ in range(args.rounds):
                for lib in libs:
                    run(lib, setup, reverse)
                    e0.record(main_stream)
                    for _ in range(args.iters):
                        run(lib, setup, reverse)
                    e1.record(main_stream)
                    torch.cuda.synchronize()
                    times[lib.path_arg].append(e0.elapsed_time(e1) / args.iters)
            row = {"per_lib": {}}
            for p in paths:
                ms = float(np.median(times[p]))
                row["per_lib"][p] = {"ms": round(ms, 3), "ms_rounds": [round(v, 3) for v in times[p]],
                                     "us_per_time_step": round(1e3 * ms / t, 3)}
            if len(libs) > 1:
                outs = []
                for lib in libs:
                    ys[0].fill_(float("nan"))
                    run(lib, "alone", reverse)
                    torch.cuda.synchronize()
                    outs.append(ys[0].clone())
                row["identical"] = all(torch.equal(outs[0].view(torch.int16), o.view(torch.int16)) for o in outs[1:])
                del outs
            result["setups"][key] = row
            print(json.dumps({key: row}), flush=True)
    print(json.dumps(result))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
