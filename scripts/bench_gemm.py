"""Per-shape timing of the wgmma GEMM at the shapes and epilogue maps the benchmarked workloads issue, alone on the GPU.

  python scripts/bench_gemm.py [--lib PATH ...] [--iters 50] [--warmup 10] [--rounds 3] [--only NAME,...] [--out FILE]

Every shape runs through the C ABI (b200_gemm_fwd_ex / b200_gemm_i8_fwd) of each `--lib` (default: the package's
libbonito_b200.so), loaded with ctypes, so that two builds of the library can be timed in one process: the libraries
alternate shape by shape, round by round, on the same inputs.  Per shape and library it prints the median over rounds of
the mean time of `--iters` back-to-back launches (CUDA events, after `--warmup` launches), the achieved TFLOP/s and GB/s,
the larger of the two floors (FLOPs at the fp16 / int8 dense data-sheet rate, bytes at the HBM data-sheet bandwidth), which
one bounds the shape and the share of it reached.  With two or more libraries the outputs of each shape are also compared
byte for byte.  The card's name and power limit are read in the same run.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
from ctypes import c_float, c_int, c_longlong, c_void_p

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# NVIDIA H100 SXM data sheet, dense, 700 W card
PEAK_F16_TFLOPS = 989.0
PEAK_I8_TOPS = 1979.0
PEAK_HBM_GBS = 3350.0


def act_codes():
    from bonito_b200 import native
    return dict(none=native.ACT_NONE, tanh=native.ACT_TANH, clamp=native.ACT_CLAMP, scale=native.ACT_SCALE,
                swiglu=native.ACT_SWIGLU)


def shapes():
    """(name, dict) of every GEMM the headline (hac, bench.py), `--quantize` and sup workloads issue per batch."""
    # hac: 512 chunks x 9996 samples, stride 6 -> T = 1666 frames; tiles of TB = 64 chunks, 8-CTA clusters (CW = 192)
    N, T, TB, CS, H = 512, 1666, 64, 8, 384
    nt = N // TB
    Tp = -(-max(9 + 9996, (T - 1) * 6 + 19) // 6)       # padded frames of the stem output (LstmCrfPlan._buffers)
    CW = 4 * H // CS
    out = [
        ("hac_conv", dict(m=N * Tp, n=H, k=19 * 16, lda=6 * 16, ldc=H, act="tanh", bias=True,
                          map=(Tp, T, TB, 1, TB, T * TB))),
        ("hac_in_proj", dict(m=nt * T * TB, n=4 * H, k=H, lda=H, ldc=CW, bias=True, map=(TB, TB, 1, CS * TB, 0, 0),
                             cb=(CW, TB))),
        ("hac_crf", dict(m=nt * T * TB, n=1024, k=H, lda=H, ldc=1024, act="clamp", lo=-5.0, hi=5.0, bias=True,
                         map=(TB, TB, T, 1, T, TB * T))),
        ("hac_in_proj_i8", dict(m=nt * T * TB, n=4 * H, k=H, lda=H, ldc=CW, bias=True, map=(TB, TB, 1, CS * TB, 0, 0),
                                cb=(CW, TB), i8=True)),
    ]
    # sup: 256 chunks x 9996 samples -> 833 tokens (upsampled x2 to 1666 frames), d_model 512, feed-forward 2048, 4096 scores
    M, d, ff = 256 * 833, 512, 2048
    out += [
        ("sup_qkv", dict(m=M, n=3 * d, k=d, lda=d, ldc=3 * d)),
        ("sup_proj", dict(m=M, n=d, k=d, lda=d, ldc=d, bias=True)),
        ("sup_fc1_swiglu", dict(m=M, n=2 * ff, k=d, lda=d, ldc=ff, act="swiglu")),
        ("sup_fc2", dict(m=M, n=d, k=ff, lda=ff, ldc=d)),
        ("sup_upsample", dict(m=M, n=2 * d, k=d, lda=d, ldc=2 * d, bias=True)),
        ("sup_crf", dict(m=2 * M, n=4096, k=d, lda=d, ldc=4096, act="scale", lo=5.0)),
    ]
    return out


def map_rows(m, rm):
    """Output row of every input row under the epilogue's row map (-1: dropped), as in common.cuh map_row."""
    rows_inner, valid_inner, s_in, s_out, group, s_group = rm
    r = np.arange(m, dtype=np.int64)
    outer, inner = r // rows_inner, r % rows_inner
    o = inner * s_in
    if group > 0:
        o = o + (outer // group) * s_group
        outer = outer % group
    o = o + outer * s_out
    return np.where(inner < valid_inner, o, -1)


class Lib:
    def __init__(self, path):
        self.path_arg = path
        self.lib = ctypes.CDLL(os.path.abspath(path))
        self.lib.b200_gemm_fwd_ex.restype = c_int
        self.lib.b200_gemm_fwd_ex.argtypes = [c_void_p, c_longlong, c_void_p, c_void_p, c_void_p, c_longlong, c_int, c_int,
                                              c_int, c_int, c_float, c_float, c_int, c_int, c_longlong, c_longlong, c_int,
                                              c_longlong, c_int, c_int, c_int, c_int, c_void_p]
        self.lib.b200_gemm_i8_fwd.restype = c_int
        self.lib.b200_gemm_i8_fwd.argtypes = [c_void_p, c_longlong, c_void_p, c_void_p, c_void_p, c_void_p, c_longlong,
                                              c_int, c_int, c_int, c_int, c_float, c_float, c_int, c_int, c_longlong,
                                              c_longlong, c_int, c_longlong, c_int, c_int, c_int, c_void_p]
        self.lib.b200_last_error.restype = ctypes.c_char_p


class Case:
    """Inputs, output buffer and one launch closure of a shape."""

    def __init__(self, name, s, dev):
        self.name, self.s = name, s
        m, n, k, lda = s["m"], s["n"], s["k"], s["lda"]
        i8 = s.get("i8", False)
        g = torch.Generator(device="cpu").manual_seed(7)
        a_elems = (m - 1) * lda + k
        if i8:
            self.a = torch.randint(-127, 128, (a_elems,), generator=g, dtype=torch.int8).to(dev)
            self.b = torch.randint(-127, 128, (n * k,), generator=g, dtype=torch.int8).to(dev)
            self.scale = (torch.rand(n, generator=g) * 1e-4).float().to(dev)
        else:
            self.a = (torch.rand(a_elems, generator=g) * 2 - 1).half().to(dev)
            self.b = ((torch.rand(n * k, generator=g) * 2 - 1) / k ** 0.5).half().to(dev)
            self.scale = None
        self.bias = (torch.rand(n, generator=g) * 0.2 - 0.1).half().to(dev) if s.get("bias") else None
        rm = s.get("map") or (1, 1, 0, 1, 0, 0)     # default: identity, row r -> r
        self.rm = rm
        rows = map_rows(m, rm)
        valid = rows >= 0
        self.valid_rows = int(valid.sum())
        cb = s.get("cb", (0, 0))
        n_out = n // 2 if s.get("act") == "swiglu" else n
        last_row = int(rows.max()) + (n_out // cb[0] - 1) * cb[1] if cb[0] else int(rows.max())
        self.c_elems = (last_row + 1) * s["ldc"]
        self.n_out = n_out
        self.c = torch.zeros(self.c_elems, dtype=torch.float16, device=dev)
        acts = act_codes()
        a = s.get("act", "none")
        self.act, self.lo, self.hi = acts[a], s.get("lo", 0.0), s.get("hi", 0.0)
        self.i8 = i8

    def flops(self):
        return 2.0 * self.s["m"] * self.s["n"] * self.s["k"]

    def bytes(self):
        es = 1 if self.i8 else 2
        a = min(self.s["m"] * self.s["k"], (self.s["m"] - 1) * self.s["lda"] + self.s["k"]) * es
        return a + self.s["n"] * self.s["k"] * es + self.valid_rows * self.n_out * 2

    def floor_ms(self):
        peak = PEAK_I8_TOPS if self.i8 else PEAK_F16_TFLOPS
        t_c = self.flops() / (peak * 1e12) * 1e3
        t_m = self.bytes() / (PEAK_HBM_GBS * 1e9) * 1e3
        return (t_c, "compute") if t_c >= t_m else (t_m, "memory")

    def launch(self, lib, stream):
        s, (ri, vi, si, so, gr, sg) = self.s, self.rm
        cbw, cbr = s.get("cb", (0, 0))
        if self.i8:
            rc = lib.lib.b200_gemm_i8_fwd(self.a.data_ptr(), s["lda"], self.b.data_ptr(), self.scale.data_ptr(),
                                          self.bias.data_ptr() if self.bias is not None else None, self.c.data_ptr(),
                                          s["ldc"], s["m"], s["n"], s["k"], self.act, self.lo, self.hi, ri, vi, si, so, gr,
                                          sg, cbw, cbr, 0, stream)
        else:
            rc = lib.lib.b200_gemm_fwd_ex(self.a.data_ptr(), s["lda"], self.b.data_ptr(),
                                          self.bias.data_ptr() if self.bias is not None else None, self.c.data_ptr(),
                                          s["ldc"], s["m"], s["n"], s["k"], self.act, self.lo, self.hi, ri, vi, si, so, gr,
                                          sg, cbw, cbr, 0, 0, stream)
        if rc:
            raise RuntimeError(f"{self.name}: {lib.lib.b200_last_error().decode()}")


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
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--only", default=None, help="comma-separated shape names")
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_gemm.py needs a CUDA device")
    from bonito_b200 import native
    paths = args.lib or [native.lib_path()]
    libs = [Lib(p) for p in paths]
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream().cuda_stream
    only = set(args.only.split(",")) if args.only else None
    result = {"card": card(), "libs": paths, "iters": args.iters, "rounds": args.rounds, "shapes": {}}
    for name, s in shapes():
        if only and name not in only:
            continue
        case = Case(name, s, dev)
        times = {p: [] for p in paths}
        for lib in libs:                       # warm-up (module load, attribute set-up)
            for _ in range(args.warmup):
                case.launch(lib, stream)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(args.rounds):
            for lib in libs:
                for _ in range(3):
                    case.launch(lib, stream)
                e0.record()
                for _ in range(args.iters):
                    case.launch(lib, stream)
                e1.record()
                torch.cuda.synchronize()
                times[lib.path_arg].append(e0.elapsed_time(e1) / args.iters)
        floor, bound = case.floor_ms()
        row = {"m": s["m"], "n": s["n"], "k": s["k"], "flop": case.flops(), "bytes": case.bytes(),
               "floor_ms": round(floor, 4), "bound": bound, "per_lib": {}}
        for p in paths:
            ms = float(np.median(times[p]))
            row["per_lib"][p] = {"ms": round(ms, 4), "ms_rounds": [round(t, 4) for t in times[p]],
                                 "tflops": round(case.flops() / ms / 1e9, 1), "gbs": round(case.bytes() / ms / 1e6, 1),
                                 "floor_share": round(floor / ms, 3)}
        if len(libs) > 1:                      # byte-for-byte comparison of the outputs of every library
            outs = []
            for lib in libs:
                case.c.zero_()
                case.launch(lib, stream)
                torch.cuda.synchronize()
                outs.append(case.c.clone())
            row["identical"] = all(torch.equal(outs[0].view(torch.int16), o.view(torch.int16)) for o in outs[1:])
            del outs
        result["shapes"][name] = row
        print(json.dumps({name: row}), flush=True)
        del case
        torch.cuda.empty_cache()
    print(json.dumps(result))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
