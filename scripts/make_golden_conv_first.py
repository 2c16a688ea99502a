"""
Record the outputs of `b200_conv_first_fwd` from a library built at an earlier commit, so that tests can check that later
builds of the entry point still compute them bit for bit (tests/golden/conv_first_outputs.npz).  Needs a GPU.

    git worktree add /tmp/base <commit> && make -C /tmp/base/bonito_b200/csrc
    python scripts/make_golden_conv_first.py /tmp/base/bonito_b200/libbonito_b200.so <commit>

Cases (the entry point's shapes: c % 8 == 0, c <= 128, odd k <= 15, zero halo rows around each chunk): the sup model's
1 -> 64 k5 swish stem, 1 -> 16 k9 tanh and 1 -> 128 k15 without activation; seeded fp16 inputs, weights and biases.
"""
import ctypes
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = [  # (name, c, k, act, n, l, padl, padr)
    ("c64_k5_swish", 64, 5, 1, 2, 300, 2, 2),
    ("c16_k9_tanh", 16, 9, 2, 3, 257, 4, 7),
    ("c128_k15_none", 128, 15, 0, 2, 100, 7, 7),
]


def inputs(c, k, n, l, seed):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(n, l, generator=gen).half()
    w = (torch.randn(c, 1, k, generator=gen) / np.sqrt(k)).half()
    b = (0.1 * torch.randn(c, generator=gen)).half()
    return x, w, b


def run(lib, case, seed):
    _, c, k, act, n, l, padl, padr = case
    x, w, b = (t.cuda() for t in inputs(c, k, n, l, seed))
    lp = padl + l + padr
    out = torch.full((n * lp, c), 3.0, dtype=torch.float16, device="cuda")
    ptr = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    rc = lib.b200_conv_first_fwd(ptr(x), n, l, c, k, ptr(w), ptr(b), act, ptr(out), lp, padl,
                                 ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, lib.b200_last_error()
    torch.cuda.synchronize()
    return out.cpu()


def load(path):
    lib = ctypes.CDLL(path)
    lib.b200_conv_first_fwd.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                        ctypes.c_int, ctypes.c_void_p]
    lib.b200_last_error.restype = ctypes.c_char_p
    return lib


def main():
    lib = load(sys.argv[1])
    out = {"commit": np.array(sys.argv[2] if len(sys.argv) > 2 else "")}
    for i, case in enumerate(CASES):
        out[case[0]] = run(lib, case, seed=100 + i).numpy()
    path = sys.argv[3] if len(sys.argv) > 3 else os.path.join(ROOT, "tests", "golden", "conv_first_outputs.npz")
    np.savez_compressed(path, **out)
    print(path, {k: v.shape for k, v in out.items()}, os.path.getsize(path))


if __name__ == "__main__":
    main()
