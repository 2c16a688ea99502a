"""
Dense kernels and the CRF decode at their tile edges, grid-stride limits and output bounds, against float64 references.

Every output buffer is allocated with margins around the region the call may write and filled with a canary bit pattern
(fp16: the NaN 0x7E5A, which no kernel produces; bytes: 0xA5).  After the call, every element the documented map addresses
must have been written, every other element must still hold the canary, and every written value must lie inside the
per-element interval the arithmetic allows (each test's docstring states it).

Intervals are built from a float64 reference with the library's fp16 rounding points (`apply_act_f16` in common.cuh):
where a value is rounded to fp16, the kernel's fp32 value v_k satisfies |v_k - v| <= g (g: the fp32 error bound of the
computation, K * 2^-23 * sum|a_k b_k| for a K-term tensor-core dot product), so the kernel's rounded value is one of
rn16(v - g) .. rn16(v + g) -- a single value unless v lies within g of an fp16 rounding midpoint.  Each later step maps
that set through the operation (with the error of its SFU approximation) and rounds again.  This is the bound
ulp16(ref) + K * 2^-24 * sum|a_k b_k|, sharpened to the fp16 value itself wherever the rounding is not ambiguous.
"""
import math

import numpy as np
import pytest
import torch

from _edges import (CANARY8, CANARY16, CANARY32, E_SFU, _lstm_inputs, _lstm_reference, _perm_hh, _swish, act_interval,
                    bits16, canary16, check_between, check_guarded, gemm_dest, pre16, rn16)
from oracle import crf_oracle as O

pytestmark = pytest.mark.gpu

LOG2E = 1.4426950408889634


# ------------------------------------------------------------------------------------------------ helpers
@pytest.fixture(scope="module")
def native():
    from bonito_b200 import native as nat
    nat.require()
    return nat


# ------------------------------------------------------------------------------------------------ fp16 GEMMs
def _run_gemm(native, impl, m, n, k, act=0, lo=0.0, hi=0.0, bias=True, ldc=None, col_off=0, rows_inner=None,
              valid_inner=None, stride_inner=1, stride_outer=0, group=0, stride_group=0, cb_width=0, cb_rows=0, seed=0):
    """One guarded b200_gemm_fwd_ex call against the interval reference (see the module docstring)."""
    g = torch.Generator().manual_seed(1000 * m + 10 * n + k + act + seed)
    a = (torch.randn(m, k, generator=g)).half()
    w = (torch.randn(n, k, generator=g) / k ** 0.5).half()
    bv = (torch.randn(n, generator=g) * 0.5).half() if bias else None
    ri = m if rows_inner is None else rows_inner
    vi = m if valid_inner is None else valid_inner
    swiglu = act == native.ACT_SWIGLU
    n_out = n // 2 if swiglu else n
    ldc = ldc or (cb_width or n_out)
    dest = gemm_dest(m, n_out, ri, vi, stride_inner, stride_outer, group, stride_group, cb_width, cb_rows, ldc)
    keep = dest >= 0
    dest = dest + col_off
    span = int(dest.max()) + 1
    front = 2 * ldc + 8                                  # margin rows (and 8 columns) before the output, 16-byte aligned
    buf = canary16(front + span + 2 * ldc + 8)
    c = buf[front:]
    native.gemm(a.cuda(), k, w.cuda(), None if bv is None else bv.cuda(), c[col_off:], ldc, m, n, k, act=act, lo=lo, hi=hi,
                rows_inner=ri, valid_inner=vi, stride_inner=stride_inner, stride_outer=stride_outer, group=group,
                stride_group=stride_group, cb_width=cb_width, cb_rows=cb_rows, impl=impl)
    torch.cuda.synchronize()
    a64, w64 = a.double().numpy(), w.double().numpy()
    v = a64 @ w64.T + (bv.double().numpy() if bias else 0.0)
    gam = k * 2.0 ** -23 * (np.abs(a64) @ np.abs(w64).T) + 2.0 ** -24 * np.abs(v)
    p_lo, p_hi = pre16(v, gam)
    if swiglu:                                       # 64-column groups [32 y | 32 gate] -> 32 outputs
        G = n // 64
        yl, yh = (x.reshape(m, G, 2, 32)[:, :, 0].reshape(m, n_out) for x in (p_lo, p_hi))
        gl, gh = (x.reshape(m, G, 2, 32)[:, :, 1].reshape(m, n_out) for x in (p_lo, p_hi))
        cands = [yy * _swish(gg) for yy in (yl, yh) for gg in (gl, gh)]
        s_lo, s_hi = np.minimum.reduce(cands), np.maximum.reduce(cands)
        e = E_SFU * (1 + np.abs(s_hi)) * (1 + np.maximum(np.abs(yl), np.abs(yh)))
        out_lo, out_hi = rn16(s_lo - e), rn16(s_hi + e)
    else:
        out_lo, out_hi = act_interval(p_lo, p_hi, act, lo, hi)
    bits = bits16(buf)
    check_guarded(bits, dest[keep] + front, CANARY16)
    got = buf.float().cpu().numpy().astype(np.float64)[dest[keep] + front]
    check_between(got, out_lo[keep], out_hi[keep], f"gemm m={m} n={n} k={k} act={act}")


WG_SHAPES = ([pytest.param(mm, 136, 72, id=f"M={mm}") for mm in (1, 63, 64, 65, 127, 128, 129, 257)]
             + [pytest.param(129, nn, 72, id=f"N={nn}") for nn in (8, 120, 128)]
             + [pytest.param(129, 136, 72, id="N=136-second-tile-8-cols"), pytest.param(129, 264, 72, id="N=264-third-tile")]
             + [pytest.param(129, 136, kk, id=f"K={kk}-{-(-kk // 64)}-stages") for kk in (8, 56, 64, 72, 136, 192, 200)])
MMA_SHAPES = ([pytest.param(mm, 136, 40, id=f"M={mm}") for mm in (1, 63, 64, 65, 127, 128, 129, 257)]
              + [pytest.param(129, nn, 40, id=f"N={nn}") for nn in (8, 120, 128, 136, 264)]
              + [pytest.param(129, 136, kk, id=f"K={kk}-{-(-kk // 32)}-stages") for kk in (8, 24, 32, 40, 104)])
ACTS = [pytest.param(0, 0.0, 0.0, id="NONE"), pytest.param(1, 0.0, 0.0, id="SWISH"), pytest.param(2, 0.0, 0.0, id="TANH"),
        pytest.param(3, -1.0, 1.5, id="CLAMP"), pytest.param(4, 3.0, 0.0, id="SCALE"),
        pytest.param(6, 5.0, 0.0, id="TANH_SCALE"), pytest.param(7, -0.5, 3.5, id="SWISH_CLAMP"),
        pytest.param(8, 0.0, 0.0, id="RELU")]
# (kwargs, m, n): the row / column maps; rows_inner = 37 does not divide the 128-row tile
MAPS = [
    pytest.param(dict(), 129, 136, id="identity"),
    pytest.param(dict(rows_inner=37, valid_inner=33, stride_inner=5, stride_outer=1), 185, 136, id="valid_inner=33<rows_inner=37"),
    # engine.py's conv GEMM into the tile layout: rows (chunk, frame) -> [tile][frame][chunk in tile], 70 chunks = 1.1 tiles
    pytest.param(dict(rows_inner=13, valid_inner=11, stride_inner=64, stride_outer=1, group=64, stride_group=11 * 64), 70 * 13,
                 136, id="group-tile-layout-TB=64"),
    pytest.param(dict(cb_width=32, cb_rows=131), 129, 136, id="cb_width=32-partial-last-block"),
    pytest.param(dict(cb_width=192, cb_rows=133), 129, 264, id="cb_width=192"),
    pytest.param(dict(ldc=160, col_off=8), 129, 136, id="ldc>n-column-window"),
]


@pytest.mark.parametrize("m,n,k", WG_SHAPES)
def test_wgmma_gemm_tile_edges(native, m, n, k):
    """wgmma GEMM (128 x 128 tiles, 64-element K stages, 3-stage ring) at partial M / N tiles and 1-4 K stages.  Bound:
    the fp16 output lies in [rn16(v - g), rn16(v + g)], v = sum a_k b_k + bias in float64, g = K 2^-23 sum|a_k b_k| +
    2^-24 |v| (fp32 accumulation, truncating adds allowed, and the bias add)."""
    _run_gemm(native, native.GEMM_TCGEN05, m, n, k)


@pytest.mark.parametrize("m,n,k", MMA_SHAPES)
def test_mma_gemm_tile_edges(native, m, n, k):
    """mma.sync GEMM (128 x 128 tiles, BK = 32) at the same M / N edges and 1-4 K stages; bound as for the wgmma test."""
    _run_gemm(native, native.GEMM_MMA_SYNC, m, n, k)


@pytest.mark.parametrize("impl", ["wgmma", "mma"])
@pytest.mark.parametrize("act,lo,hi", ACTS)
def test_gemm_epilogue_activations(native, impl, act, lo, hi):
    """Every epilogue activation on a partial tile (M = 129, N = 136).  Bound: the fp16 pre-activation is rn16(v -/+ g) as
    in the tile-edge tests; the activation of each candidate is taken in float64 with +-2^-19 (1 + |x|) for the ex2 / rcp
    approximations (their relative errors are below 2^-21), then rounded to fp16 (SCALE / TANH_SCALE: +-2^-24 relative for
    the fp32 multiply; TANH_SCALE rounds tanh to fp16 before it).  The interval is a single fp16 value unless a rounding
    is within these errors of a midpoint."""
    _run_gemm(native, native.GEMM_TCGEN05 if impl == "wgmma" else native.GEMM_MMA_SYNC, 129, 136, 72, act=act, lo=lo, hi=hi)


@pytest.mark.parametrize("n", [pytest.param(64, id="N=64-one-group"), pytest.param(128, id="N=128-one-tile"),
                               pytest.param(192, id="N=192-partial-second-tile")])
def test_wgmma_gemm_swiglu(native, n):
    """The fused SwiGLU epilogue: c[:, 32G + j] = fp16(g y / (1 + e^-g)) from the fp16-rounded y (column 64G + j) and gate
    (column 64G + 32 + j).  Bound: y and g each take their candidates rn16(v -/+ g); the product over all four
    combinations, widened by 2^-19 (1 + |out|)(1 + |y|) for __expf and rcp.approx, then rounded."""
    _run_gemm(native, native.GEMM_TCGEN05, 129, n, 72, act=native.ACT_SWIGLU, bias=False)


@pytest.mark.parametrize("impl", ["wgmma", "mma"])
@pytest.mark.parametrize("kw,m,n", MAPS)
def test_gemm_row_and_column_maps(native, impl, kw, m, n):
    """The epilogue row map (rows dropped by valid_inner, the two-level group map of the tile layout), column blocks (the
    gaps between blocks and the unwritten columns of a partial last block) and a column window of a wider output: every
    mapped element written and inside the tile-edge bound, every other element of the buffer untouched."""
    _run_gemm(native, native.GEMM_TCGEN05 if impl == "wgmma" else native.GEMM_MMA_SYNC, m, n, 72, **kw)


# ------------------------------------------------------------------------------------------------ int8 GEMM
I8_CASES = ([pytest.param(129, 136, kk, 0, {}, id=f"K={kk}") for kk in (16, 112, 128, 144, 400)]
            + [pytest.param(129, 8, 144, 0, {}, id="N=8"), pytest.param(1, 136, 144, 0, {}, id="M=1"),
               pytest.param(257, 136, 144, 0, {}, id="M=257-tail-1"),
               pytest.param(129, 136, 144, 3, {}, id="CLAMP"), pytest.param(129, 136, 144, 2, {}, id="TANH"),
               pytest.param(70 * 13, 136, 144, 0, dict(rows_inner=13, valid_inner=11, stride_inner=64, stride_outer=1,
                                                        group=64, stride_group=11 * 64), id="group-tile-layout-TB=64")])


@pytest.mark.parametrize("m,n,k,act,kw", I8_CASES)
def test_int8_gemm_edges(native, m, n, k, act, kw):
    """int8 GEMM (wgmma s8, 128-byte K stages): the s32 accumulation is exact, the epilogue is one fmaf(acc, scale, bias)
    (|acc| < 2^24, so acc is exact in fp32).  Bound: rn16(v -/+ 2^-24 |v|) with v = acc * scale + bias in float64, then
    the activation as in the fp16 epilogue test."""
    g = torch.Generator().manual_seed(m + n + k + act)
    a = torch.randint(-127, 128, (m, k), generator=g, dtype=torch.int8)
    w = torch.randint(-127, 128, (n, k), generator=g, dtype=torch.int8)
    scale = ((torch.rand(n, generator=g) + 0.5) / (k ** 0.5 * 4000.0)).float()
    bv = (torch.randn(n, generator=g) * 0.5).half()
    lo, hi = (-1.0, 1.5) if act == 3 else (0.0, 0.0)
    ri, vi = kw.get("rows_inner", m), kw.get("valid_inner", m)
    dest = gemm_dest(m, n, ri, vi, kw.get("stride_inner", 1), kw.get("stride_outer", 0), kw.get("group", 0),
                     kw.get("stride_group", 0), 0, 0, n)
    front = 2 * n + 8
    buf = canary16(front + int(dest.max()) + 1 + 2 * n + 8)
    native.gemm_i8(a.cuda(), k, w.cuda(), scale.cuda(), bv.cuda(), buf[front:], n, m, n, k, act=act, lo=lo, hi=hi,
                   rows_inner=ri, valid_inner=vi, stride_inner=kw.get("stride_inner", 1),
                   stride_outer=kw.get("stride_outer", 0), group=kw.get("group", 0), stride_group=kw.get("stride_group", 0))
    torch.cuda.synchronize()
    acc = a.double().numpy() @ w.double().numpy().T
    assert np.abs(acc).max() < 2 ** 24
    v = acc * scale.double().numpy() + bv.double().numpy()
    p_lo, p_hi = pre16(v, 2.0 ** -24 * np.abs(v))
    out_lo, out_hi = act_interval(p_lo, p_hi, act, lo, hi)
    keep = dest >= 0
    check_guarded(bits16(buf), dest[keep] + front, CANARY16)
    got = buf.float().cpu().numpy().astype(np.float64)[dest[keep] + front]
    check_between(got, out_lo[keep], out_hi[keep], "gemm_i8")


# ------------------------------------------------------------------------------------------------ rmsnorm, swiglu
RMS_CASES = ([pytest.param(d, 9, id=f"d={d}") for d in (256, 768, 1024)]
             + [pytest.param(512, mm, id=f"M={mm}") for mm in (1, 7, 8, 9, 1001)]
             + [pytest.param(768, 1001, id="d=768-M=1001")])


@pytest.mark.parametrize("d,m", RMS_CASES)
def test_rmsnorm_residual_edges(native, d, m):
    """rmsnorm_residual (8 rows per CTA, one warp per row): out = fp16(s * rsqrt(mean(s^2) + eps) * w), s = a + fp16(alpha x).
    Bound: fp16(alpha x) takes its candidates rn16(u -/+ 2^-24 |u|) (the fp32 product rounds first); with those,
    v = s rstd w in float64 and the relative error of the fp32 path is at most 2^-24 (d/2 + 4) (sum of squares,
    halved by the square root, the add and two multiplies) + 2^-21 (rsqrt.approx), plus the effect of the candidate
    spread on the mean square; the output lies in [rn16(v - e), rn16(v + e)].  Rows >= M stay untouched."""
    g = torch.Generator().manual_seed(d + m)
    a = torch.randn(m, d, generator=g).half()
    x = torch.randn(m, d, generator=g).half()
    w = (torch.rand(d, generator=g) + 0.5).half()
    alpha, eps = 2.4494897, 1e-5
    front = 2 * d
    buf = canary16(front + m * d + 3 * d)
    native.rmsnorm_residual(a.cuda(), x.cuda(), w.cuda(), alpha, eps, buf[front:], m, d)
    torch.cuda.synchronize()
    u = np.float32(alpha) * x.double().numpy()
    h_lo, h_hi = pre16(u, 2.0 ** -24 * np.abs(u))
    a64, w64 = a.double().numpy(), w.double().numpy()
    s = a64 + rn16(u)
    ms = (s * s).mean(axis=1, keepdims=True)
    spread = np.maximum(np.abs(a64 + h_lo - s), np.abs(a64 + h_hi - s))
    rel = 2.0 ** -24 * (d / 2 + 4) + 2.0 ** -21 + (2 * np.abs(s) * spread + spread ** 2).sum(axis=1, keepdims=True) / (2 * d * ms)
    lo_v = np.minimum(a64 + h_lo, a64 + h_hi) / np.sqrt(ms + eps) * w64
    hi_v = np.maximum(a64 + h_lo, a64 + h_hi) / np.sqrt(ms + eps) * w64
    v_lo, v_hi = np.minimum(lo_v, hi_v), np.maximum(lo_v, hi_v)
    out_lo, out_hi = rn16(v_lo - rel * np.abs(v_lo)), rn16(v_hi + rel * np.abs(v_hi))
    check_guarded(bits16(buf), front + np.arange(m * d), CANARY16)
    got = buf[front:front + m * d].float().cpu().numpy().astype(np.float64).reshape(m, d)
    check_between(got, out_lo, out_hi, f"rmsnorm d={d} M={m}")


def test_rmsnorm_refuses_an_unsupported_width(native):
    z = torch.zeros(4 * 640, dtype=torch.float16, device="cuda")
    with pytest.raises(native.NativeError, match="not supported"):
        native.rmsnorm_residual(z, z, z, 1.0, 1e-5, z, 4, 640)


@pytest.mark.parametrize("m,f", [pytest.param(3, 8, id="M=3-F=8-one-partial-block"),
                                 pytest.param(1001, 96, id="M=1001-F=96-partial-last-block"),
                                 pytest.param(257, 512, id="M=257-F=512-whole-blocks")])
def test_swiglu_partial_blocks(native, m, f):
    """swiglu (256 threads x 8 elements per block): out = fp16(g y / (1 + __expf(-g))) on fp16 inputs.  Bound: the
    float64 value v within 2^-19 |v| + 2^-30 (ex2.approx, the add, the IEEE division), rounded: [rn16(v - e), rn16(v + e)].
    Nothing past M * F is written."""
    g = torch.Generator().manual_seed(m * f)
    h = (torch.randn(m, 2 * f, generator=g) * 2).half()
    buf = canary16(64 + m * f + 64)
    native.swiglu(h.cuda(), buf[64:], m, f)
    torch.cuda.synchronize()
    y, gt = h[:, :f].double().numpy(), h[:, f:].double().numpy()
    v = y * _swish(gt)
    e = 2.0 ** -19 * np.abs(v) + 2.0 ** -30
    check_guarded(bits16(buf), 64 + np.arange(m * f), CANARY16)
    got = buf[64:64 + m * f].float().cpu().numpy().astype(np.float64).reshape(m, f)
    check_between(got, rn16(v - e), rn16(v + e), "swiglu")


# ------------------------------------------------------------------------------------------------ first convolutions
def _conv_first_reference(x, w, bias, stride, T, lp, padl):
    """float64 pre-activations [N, lp, C] of Conv1d(1 -> C, k, stride, pad k/2) at rows padl .. padl + T, and the
    fp32 error bound of each (K fmaf roundings of the running sum)."""
    n, L = x.shape
    c, _, k = w.shape
    P = k // 2
    xp = np.zeros((n, L + 2 * P + stride * T), dtype=np.float64)
    xp[:, P:P + L] = x
    win = np.stack([xp[:, t * stride:t * stride + k] for t in range(T)], axis=1)       # [N, T, K]
    w2 = w[:, 0, :].T                                                                    # [K, C]
    v = win @ w2 + bias
    gam = (k + 1) * 2.0 ** -24 * (np.abs(win) @ np.abs(w2) + np.abs(bias))
    return v, gam


def _check_conv_first(buf, front, n, lp, padl, T, c, ldo, col, v, gam, act, lo=0.0, hi=0.0):
    rows = np.arange(n * lp).reshape(n, lp)
    dest = (rows[:, :, None] * ldo + col + np.arange(c)[None, None, :]) + front
    check_guarded(bits16(buf), dest, CANARY16)
    got = buf.float().cpu().numpy().astype(np.float64)[dest]
    frames = slice(padl, padl + T)
    assert (got[:, :padl] == 0).all() and (got[:, padl + T:] == 0).all(), "rows outside the frames are not zero"
    out_lo, out_hi = act_interval(*pre16(v, gam), act, lo, hi)
    check_between(got[:, frames], out_lo, out_hi, "conv_first")


CF_CASES = ([pytest.param(8, 15, 129, 9, id="C=8-K=15-lp=129-padl>K/2")]
            + [pytest.param(128, 15, 129, 9, id="C=128"), pytest.param(8, 1, 129, 9, id="K=1")]
            + [pytest.param(8, 15, lp, 9, id=f"lp={lp}") for lp in (127, 128, 257)]
            + [pytest.param(8, 15, 129, 0, id="padl=0")])


@pytest.mark.parametrize("c,k,lp,padl", CF_CASES)
def test_conv_first_row_blocks(native, c, k, lp, padl):
    """conv_first (128 output rows per CTA, C <= 128, odd K <= 15) + swish, channels-last with a zero halo.  Bound: the
    pre-activation rounds to rn16(v -/+ g), g = (K + 1) 2^-24 sum|w x| (fmaf chain from the bias), then swish as in the
    GEMM epilogue test; halo rows are exactly 0; nothing outside [N][lp][C] is written."""
    n = 3
    L = lp - padl - 3
    g = torch.Generator().manual_seed(c + k + lp + padl)
    x = torch.randn(n, L, generator=g).half()
    w = (torch.randn(c, 1, k, generator=g) / k ** 0.5).half()
    b = (torch.randn(c, generator=g) * 0.3).half()
    front = 2 * c
    buf = canary16(front + n * lp * c + 2 * c)
    native.conv_first(x.cuda(), w.cuda(), b.cuda(), native.ACT_SWISH, buf[front:], lp, padl)
    torch.cuda.synchronize()
    v, gam = _conv_first_reference(x.double().numpy(), w.double().numpy(), b.double().numpy(), 1, L, lp, padl)
    _check_conv_first(buf, front, n, lp, padl, L, c, c, 0, v, gam, native.ACT_SWISH)


@pytest.mark.parametrize("c", [pytest.param(8, id="C=8"), pytest.param(72, id="C=72-second-64-channel-CTA"),
                               pytest.param(512, id="C=512")])
def test_conv_first_ex_column_window(native, c):
    """conv_first_ex (64 channels per CTA) with stride 8 and K = 33, writing columns [8, 8 + C) of rows with pitch
    C + 24: the frames, the zero rows around them, and nothing in the other columns or the margins.  Bound as for
    conv_first, with swish-and-clamp."""
    n, stride, k, padl = 2, 8, 33, 5
    L = 8 * 150 + 3
    T = (L - 1) // stride + 1
    lp = padl + T + 4
    ldo, col = c + 24, 8
    g = torch.Generator().manual_seed(c)
    x = torch.randn(n, L, generator=g).half()
    w = (torch.randn(c, 1, k, generator=g) / k ** 0.5).half()
    b = (torch.randn(c, generator=g) * 0.3).half()
    front = 2 * ldo
    buf = canary16(front + n * lp * ldo + 2 * ldo)
    native.conv_first_ex(x.cuda(), w.cuda(), b.cuda(), native.ACT_SWISH_CLAMP, buf[front + col:], ldo, lp, padl,
                         stride=stride, lo=-0.5, hi=3.5)
    torch.cuda.synchronize()
    v, gam = _conv_first_reference(x.double().numpy(), w.double().numpy(), b.double().numpy(), stride, T, lp, padl)
    _check_conv_first(buf, front, n, lp, padl, T, c, ldo, col, v, gam, native.ACT_SWISH_CLAMP, -0.5, 3.5)


# ------------------------------------------------------------------------------------------------ ctc_head
def _ctc_cases():
    cases = [pytest.param(f, 1001, id=f"F={f}-lanes={lpr}") for f, lpr in ((8, 1), (16, 2), (32, 4), (64, 8), (136, 16))]
    cases.append(pytest.param(2048, 1001, id="F=2048-limit-lanes=32"))
    cases += [pytest.param(64, mm, id=f"M={mm}") for mm in (1, 31, 33)]        # F = 64: 32 rows per CTA
    cases += [pytest.param(64, "stride", id="F=64-grid-stride"), pytest.param(8, "stride", id="F=8-grid-stride"),
              pytest.param(2048, "stride", id="F=2048-grid-stride")]
    return cases


@pytest.mark.parametrize("f,m", _ctc_cases())
def test_ctc_head_lanes_and_grid_stride(native, f, m):
    """ctc_head: logits = fp16(x w^T + b), logp = fp16(log_softmax) in fp32, label = argmax (ties: highest index), prob =
    exp(logp[label]).  Bound: each logit rounds to rn16(l -/+ g), g = (F + 1) 2^-24 sum|x w| (fmaf chains and the lane
    reduction); log_softmax is increasing in its own logit and decreasing in the others, so logp[c] lies between its values
    at the extreme candidates, widened by 2^-20 (2 + |max logit| + |lse|) for expf / logf / the fp32 sums, then rounded.
    The label is the kernel's own argmax and equals the reference's wherever the top class's interval is strictly above
    the others; prob = exp(kernel logp[label]) within 2^-21 relative.  Grid-stride cases use M > 8 x SMs x rows-per-CTA."""
    lpr = 32 if f // 8 >= 32 else 16 if f // 8 > 8 else 8 if f // 8 > 4 else 4 if f // 8 > 2 else 2 if f // 8 > 1 else 1
    rows_per_cta = 8 * (32 // lpr)
    if m == "stride":
        m = 8 * torch.cuda.get_device_properties(0).multi_processor_count * rows_per_cta + rows_per_cta + 3
    g = torch.Generator().manual_seed(f + m)
    x = torch.randn(m, f, generator=g).half()
    w = (torch.randn(5, f, generator=g) * 2.0 / f ** 0.5).half()
    b = (torch.randn(5, generator=g) * 0.5).half()
    lp_buf = canary16(8 + 5 * m + 8)
    lab_buf = torch.full((64 + m + 64,), CANARY8, dtype=torch.uint8, device="cuda")
    pr_buf = torch.full((4 + m + 4,), CANARY32, dtype=torch.int32, device="cuda")
    native.ctc_head(x.cuda(), m, w.cuda(), b.cuda(), lab_buf[64:], pr_buf[4:].view(torch.float32), lp_buf[8:])
    torch.cuda.synchronize()
    x64, w64 = x.double().numpy(), w.double().numpy()
    l = x64 @ w64.T + b.double().numpy()
    gam = (f + 1) * 2.0 ** -24 * (np.abs(x64) @ np.abs(w64).T + np.abs(b.double().numpy()))
    l_lo, l_hi = pre16(l, gam)

    def lse(z):
        mx = z.max(axis=1, keepdims=True)
        return mx + np.log(np.exp(z - mx).sum(axis=1, keepdims=True))

    lp_lo, lp_hi = np.empty_like(l), np.empty_like(l)
    for c in range(5):
        z = l_hi.copy()
        z[:, c] = l_lo[:, c]
        lp_lo[:, c] = l_lo[:, c] - lse(z)[:, 0]
        z = l_lo.copy()
        z[:, c] = l_hi[:, c]
        lp_hi[:, c] = l_hi[:, c] - lse(z)[:, 0]
    e = 2.0 ** -20 * (2 + np.abs(l_hi).max(axis=1, keepdims=True) + np.abs(lse(l_hi)))
    out_lo, out_hi = rn16(lp_lo - e), rn16(lp_hi + e)
    check_guarded(bits16(lp_buf), 8 + np.arange(5 * m), CANARY16)
    lab_bits = lab_buf.cpu().numpy()
    check_guarded(lab_bits, 64 + np.arange(m), CANARY8)
    assert (lab_bits[64:64 + m] < 5).all()
    pr_bits = pr_buf.cpu().numpy().view(np.uint32).astype(np.int64)
    check_guarded(pr_bits, 4 + np.arange(m), CANARY32)
    got_lp = lp_buf[8:8 + 5 * m].float().cpu().numpy().astype(np.float64).reshape(m, 5)
    check_between(got_lp, out_lo, out_hi, "ctc_head logp")
    labels = lab_bits[64:64 + m].astype(np.int64)
    own = 4 - np.argmax(got_lp[:, ::-1], axis=1)                     # highest index among equal maxima
    assert np.array_equal(labels, own)
    top = np.argmax(out_lo, axis=1)
    others = np.where(np.arange(5)[None, :] == top[:, None], -np.inf, out_hi)
    clear = out_lo[np.arange(m), top] > others.max(axis=1)
    assert clear.mean() > 0.9 and np.array_equal(labels[clear], top[clear])
    probs = pr_buf[4:4 + m].view(torch.float32).cpu().numpy().astype(np.float64)
    want = np.exp(got_lp[np.arange(m), labels])
    assert (np.abs(probs - want) <= 2.0 ** -21 * want).all()


# ------------------------------------------------------------------------------------------------ LSTM recurrences
LSTM_CASES = ([pytest.param(128, 33, 37, False, id="base-H=128-n=33-T=37")]
              + [pytest.param(H, 33, 37, False, id=f"H={H}") for H in (96, 256)]
              + [pytest.param(128, nn, 37, False, id=f"n={nn}") for nn in (31, 32, 65)]
              + [pytest.param(256, 65, 37, False, id="H=256-n=65-three-clusters")]
              + [pytest.param(128, 33, tt, False, id=f"T={tt}") for tt in (1, 2)]
              + [pytest.param(128, 33, 37, True, id="reverse"), pytest.param(256, 33, 2, True, id="H=256-T=2-reverse")])


@pytest.mark.parametrize("H,n,T,reverse", LSTM_CASES)
def test_lstm_rec_clusters(native, H, n, T, reverse):
    """mma.sync recurrent kernel (32-chunk clusters): partial and multiple clusters, T = 1, 2, 37, both directions.  Bound:
    carried per element through the recurrence -- gate errors from the h error (|W_hh| e_h), fp32 accumulation (H 2^-23
    sum|w h|) and the gx add; sigma' <= 1/4 and tanh' <= 1 into c and h, plus 2^-19 per SFU evaluation; the fp16 output
    in [rn16(h - e), rn16(h + e)].  Nothing around y [T][n][H] is written."""
    gx, whh = _lstm_inputs(T, n, H, seed=H + n + T)
    gx_k = gx.permute(0, 1, 3, 2).reshape(T, n, 4 * H).contiguous()       # columns [unit][gate]
    front = 64
    buf = canary16(front + T * n * H + 64)
    native.lstm_rec(gx_k.cuda(), whh[_perm_hh(H)].cuda(), buf[front:], T, n, H, reverse)
    torch.cuda.synchronize()
    lo, hi = _lstm_reference(gx, whh, reverse)
    check_guarded(bits16(buf), front + np.arange(T * n * H), CANARY16)
    got = buf[front:front + T * n * H].float().cpu().numpy().astype(np.float64).reshape(T, n, H)
    check_between(got, lo, hi, f"lstm_rec H={H} n={n} T={T}")


@pytest.mark.parametrize("n,T,reverse", [pytest.param(65, 5, False, id="n=65-second-tile-1-chunk"),
                                         pytest.param(128, 5, True, id="n=128-two-full-tiles"),
                                         pytest.param(129, 3, False, id="n=129-third-tile")])
def test_lstm_rec_tile_tiles(native, n, T, reverse):
    """Width-384 tile kernel (64-chunk tiles, 8-CTA clusters): a third tile, a one-chunk tile; bound as for lstm_rec (its
    cell math has the same derivatives; the clamp of the exponent arguments changes sigma by < 1e-9).  Rows of chunks >= n
    in the last tile and the margins stay untouched."""
    H, TBK, CS = 384, 64, 8
    assert (native.lstm_tile_chunks(H), native.lstm_tile_cluster(H)) == (TBK, CS)
    tiles = -(-n // TBK)
    gx, whh = _lstm_inputs(T, n, H, seed=n + T)
    pad = torch.zeros(T, tiles * TBK, 4, H, dtype=torch.float16)
    pad[:, :n] = gx
    # [T][tiles*64][gate][rank*48 + u] -> [tiles][T][rank][64][u][gate]
    gx_k = pad.view(T, tiles, TBK, 4, CS, H // CS).permute(1, 0, 4, 2, 5, 3).contiguous()
    front = 64
    size = tiles * T * TBK * H
    buf = canary16(front + size + 64)
    native.lstm_rec_tile(gx_k.cuda(), whh[_perm_hh(H)].cuda(), buf[front:], T, n, H, reverse)
    torch.cuda.synchronize()
    lo, hi = _lstm_reference(gx, whh, reverse)
    idx = (np.arange(tiles * T * TBK * H).reshape(tiles, T, TBK, H).transpose(1, 0, 2, 3).reshape(T, tiles * TBK, H)[:, :n])
    check_guarded(bits16(buf), front + idx, CANARY16)
    got = buf.float().cpu().numpy().astype(np.float64)[front + idx]
    check_between(got, lo, hi, f"lstm_rec_tile n={n}")


# ------------------------------------------------------------------------------------------------ CRF decode
# Relative error bound of the kernel's posterior move mass p (fp32 posteriors from ex2.approx / lg2.approx, normalised
# every step with an fp64 k_t): 2^-21 from the two ex2.approx of each posterior, 2^-24 log2(S) for the summation over
# states, and per frame of the two log2-domain recursions (alpha' forward, beta' backward) one lg2.approx (<= 2^-22
# absolute) and three fp32 roundings of re-centred values below 2^6 (<= 2^-18 each) that the posteriors of later frames
# inherit: eta(T) = 2^-20 + 2^-18 (1 + 2T) for the worst case in which every rounding has the same sign.
# Measured on an H100 80GB HBM3 (700 W power limit) over the 36 cases below: every quality equals rint(q*) + 33, so no
# case needed the band (worst implied relative error of p: 0; eta ranges from 3.5e-5 at T = 4 to 2.0e-3 at T = 513).
def decode_eta(T):
    return 2.0 ** -20 + 2.0 ** -18 * (1 + 2 * T)


def _check_qualities(qual, moves, seq, mass, T, qscale, qbias):
    """The kernel quality equals rint(q*) + 33 for every emitted base, except where q* is within delta of a rounding
    midpoint; returns the largest relative error of p that any observed mismatch implies (0 if none)."""
    base = np.searchsorted(np.frombuffer(b"ACGT", dtype=np.uint8), seq)
    emit = moves == 1
    p = np.take_along_axis(mass, np.clip(base, 0, 3)[..., None], axis=-1)[..., 0]
    err = np.maximum(1.0 - p, 1e-4)
    qs = -10.0 * np.log10(err) * qscale + qbias
    slope = qscale * 10.0 / math.log(10.0) * p / err                     # dq*/d(ln p)
    delta = slope * decode_eta(T) + 2.0 ** -16 * (1 + np.abs(qs))        # + log10f / fp32 rounding of q
    dist = np.abs(qs - (np.floor(qs) + 0.5))                             # distance to the nearest midpoint
    want = np.clip(np.rint(qs) + 33, 33, 126)
    q = qual.astype(np.int64)
    assert (q[~emit] == 0).all()
    dq = np.abs(q - want)[emit]
    assert (dq <= 1).all(), f"a quality differs by {dq.max()}"
    bad = emit & (q != want)
    assert (dist[bad] <= delta[bad]).all(), \
        f"{int((dist[bad] > delta[bad]).sum())} qualities differ from rint(q*) outside the derived band"
    return float((dist[bad] / np.maximum(slope[bad], 1e-30)).max()) if bad.any() else 0.0


def _decode_cases():
    out = []
    for k in (3, 4, 5):
        tb = 16384 // 4 ** k
        for T, name in ((4, "4"), (5, "5"), (tb - 1, "TB-1"), (tb, "TB"), (tb + 1, "TB+1"), (2 * tb + 1, "2TB+1")):
            for lb in (False, True):
                out.append(pytest.param(k, T, lb, id=f"k={k}-T={name}={T}-{'learned' if lb else 'fixed'}-blank"))
    return out


@pytest.mark.parametrize("k,T,lb", _decode_cases())
def test_crf_decode_traceback_blocks(native, k, T, lb):
    """crf_decode / crf_decode_lb at the trace-back block (TB = 16384 / 4^k rows) and prefetch-ring seams.  Moves and
    sequences exactly as decode_native / decode_native_lb; qualities under the quality rule of `_check_qualities` with
    delta = dq*/d(ln p) * eta(T) (`decode_eta`).  The output rows of the batch are written, nothing around them."""
    from _oracle_v40_v3 import decode_native_lb
    n, qscale, qbias = 3, 1.05, 0.2
    S = 4 ** k
    g = torch.Generator().manual_seed(k * 1000 + T + lb)
    scores = (torch.randn(n, T, (5 if lb else 4) * S, generator=g) * 1.7).clamp(-5, 5).half()
    ws = torch.empty(native.crf_decode_workspace_bytes(n, T, k), dtype=torch.uint8, device="cuda")
    bufs = [torch.full((64 + n * T + 64,), CANARY8, dtype=torch.uint8, device="cuda") for _ in range(3)]
    outs = [b[64:64 + n * T] for b in bufs]
    if lb:
        native.crf_decode_lb(scores.cuda(), k, qscale, qbias, ws, *outs)
        o_moves, o_seq, _, mass = decode_native_lb(scores.float().numpy(), k, qscale, qbias)
    else:
        native.crf_decode(scores.cuda(), k, 2.0, qscale, qbias, ws, *outs)
        o_moves, o_seq, _, mass = O.decode_native(scores.float().numpy(), k, 2.0, qscale, qbias)
    torch.cuda.synchronize()
    host = [b.cpu().numpy() for b in bufs]
    for h in host:
        assert (h[:64] == CANARY8).all() and (h[64 + n * T:] == CANARY8).all()
    moves, seq, qual = (h[64:64 + n * T].reshape(n, T) for h in host)
    assert np.array_equal(moves, o_moves)
    assert np.array_equal(seq, o_seq)
    worst = _check_qualities(qual, moves, seq, mass, T, qscale, qbias)
    print(f"decode k={k} T={T} {'lb' if lb else 'fixed'}: worst implied relative error of p {worst:.3e} "
          f"(eta {decode_eta(T):.3e})")
