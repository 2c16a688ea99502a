"""
Shared pieces of the edge tests (test_gpu_kernel_edges.py, test_gpu_attention_edges.py, test_gpu_lstm_wide_edges.py,
test_gpu_stem_edges.py):
canary-filled output buffers, the fp16 interval checks, the interval of every epilogue activation, the GEMM epilogue's
output map and the float64 LSTM recurrence with its carried error bound.

Every output buffer is allocated with margins around the region a call may write and filled with a canary bit pattern
(fp16: the NaN 0x7E5A, which no kernel produces; bytes: 0xA5).  After the call, every element the documented map addresses
must have been written, every other element must still hold the canary (`check_guarded`), and every written value must lie
inside the per-element interval its arithmetic allows (`check_between`).
"""
import numpy as np
import torch

CANARY16 = 0x7E5A            # an fp16 NaN payload the kernels never produce
CANARY8 = 0xA5
CANARY32 = 0x7FA5A5A5        # an fp32 NaN payload
E_SFU = 2.0 ** -19           # abs error bound of sigmoid / tanh / swish from ex2.approx + rcp.approx (each <= 2^-21 rel)


def rn16(x):
    """Round to nearest fp16 (numpy rounds float64 -> float16 directly, ties to even), back to float64."""
    return np.asarray(x, dtype=np.float64).astype(np.float16).astype(np.float64)


def canary16(n):
    return torch.full((n,), CANARY16, dtype=torch.int16, device="cuda").view(torch.float16)


def bits16(t):
    return t.view(torch.int16).cpu().numpy().astype(np.int64) & 0xFFFF


def check_guarded(buf_bits, idx, canary):
    """Every flat index in `idx` was written; every other element of the buffer still holds the canary."""
    mask = np.zeros(buf_bits.size, dtype=bool)
    mask[np.asarray(idx).ravel()] = True
    assert (buf_bits.ravel()[mask] != canary).all(), f"{int((buf_bits.ravel()[mask] == canary).sum())} elements not written"
    stray = np.flatnonzero(buf_bits.ravel()[~mask] != canary)
    assert stray.size == 0, f"{stray.size} elements outside the output map were written (first flat index " \
                            f"{np.flatnonzero(~mask)[stray[0]]})"


def check_between(got, lo, hi, what):
    got, lo, hi = (np.asarray(a, dtype=np.float64) for a in (got, lo, hi))
    bad = ~((got >= lo) & (got <= hi))
    if bad.any():
        i = np.flatnonzero(bad.ravel())[0]
        raise AssertionError(f"{what}: {int(bad.sum())}/{bad.size} outside their interval; first at flat {i}: "
                             f"got {got.ravel()[i]!r}, allowed [{lo.ravel()[i]!r}, {hi.ravel()[i]!r}]")


def fp16_values_admitted(lo, hi):
    """Number of fp16 values in [lo, hi] per element (lo, hi themselves fp16 values): the width of an interval."""
    def key(x):
        b = np.asarray(x, dtype=np.float64).astype(np.float16).view(np.int16).astype(np.int64)
        return np.where(b < 0, -(b & 0x7FFF), b)            # monotone in the value; -0 and +0 share 0
    return key(hi) - key(lo) + 1


def pre16(v, g):
    """The fp16 values a kernel may hold for an fp32 value within g of v: rn16(v - g) and rn16(v + g) (equal unless v is
    within g of a rounding midpoint)."""
    return rn16(v - g), rn16(v + g)


def _sigmoid(x):
    return 0.5 * (1.0 + np.tanh(0.5 * x))


def _swish(x):
    return x * _sigmoid(x)


SWISH_ARGMIN = -1.278464542761074            # swish's only stationary point: 1 + x (1 - sigmoid(x)) = 0


def act_interval(p_lo, p_hi, act, lo, hi):
    """Interval of apply_act_f16's result when its fp16-rounded input is any fp16 value in [p_lo, p_hi].  Every activation
    but swish is monotone, so its ends are those of the end points; swish falls to its minimum at SWISH_ARGMIN, which is
    taken in wherever the interval straddles it."""
    p_lo, p_hi = np.asarray(p_lo, dtype=np.float64), np.asarray(p_hi, dtype=np.float64)
    out_lo, out_hi = None, None
    for p in (p_lo, p_hi):
        if act == 0:                                 # NONE
            a, b = p, p
        elif act in (1, 7):                          # SWISH, SWISH_CLAMP
            s = _swish(p)
            a, b = rn16(s - E_SFU * (1 + np.abs(p))), rn16(s + E_SFU * (1 + np.abs(p)))
        elif act == 2:                               # TANH
            t = np.tanh(p)
            a, b = rn16(t - E_SFU), rn16(t + E_SFU)
        elif act == 3:                               # CLAMP
            a = b = np.clip(p, lo, hi)
        elif act == 4:                               # SCALE: one fp32 multiply, then fp16
            s = p * np.float32(lo)
            a, b = rn16(s - 2.0 ** -24 * np.abs(s)), rn16(s + 2.0 ** -24 * np.abs(s))
        elif act == 6:                               # TANH_SCALE: fp16(fp16(tanh) * lo)
            t = np.tanh(p)
            m_lo, m_hi = rn16(t - E_SFU), rn16(t + E_SFU)
            s1, s2 = m_lo * np.float32(lo), m_hi * np.float32(lo)
            s_lo, s_hi = np.minimum(s1, s2), np.maximum(s1, s2)
            a, b = rn16(s_lo - 2.0 ** -24 * np.abs(s_lo)), rn16(s_hi + 2.0 ** -24 * np.abs(s_hi))
        elif act == 8:                               # RELU
            a = b = np.maximum(p, 0.0)
        else:
            raise ValueError(act)
        out_lo = a if out_lo is None else np.minimum(out_lo, a)
        out_hi = b if out_hi is None else np.maximum(out_hi, b)
    if act in (1, 7):
        s_min = rn16(_swish(SWISH_ARGMIN) - E_SFU * (1 - SWISH_ARGMIN))
        out_lo = np.where((p_lo < SWISH_ARGMIN) & (p_hi > SWISH_ARGMIN), np.minimum(out_lo, s_min), out_lo)
        if act == 7:
            out_lo, out_hi = np.clip(out_lo, lo, hi), np.clip(out_hi, lo, hi)
    return out_lo, out_hi


def gemm_rows(m, rows_inner, valid_inner, stride_inner, stride_outer, group, stride_group):
    """Output row of every input row under the GEMM epilogue's row map (b200_gemm_fwd_ex), -1 for dropped rows."""
    r = np.arange(m)
    outer, inner = r // rows_inner, r % rows_inner
    if group > 0:
        row = inner * stride_inner + (outer % group) * stride_outer + (outer // group) * stride_group
    else:
        row = inner * stride_inner + outer * stride_outer
    return np.where(inner < valid_inner, row, -1)


def gemm_dest(m, n, rows_inner, valid_inner, stride_inner, stride_outer, group, stride_group, cb_width, cb_rows, ldc):
    """Flat output index (relative to c) of every (input row, column) the documented map writes, -1 for dropped rows."""
    row = gemm_rows(m, rows_inner, valid_inner, stride_inner, stride_outer, group, stride_group)
    col = np.arange(n)
    if cb_width > 0:
        rows = row[:, None] + (col // cb_width)[None, :] * cb_rows
        cols = np.broadcast_to(col % cb_width, (m, n))
    else:
        rows, cols = np.broadcast_to(row[:, None], (m, n)), np.broadcast_to(col, (m, n))
    dest = rows * ldc + cols
    return np.where((row >= 0)[:, None], dest, -1)


# ------------------------------------------------------------------------------------------------ LSTM recurrences
def _lstm_inputs(t, n, H, seed):
    """gx [T, n, 4, H] (natural gate order i, f, g, o) and W_hh [4H, H]; W_hh has row sums of |w| near 1.2 so the error
    bound contracts from step to step instead of compounding."""
    g = torch.Generator().manual_seed(seed)
    gx = (torch.randn(t, n, 4, H, generator=g) * 0.8).half()
    whh = (torch.randn(4 * H, H, generator=g) * 1.5 / H).half()
    return gx, whh


def _perm_hh(H):
    return (torch.arange(H // 8)[:, None, None] * 8 + torch.arange(4)[None, :, None] * H
            + torch.arange(8)[None, None, :]).reshape(-1)


def _lstm_reference(gx, whh, reverse):
    """float64 recurrence with the kernels' rounding points (gx and h_{t-1} are fp16, c stays fp32) and a per-element
    bound on |h_kernel - h| carried through it.  Returns lo, hi of the fp16 output [T, n, H]."""
    gx64, w = gx.double().numpy(), whh.double().numpy()
    T, n, _, H = gx64.shape
    aw = np.abs(w)
    h16 = np.zeros((n, H))
    eh = np.zeros((n, H))                      # bound on |h_kernel(fp16) - h16|
    c = np.zeros((n, H))
    ec = np.zeros((n, H))
    lo = np.empty((T, n, H))
    hi = np.empty((T, n, H))
    steps = range(T - 1, -1, -1) if reverse else range(T)
    for t in steps:
        G = gx64[t].reshape(n, 4 * H) + h16 @ w.T
        eG = eh @ aw.T + H * 2.0 ** -23 * (np.abs(h16) @ aw.T) + 2.0 ** -24 * np.abs(G)
        gi, gf, gg, go = (G[:, q * H:(q + 1) * H] for q in range(4))
        ei, ef, eg, eo = (eG[:, q * H:(q + 1) * H] for q in range(4))
        si, sf, tg, so = _sigmoid(gi), _sigmoid(gf), np.tanh(gg), _sigmoid(go)
        c_new = sf * c + si * tg
        ec = 0.25 * ef * np.abs(c) + sf * ec + 0.25 * ei * np.abs(tg) + si * eg + E_SFU * (1 + np.abs(c_new))
        c = c_new
        h = so * np.tanh(c)
        ehu = (0.25 * eo * np.abs(np.tanh(c)) + so * ec + E_SFU) * (1 + 2.0 ** -8)
        lo[t], hi[t] = rn16(h - ehu), rn16(h + ehu)
        h16 = rn16(h)
        eh = np.maximum(hi[t] - h16, h16 - lo[t])
    return lo, hi
