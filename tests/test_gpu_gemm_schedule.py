"""
The wgmma GEMM's schedule at the sizes the workloads run: a CTA owns a 128-row block and streams a run of 128-column tiles
through one 3-stage TMA / mbarrier ring, so the ring wraps inside a tile and across tile boundaries, and the column tiles
are split into runs (blockIdx.y) when the row blocks alone would leave too few CTAs.  The tests of test_gpu_kernel_edges.py
use M <= 910, where every CTA does a single column tile; these use 76k-136k rows, where (on a 132-SM H100) a CTA sweeps
all the column tiles of its row block, or runs of 2 of 3 tiles.

Each case is checked against a float64 reference on ~900 rows (the first, middle and last row blocks), within the
interval bound of test_gpu_kernel_edges.py (see its docstring); every element of the output map must be written and
nothing around it; and the output must be bit-identical for every `max_ctas`.  The kernel is not persistent and accepts
`max_ctas` only for the ABI, so those three launches share one grid: that comparison pins the ABI contract (the argument
never changes a result), not the schedule.  The schedule itself varies with M (the column-tile split), and
`test_column_split_does_not_change_rows` compares the same rows computed under three different splits bit for bit.
"""
import numpy as np
import pytest
import torch

from _edges import CANARY16, E_SFU, _swish, act_interval, pre16, rn16

pytestmark = pytest.mark.gpu

MAX_CTAS = (0, 1, 7)


@pytest.fixture(scope="module")
def native():
    from bonito_b200 import native as nat
    nat.require()
    return nat


def _dest_rows(m, rows_inner, valid_inner, stride_inner, stride_outer, group, stride_group, dev):
    r = torch.arange(m, device=dev, dtype=torch.int64)
    outer, inner = r // rows_inner, r % rows_inner
    if group > 0:
        row = inner * stride_inner + (outer % group) * stride_outer + (outer // group) * stride_group
    else:
        row = inner * stride_inner + outer * stride_outer
    return torch.where(inner < valid_inner, row, torch.full_like(row, -1))


def _check_rows(m):
    """Reference rows: the first, a window around the middle and the last row blocks (row-block edges included)."""
    mid = (m // 2) // 128 * 128
    return np.unique(np.concatenate([np.arange(0, min(m, 300)), np.arange(max(0, mid - 150), min(m, mid + 150)),
                                     np.arange(max(0, m - 300), m)]))


def _case(native, m, n, k, lda=None, act=0, lo=0.0, hi=0.0, bias=True, i8=False, rows_inner=None, valid_inner=None,
          stride_inner=1, stride_outer=0, group=0, stride_group=0, cb_width=0, cb_rows=0, seed=0):
    dev = torch.device("cuda")
    lda = lda or k
    g = torch.Generator().manual_seed(seed)
    a_len = (m - 1) * lda + k
    if i8:
        a = torch.randint(-127, 128, (a_len,), generator=g, dtype=torch.int8)
        w = torch.randint(-127, 128, (n, k), generator=g, dtype=torch.int8)
        scale = ((torch.rand(n, generator=g) + 0.5) / (k ** 0.5 * 4000.0)).float()
    else:
        a = torch.randn(a_len, generator=g).half()
        w = (torch.randn(n, k, generator=g) / k ** 0.5).half()
        scale = None
    bv = (torch.randn(n, generator=g) * 0.5).half() if bias else None
    swiglu = act == native.ACT_SWIGLU
    n_out = n // 2 if swiglu else n
    ldc = cb_width or n_out
    ri = rows_inner or m
    vi = ri if valid_inner is None else valid_inner

    row = _dest_rows(m, ri, vi, stride_inner, stride_outer, group, stride_group, dev)
    col = torch.arange(n_out, device=dev, dtype=torch.int64)
    if cb_width:
        dest = (row[:, None] + (col // cb_width)[None, :] * cb_rows) * ldc + (col % cb_width)[None, :]
    else:
        dest = row[:, None] * ldc + col[None, :]
    keep = row >= 0
    front = 2 * ldc + 8
    size = front + int(dest[keep].max()) + 1 + 2 * ldc + 8
    ad, wd = a.to(dev), w.to(dev)
    bd = None if bv is None else bv.to(dev)

    outs = []
    for mc in MAX_CTAS:
        buf = torch.full((size,), CANARY16, dtype=torch.int16, device=dev).view(torch.float16)
        kw = dict(act=act, lo=lo, hi=hi, rows_inner=ri, valid_inner=vi, stride_inner=stride_inner, stride_outer=stride_outer,
                  group=group, stride_group=stride_group, cb_width=cb_width, cb_rows=cb_rows, max_ctas=mc)
        if i8:
            native.gemm_i8(ad, lda, wd, scale.to(dev), bd, buf[front:], ldc, m, n, k, **kw)
        else:
            native.gemm(ad, lda, wd, bd, buf[front:], ldc, m, n, k, **kw)
        torch.cuda.synchronize()
        outs.append(buf.view(torch.int16))
    for mc, o in zip(MAX_CTAS[1:], outs[1:]):
        assert torch.equal(outs[0], o), f"max_ctas={mc} changed the result"

    # every mapped element written, nothing else
    bits = outs[0]
    mask = torch.zeros(size, dtype=torch.bool, device=dev)
    mask[dest[keep].reshape(-1) + front] = True
    assert bool((bits[mask] != CANARY16).all()), f"{int((bits[mask] == CANARY16).sum())} mapped elements not written"
    assert bool((bits[~mask] == CANARY16).all()), f"{int((bits[~mask] != CANARY16).sum())} elements outside the map written"

    rows = _check_rows(m)
    rows = rows[keep.cpu().numpy()[rows]]
    a_rows = np.stack([a[r * lda:r * lda + k].double().numpy() for r in rows])
    w64 = w.double().numpy()
    if i8:
        acc = a_rows @ w64.T
        v = acc * scale.double().numpy() + bv.double().numpy()
        p_lo, p_hi = pre16(v, 2.0 ** -24 * np.abs(v))
    else:
        v = a_rows @ w64.T + (bv.double().numpy() if bias else 0.0)
        p_lo, p_hi = pre16(v, k * 2.0 ** -23 * (np.abs(a_rows) @ np.abs(w64).T) + 2.0 ** -24 * np.abs(v))
    if swiglu:
        G, mm = n // 64, len(rows)
        yl, yh = (x.reshape(mm, G, 2, 32)[:, :, 0].reshape(mm, n_out) for x in (p_lo, p_hi))
        gl, gh = (x.reshape(mm, G, 2, 32)[:, :, 1].reshape(mm, n_out) for x in (p_lo, p_hi))
        cands = [yy * _swish(gg) for yy in (yl, yh) for gg in (gl, gh)]
        s_lo, s_hi = np.minimum.reduce(cands), np.maximum.reduce(cands)
        e = E_SFU * (1 + np.abs(s_hi)) * (1 + np.maximum(np.abs(yl), np.abs(yh)))
        out_lo, out_hi = rn16(s_lo - e), rn16(s_hi + e)
    else:
        out_lo, out_hi = act_interval(p_lo, p_hi, act, lo, hi)
    idx = dest[torch.as_tensor(rows, device=dev)] + front
    got = bits.view(torch.float16)[idx].double().cpu().numpy()
    bad = ~((got >= out_lo) & (got <= out_hi))
    assert not bad.any(), f"{int(bad.sum())}/{bad.size} outside their interval; first: got {got[bad][0]!r}, " \
                          f"allowed [{out_lo[bad][0]!r}, {out_hi[bad][0]!r}]"


def test_sweep_all_column_tiles(native):
    """1057 row blocks (partial last): every CTA sweeps 3 column tiles (partial third), 4 K stages (partial fourth) through
    the 3-stage ring, so the ring wraps inside and across tiles."""
    _case(native, 1056 * 128 + 37, 264, 200, seed=1)


def test_column_runs_do_not_divide_the_tiles(native):
    """601 row blocks: 3 column tiles split into runs of 2 and 1 over blockIdx.y; TANH epilogue."""
    _case(native, 600 * 128 + 37, 264, 200, act=native.ACT_TANH, seed=2)


def test_column_blocks_cross_tile_boundaries(native):
    """The LSTM input projection's map on 1057 row blocks: 192-column blocks (cb_width) across 128-column tiles, rows
    (chunk group, chunk) -> [group][block][chunk]."""
    _case(native, 1056 * 128 + 37, 768, 72, rows_inner=64, valid_inner=64, stride_inner=1, stride_outer=4 * 64,
          cb_width=192, cb_rows=64, seed=3)


def test_swiglu_sweep(native):
    """The fused SwiGLU epilogue with a CTA sweeping 2 column tiles."""
    _case(native, 1056 * 128 + 37, 256, 72, act=native.ACT_SWIGLU, bias=False, seed=4)


def test_overlapping_rows_sweep(native):
    """The strided-convolution GEMM (A rows 96 elements apart, K = 304) with the group map of the tile layout, 1060 row
    blocks, 3 column tiles per CTA."""
    _case(native, 13 * 64 * 163, 384, 304, lda=96, act=native.ACT_TANH, rows_inner=13, valid_inner=11, stride_inner=64,
          stride_outer=1, group=64, stride_group=11 * 64, seed=5)


def test_int8_sweep(native):
    """int8 operands, 400-byte K (4 stages, partial fourth), CLAMP, a CTA sweeping 3 column tiles."""
    _case(native, 1056 * 128 + 37, 264, 400, act=native.ACT_CLAMP, lo=-1.0, hi=1.5, i8=True, seed=6)


def test_column_split_does_not_change_rows(native):
    """The same A and B under three grids: M of 1057, 601 and 300 row blocks gives (on a 132-SM H100) runs of 3, of 2 + 1
    and of 1 column tile per CTA over N = 264 (3 tiles, the last partial), K = 200 (4 stages through the 3-stage ring).  A
    row's result does not depend on the grid, so the rows the three problems share must be bit-identical."""
    dev = torch.device("cuda")
    n, k = 264, 200
    ms = (1056 * 128 + 37, 600 * 128 + 37, 300 * 128)
    g = torch.Generator().manual_seed(8)
    a = torch.randn(ms[0], k, generator=g).half().to(dev)
    w = (torch.randn(n, k, generator=g) / k ** 0.5).half().to(dev)
    bv = (torch.randn(n, generator=g) * 0.5).half().to(dev)
    outs = []
    for m in ms:
        c = torch.full((m, n), CANARY16, dtype=torch.int16, device=dev).view(torch.float16)
        native.gemm(a, k, w, bv, c, n, m, n, k, act=native.ACT_TANH)
        torch.cuda.synchronize()
        assert bool((c.view(torch.int16) != CANARY16).all()), f"M={m}: elements not written"
        outs.append(c.view(torch.int16))
    for m, o in zip(ms[1:], outs[1:]):
        assert torch.equal(outs[0][:m], o), f"M={m}: rows differ from the M={ms[0]} problem"
