"""
The wgmma GEMM's epilogue stores: each consumer warp passes its rounded fp16 results through a shared-memory buffer of
16 rows x 32 columns and writes them back as 16-byte row segments.  These cases put the edges of that staging where the
workloads' shapes do not: rows dropped by `valid_inner` in the middle of a warp's 16 rows, column blocks narrower than a
128-column tile and not a multiple of 64 columns, N not a multiple of 32, and SwiGLU whose last 128-column tile holds a
single 64-column group.

Each case runs at 1057 row blocks, where a CTA sweeps a run of two column tiles, and is checked there as in
test_gpu_gemm_schedule.py: float64 reference on the first, middle and last row blocks, every mapped element written and
nothing around it.  The same A and B then run at 300 row blocks, where every CTA does a single column tile (on a 132-SM
H100), and the rows both problems share must be bit-identical.
"""
import pytest
import torch

from _edges import CANARY16
from test_gpu_gemm_schedule import _case, _dest_rows

pytestmark = pytest.mark.gpu

M_SWEEP, M_SPLIT = 1056 * 128 + 37, 300 * 128


@pytest.fixture(scope="module")
def native():
    from bonito_b200 import native as nat
    nat.require()
    return nat


def _split_check(native, n, k, act=0, lo=0.0, hi=0.0, bias=True, i8=False, rows_inner=None, valid_inner=None,
                 stride_inner=1, stride_outer=0, group=0, stride_group=0, cb_width=0, cb_rows=0, seed=0):
    """The M_SWEEP and M_SPLIT problems on the same A and B: the output positions of the first M_SPLIT rows agree bit for
    bit, and the smaller problem writes nothing else."""
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(100 + seed)
    if i8:
        a = torch.randint(-127, 128, (M_SWEEP, k), generator=g, dtype=torch.int8).to(dev)
        w = torch.randint(-127, 128, (n, k), generator=g, dtype=torch.int8).to(dev)
        scale = ((torch.rand(n, generator=g) + 0.5) / (k ** 0.5 * 4000.0)).float().to(dev)
    else:
        a = torch.randn(M_SWEEP, k, generator=g).half().to(dev)
        w = (torch.randn(n, k, generator=g) / k ** 0.5).half().to(dev)
    bv = (torch.randn(n, generator=g) * 0.5).half().to(dev) if bias else None
    n_out = n // 2 if act == native.ACT_SWIGLU else n
    ldc = cb_width or n_out
    col = torch.arange(n_out, device=dev, dtype=torch.int64)
    dests = []
    for m in (M_SWEEP, M_SPLIT):
        ri = rows_inner or m
        vi = ri if valid_inner is None else valid_inner
        row = _dest_rows(m, ri, vi, stride_inner, stride_outer, group, stride_group, dev)
        if cb_width:
            dest = (row[:, None] + (col // cb_width)[None, :] * cb_rows) * ldc + (col % cb_width)[None, :]
        else:
            dest = row[:, None] * ldc + col[None, :]
        dests.append(dest[row >= 0].reshape(-1))
    size = int(dests[0].max()) + 1
    outs = []
    for m in (M_SWEEP, M_SPLIT):
        c = torch.full((size,), CANARY16, dtype=torch.int16, device=dev).view(torch.float16)
        ri = rows_inner or m
        vi = ri if valid_inner is None else valid_inner
        kw = dict(act=act, lo=lo, hi=hi, rows_inner=ri, valid_inner=vi, stride_inner=stride_inner,
                  stride_outer=stride_outer, group=group, stride_group=stride_group, cb_width=cb_width, cb_rows=cb_rows)
        if i8:
            native.gemm_i8(a, k, w, scale, bv, c, ldc, m, n, k, **kw)
        else:
            native.gemm(a, k, w, bv, c, ldc, m, n, k, **kw)
        torch.cuda.synchronize()
        outs.append(c.view(torch.int16))
    shared = dests[1]
    assert torch.equal(outs[0][shared], outs[1][shared]), "rows differ between the two column splits"
    mask = torch.zeros(size, dtype=torch.bool, device=dev)
    mask[shared] = True
    assert bool((outs[1][~mask] == CANARY16).all()), "the smaller problem wrote outside its map"


# (kwargs; act by name): every case runs through the float64 check at M_SWEEP and the column-split comparison
CASES = [
    # rows (chunk, frame) with 24 rows per chunk, the last 5 dropped: the dropped rows 19-23 sit in the middle of the
    # second warp's rows 16-31; N = 200 ends 8 columns into the third 32-column block of the second tile
    pytest.param(dict(n=200, k=72, act="ACT_TANH", rows_inner=24, valid_inner=19, stride_inner=64, stride_outer=1, group=64,
                      stride_group=19 * 64), id="valid_inner-mid-warp-N=200"),
    # 96-column blocks: block boundaries at column 96 of the first tile and 64 of the second
    pytest.param(dict(n=288, k=72, rows_inner=64, valid_inner=64, stride_inner=1, stride_outer=3 * 64, cb_width=96,
                      cb_rows=64), id="cb_width=96-N=288"),
    # 192-column blocks as in the hac input projection, N = 416 (13 blocks of 32, the last tile 32 columns wide)
    pytest.param(dict(n=416, k=72, act="ACT_CLAMP", lo=-1.0, hi=1.5, rows_inner=37, valid_inner=29, stride_inner=1,
                      stride_outer=29, cb_width=192, cb_rows=M_SWEEP), id="cb_width=192-N=416-valid_inner"),
    # N = 216: the last tile is 88 columns wide, its third 32-column block holds 24
    pytest.param(dict(n=216, k=136), id="N=216"),
    # SwiGLU with N = 320: the last 128-column tile is a single 64-column group
    pytest.param(dict(n=320, k=72, act="ACT_SWIGLU", bias=False), id="swiglu-N=320-partial-last-tile"),
    # int8 with dropped rows and 96-column blocks
    pytest.param(dict(n=232, k=144, act="ACT_CLAMP", lo=-1.0, hi=1.5, i8=True, rows_inner=24, valid_inner=19, stride_inner=1,
                      stride_outer=19, cb_width=96, cb_rows=M_SWEEP), id="int8-valid_inner-cb_width=96-N=232"),
]


@pytest.mark.parametrize("kw", CASES)
def test_staged_store_edges(native, kw):
    kw = dict(kw)
    if "act" in kw:
        kw["act"] = getattr(native, kw["act"])
    _case(native, M_SWEEP, seed=11, **kw)
    _split_check(native, seed=11, **kw)
