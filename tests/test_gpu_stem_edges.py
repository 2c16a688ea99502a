"""
The input side of every LSTM-CRF basecall at its tile, halo and buffer edges, against float64 references: the fused conv
stem (conv_stem.cu, both kernels), the strided conv3 as one GEMM over the overlapping rows of the stem buffer (engine.py
`_conv_gemm`, encoder_fwd.cu), the engine's front end end to end, and the int8 quantiser of --quantize (quantize.cu).

As in test_gpu_kernel_edges.py, every output buffer has canary margins, every element the call may write must be written
and nothing else, and every written value must lie in a per-element interval derived from the arithmetic:

* conv1 (fmaf chain from the bias): v1 = b1 + sum w1 x in float64, |v1_kernel - v1| <= (K1 + 1) 2^-24 (|b1| + sum|w1 x|),
  so the kernel holds a1 in act_interval(rn16(v1 -/+ g1), act1); conv1 outside [0, L) is exactly 0 (conv2's 'same'
  padding).
* conv2 carries a1's interval: v2 in b2 + sum w2 [a1_lo, a1_hi] = mid +- sum|w2| halfwidth, widened by the fp32
  accumulation bound of the GEMM edge tests (C1 K2 + 1) 2^-23 (|b2| + sum|w2| max|a1|) (an fmaf chain or mma.sync, whose
  adds may truncate), rounded to [rn16(v2_lo), rn16(v2_hi)], then act2 over that whole interval.  Rows [0, padl) and
  [padl + L, lp) are exactly 0.
* the conv3 GEMM takes the stem's fp16 values as exact inputs: rn16(v -/+ K 2^-23 sum|a w| + 2^-24 |v|), then act3.
* quantize_i8 is exact: clamp(rint_even(x * scale), -127, 127).

Most stem outputs admit one fp16 value and a few two; every stem test asserts a median of at most 2 admitted values
(`fp16_values_admitted`) so that the bound cannot silently become vacuous, and every conv3 test a median of at most 8
(see `_check_gemm_width`); each prints its largest.  The largest widths, thousands of values, belong to outputs within
~1e-3 of zero, where an absolute error of that size spans the densely spaced small fp16 values.
"""
import numpy as np
import pytest
import torch

from _edges import (CANARY8, CANARY16, act_interval, bits16, canary16, check_between, check_guarded, fp16_values_admitted,
                    gemm_rows, pre16, rn16)
from oracle import synth

pytestmark = pytest.mark.gpu

NONE, SWISH, TANH, SWISH_CLAMP = 0, 1, 2, 7        # B200_ACT_*: what engine._conv_act can return for a convolution
V40 = (-0.5, 3.5)                                   # dna_r10.4.1@v4.0's Clamp behind every convolution
TL = 256                                            # stem output positions per CTA (conv_stem.cu)
K3, PAD3 = 19, 9                                    # conv3 of every LSTM-CRF config: k19, padding 9, stride 6 or 5


@pytest.fixture(scope="module")
def native():
    from bonito_b200 import native as nat
    nat.require()
    return nat


def engine_geometry(L, k3, s3, pad3):
    """(T, Tp, Lp, need) of LstmCrfPlan._buffers: T frames, the stem buffer holds Tp * s3 rows per chunk."""
    T = (L + 2 * pad3 - k3) // s3 + 1
    need = max(pad3 + L, (T - 1) * s3 + k3)
    Tp = -(-need // s3)
    return T, Tp, Tp * s3, need


# ------------------------------------------------------------------------------------------------ conv stem
def stem_reference(x, w1, b1, act1, w2, b2, act2, lp, padl, bounds=None):
    """lo, hi [N, lp, C2] of the fused stem's fp16 output (see the module docstring); inputs are float64 arrays."""
    lo1, hi1, lo2, hi2 = bounds or (0.0, 0.0, 0.0, 0.0)
    n, L = x.shape
    c1, _, k1 = w1.shape
    c2, _, k2 = w2.shape
    p1, p2 = k1 // 2, k2 // 2
    b1 = np.zeros(c1) if b1 is None else b1
    b2 = np.zeros(c2) if b2 is None else b2
    xp = np.zeros((n, L + 2 * p1))
    xp[:, p1:p1 + L] = x
    win = np.stack([xp[:, j:j + L] for j in range(k1)], axis=-1)               # [N, L, K1]
    w1m = w1[:, 0, :].T                                                         # [K1, C1]
    v1 = win @ w1m + b1
    g1 = (k1 + 1) * 2.0 ** -24 * (np.abs(win) @ np.abs(w1m) + np.abs(b1))
    a_lo, a_hi = act_interval(*pre16(v1, g1), act1, lo1, hi1)                   # [N, L, C1]
    A_lo, A_hi = np.zeros((n, L + 2 * p2, c1)), np.zeros((n, L + 2 * p2, c1))   # exact zeros outside [0, L)
    A_lo[:, p2:p2 + L], A_hi[:, p2:p2 + L] = a_lo, a_hi

    def conv2(a, w):                                                            # [N, L + 2 p2, C1] -> [N, L, C2]
        return sum(a[:, j:j + L] @ w[:, :, j].T for j in range(k2))

    v2 = conv2((A_lo + A_hi) / 2, w2) + b2
    spread = conv2((A_hi - A_lo) / 2, np.abs(w2))
    g2 = (c1 * k2 + 1) * 2.0 ** -23 * (conv2(np.maximum(np.abs(A_lo), np.abs(A_hi)), np.abs(w2)) + np.abs(b2))
    o_lo, o_hi = act_interval(rn16(v2 - spread - g2), rn16(v2 + spread + g2), act2, lo2, hi2)
    lo, hi = np.zeros((n, lp, c2)), np.zeros((n, lp, c2))
    lo[:, padl:padl + L], hi[:, padl:padl + L] = o_lo, o_hi
    return lo, hi


def _stem_weights(c1, seed, bias=True):
    """Stem weights of the synth models' scale (conv gain 2.5), with larger biases so that a conv1 value act1(b1) where 0
    belongs moves conv2 by far more than its bound."""
    g = torch.Generator().manual_seed(seed)
    w1 = (torch.randn(c1, 1, 5, generator=g) * 2.5 / 5 ** 0.5).half()
    b1 = (torch.randn(c1, generator=g) * 0.5).half()
    w2 = (torch.randn(16, c1, 5, generator=g) * 2.5 / (5 * c1) ** 0.5).half()
    b2 = (torch.randn(16, generator=g) * 0.3).half()
    return (w1, b1 if bias else None, w2, b2 if bias else None)


def _signal(n, L, seed):
    """Squiggle chunks whose scales alternate between 1 and 10: a read across a chunk boundary lands far outside the
    interval."""
    scale = torch.where(torch.arange(n) % 2 == 1, 10.0, 1.0)[:, None]
    return (synth.squiggle(n, L, seed=seed)[:, 0] * scale).half()


def _set_impl(monkeypatch, impl):
    monkeypatch.setenv("B200_STEM_IMPL", "fma" if impl == "fma" else "tc")     # read on every launch


def _run_stem(native, x, weights, act1, act2, lp, padl, bounds=None):
    """One guarded stem call: x sits inside an fp16 buffer whose margins are NaN (a read before chunk 0 or after chunk
    N - 1 makes a NaN output); returns the output [N, lp, 16] after checking its canaries."""
    n, L = x.shape
    xbuf = torch.full((8 + n * L + 8,), float("nan"), dtype=torch.float16, device="cuda")
    xbuf[8:8 + n * L] = x.reshape(-1).cuda()
    w1, b1, w2, b2 = (None if t is None else t.cuda() for t in weights)
    front, size = 64, n * lp * 16
    buf = canary16(front + size + 64)
    native.conv_stem(xbuf[8:8 + n * L].view(n, L), w1, b1, act1, w2, b2, act2, buf[front:], lp, padl, bounds=bounds)
    torch.cuda.synchronize()
    check_guarded(bits16(buf), front + np.arange(size), CANARY16)
    return buf[front:front + size].double().cpu().numpy().reshape(n, lp, 16)


def _check_stem(got, x, weights, act1, act2, lp, padl, bounds, what):
    w1, b1, w2, b2 = (None if t is None else t.double().numpy() for t in weights)
    lo, hi = stem_reference(x.double().numpy(), w1, b1, act1, w2, b2, act2, lp, padl, bounds)
    check_between(got, lo, hi, what)
    L = x.shape[1]
    admitted = fp16_values_admitted(lo[:, padl:padl + L], hi[:, padl:padl + L])
    print(f"{what}: fp16 values admitted: median {np.median(admitted):.0f}, max {admitted.max()}")
    assert np.median(admitted) <= 2
    return lo, hi


STEM_KERNELS = [pytest.param("tc", 16, id="tc-16"), pytest.param("fma", 16, id="fma-16"),
                pytest.param("fma", 4, id="fma-4")]

# (n, L, lp, padl)
STEM_GEOMETRY = (
    [pytest.param(3, lp - 3, lp, 2, id=f"seam-lp={lp}") for lp in (255, 256, 257, 511, 513)]
    + [pytest.param(3, 700, padl + 705, padl, id=f"padl={padl}") for padl in (0, 2, 9, 255, 256, 300)]
    + [pytest.param(3, 300, 609, 9, id="trailing-zero-tile"),            # lp - padl - L = 300: the third tile is all zeros
       pytest.param(3, 245, 256, 9, id="signal-ends-at-tile-edge")]      # padl + L = 254: conv1 halo straddles the seam
    + [pytest.param(3, L, 9 + L + 4, 9, id=f"L={L}") for L in (1, 2, 3, 5)]
    + [pytest.param(2, 1, 1, 0, id="L=1-lp=1"), pytest.param(2, 2, 2, 0, id="L=2-lp=2")]
    + [pytest.param(n, 1000, 1020, 9, id=f"N={n}") for n in (1, 65)])


@pytest.mark.parametrize("n,L,lp,padl", STEM_GEOMETRY)
@pytest.mark.parametrize("impl,c1", STEM_KERNELS)
def test_stem_tiles_and_padding(native, monkeypatch, impl, c1, n, L, lp, padl):
    """The stem (swish, swish) across 256-position tile seams, with the whole first tile in the left padding, an all-zero
    trailing tile, signals shorter than the kernel (every conv1 window touches the padding) and 1 to 65 chunks of scales
    1 and 10."""
    _set_impl(monkeypatch, impl)
    weights = _stem_weights(c1, seed=n + L + lp + padl)
    x = _signal(n, L, seed=L + padl)
    got = _run_stem(native, x, weights, SWISH, SWISH, lp, padl)
    _check_stem(got, x, weights, SWISH, SWISH, lp, padl, None, f"stem {impl} c1={c1} n={n} L={L} lp={lp} padl={padl}")


# (act1, act2, bounds, bias)
STEM_ACTS = [pytest.param(SWISH, SWISH, None, True, id="swish"), pytest.param(TANH, TANH, None, True, id="tanh"),
             pytest.param(NONE, NONE, None, True, id="none"), pytest.param(TANH, SWISH, None, True, id="tanh-swish"),
             pytest.param(SWISH_CLAMP, SWISH_CLAMP, V40 + V40, True, id="swish-clamp-v4.0"),
             pytest.param(SWISH, SWISH, None, False, id="no-bias")]


@pytest.mark.parametrize("act1,act2,bounds,bias", STEM_ACTS)
@pytest.mark.parametrize("impl,c1", STEM_KERNELS)
def test_stem_activations(native, monkeypatch, impl, c1, act1, act2, bounds, bias):
    """Every activation the engine passes to the stem; swish-and-clamp with the v4.0 bounds (-0.5, 3.5), where the clamp
    binds on more than 3 % of the outputs; and no biases (a null pointer: the kernels read the bias as 0)."""
    _set_impl(monkeypatch, impl)
    n, L, lp, padl = 3, 1000, 1020, 9
    weights = _stem_weights(c1, seed=10 * act1 + act2, bias=bias)
    x = _signal(n, L, seed=act1 + act2)
    got = _run_stem(native, x, weights, act1, act2, lp, padl, bounds=bounds)
    lo, hi = _check_stem(got, x, weights, act1, act2, lp, padl, bounds, f"stem {impl} c1={c1} act={act1},{act2}")
    if bounds is not None:
        at_bound = ((lo == V40[1]) & (hi == V40[1]))[:, padl:padl + L].mean()
        assert at_bound > 0.03 and got.max() == V40[1], at_bound


@pytest.mark.parametrize("s3", [pytest.param(6, id="stride6-fast-hac"), pytest.param(5, id="stride5-sup_lstm-v4.0-v3")])
@pytest.mark.parametrize("L", [995, 1000, 1995, 3996])
@pytest.mark.parametrize("impl,c1", STEM_KERNELS)
def test_stem_engine_geometry(native, monkeypatch, impl, c1, L, s3):
    """The (L, padl, Lp) triples LstmCrfPlan derives for conv3 k19, padding 9, strides 6 and 5."""
    _set_impl(monkeypatch, impl)
    T, Tp, Lp, need = engine_geometry(L, K3, s3, PAD3)
    weights = _stem_weights(c1, seed=L + s3)
    x = _signal(2, L, seed=L)
    got = _run_stem(native, x, weights, SWISH, SWISH, Lp, PAD3)
    _check_stem(got, x, weights, SWISH, SWISH, Lp, PAD3, None, f"stem {impl} c1={c1} L={L} Lp={Lp}")


@pytest.mark.parametrize("impl", ["tc", "fma"])
def test_stem_65535_chunks(native, monkeypatch, impl):
    """The largest batch one launch takes (the chunk index is gridDim.y): 65535 chunks of one sample."""
    _set_impl(monkeypatch, impl)
    n, L, lp, padl = 65535, 1, 3, 1
    weights = _stem_weights(16, seed=65535)
    x = (torch.randn(n, L, generator=torch.Generator().manual_seed(1)) * 2).half()
    got = _run_stem(native, x, weights, SWISH, SWISH, lp, padl)
    _check_stem(got, x, weights, SWISH, SWISH, lp, padl, None, f"stem {impl} n=65535")


def test_more_than_65535_chunks_are_refused_before_a_launch(native):
    """Kernels with the chunk index in gridDim.y / z refuse N > 65535 with a message naming the limit; nothing is
    written."""
    z16 = torch.zeros(65536 * 8, dtype=torch.float16, device="cuda")
    x = z16[:65536].view(65536, 1)
    out = canary16(4096)
    w1, b1, w2, b2 = (t.cuda() for t in _stem_weights(16, seed=0))
    wf = torch.zeros(8, 1, 15, dtype=torch.float16, device="cuda")
    calls = {
        "conv_stem": lambda: native.conv_stem(x, w1, b1, SWISH, w2, b2, SWISH, out, 1, 0),
        "conv_first": lambda: native.conv_first(x, wf, None, SWISH, out, 1, 0),
        "conv_first_ex": lambda: native.conv_first_ex(x, wf, None, SWISH, out, 8, 1, 0),
        "depthwise": lambda: native.depthwise_conv(z16, 8, wf, out, 8, 65536, 1),
        "chunk_signal": lambda: native.chunk_signal(z16[:65537], 2, 1, out=out),       # 65536 windows of 2 samples
    }
    for name, call in calls.items():
        with pytest.raises(native.NativeError, match="65535"):
            call()
    torch.cuda.synchronize()
    assert (bits16(out) == CANARY16).all()


# ------------------------------------------------------------------------------------------------ strided conv3 GEMM
def _guard_rows(buf, front, span, ldc, rows):
    """check_guarded on the device, row by row (the large cases' buffers hold ~65M elements): the margins before `front` and
    after `front + span` keep the canary; of the span's rows of `ldc` elements, the `rows` the map addresses are written
    in full and every other row keeps the canary."""
    bits = buf.view(torch.int16)
    assert bool((bits[:front] == CANARY16).all()) and bool((bits[front + span:] == CANARY16).all()), "a margin was written"
    body = bits[front:front + span].view(-1, ldc)
    mask = torch.zeros(body.shape[0], dtype=torch.bool, device=body.device)
    mask[torch.as_tensor(rows, device=body.device)] = True
    written = (body != CANARY16).all(dim=1)
    untouched = (body == CANARY16).all(dim=1)
    assert bool(written[mask].all()), f"{int((~written[mask]).sum())} mapped rows not written in full"
    assert bool(untouched[~mask].all()), f"{int((~untouched[~mask]).sum())} rows outside the map written"


def _check_gemm_width(lo, hi, what):
    """The conv3 intervals admit 1 fp16 value at the median behind tanh and up to 4 behind swish, where the k3 * 16 terms
    of the windows over large stem values cancel and K 2^-23 sum|a w| spans a few fp16 values of the pre-activation; a
    median above 8 means the bound has at least doubled."""
    admitted = fp16_values_admitted(lo, hi)
    print(f"{what}: fp16 values admitted: median {np.median(admitted):.0f}, max {admitted.max()}")
    assert np.median(admitted) <= 8


def conv_gemm_reference(stem, N, T, Tp, s3, k3, w3, b3, act, lo, hi, chunks):
    """lo, hi [len(chunks), T, H] of the conv3 GEMM on the stem's fp16 values (float64, [N * Lp * 16 + tail] flat)."""
    c2 = 16
    lda, K = s3 * c2, k3 * c2
    rows = (np.asarray(chunks)[:, None] * Tp + np.arange(T)[None, :]).reshape(-1)
    a = np.stack([stem[r * lda:r * lda + K] for r in rows])
    w = w3.double().numpy()
    bias = 0.0 if b3 is None else b3.double().numpy()
    v = a @ w.T + bias
    p_lo, p_hi = pre16(v, K * 2.0 ** -23 * (np.abs(a) @ np.abs(w).T) + 2.0 ** -24 * np.abs(v))
    o_lo, o_hi = act_interval(p_lo, p_hi, act, lo, hi)
    return o_lo.reshape(len(chunks), T, -1), o_hi.reshape(len(chunks), T, -1)


# (H, N, L, s3, k3, pad3, act, lo, hi, layout)
CONV_CASES = (
    [pytest.param(384, 3, L, 6, K3, PAD3, TANH, 0.0, 0.0, "generic", id=f"hac-L={L}") for L in (995, 1000, 1995, 3996)]
    + [pytest.param(1024, 3, L, 5, K3, PAD3, SWISH_CLAMP, *V40, "generic", id=f"v4.0-L={L}") for L in (995, 1000, 1995)]
    + [pytest.param(768, 2, 3996, 5, K3, PAD3, SWISH, 0.0, 0.0, "generic", id="v3.1-L=3996"),
       pytest.param(96, 1, 200, 6, K3, PAD3, TANH, 0.0, 0.0, "generic", id="fast-one-partial-row-block"),
       pytest.param(384, 70, 1000, 6, K3, PAD3, TANH, 0.0, 0.0, "tile", id="hac-tile-layout-70-chunks"),
       # 203 x 669 rows = 1061 row blocks: every CTA sweeps all three column tiles (test_gpu_gemm_schedule.py)
       pytest.param(384, 203, 3996, 6, K3, PAD3, TANH, 0.0, 0.0, "tile", id="hac-tile-layout-sweep"),
       # geometries of other conv3 shapes: the last window ends exactly at row Lp - 1 (k3 a multiple of s3), and a small
       # padding where need = pad3 + L
       pytest.param(128, 3, 1002, 6, 18, 9, TANH, 0.0, 0.0, "generic", id="k18-s6-last-window-ends-at-Lp"),
       pytest.param(128, 3, 1000, 6, 8, 0, TANH, 0.0, 0.0, "generic", id="k8-s6-pad0-need=pad3+L")])


@pytest.mark.parametrize("H,N,L,s3,k3,pad3,act,lo,hi,layout", CONV_CASES)
@pytest.mark.parametrize("impl", ["wgmma", "mma"])
def test_conv_gemm_over_the_stem(native, monkeypatch, impl, H, N, L, s3, k3, pad3, act, lo, hi, layout):
    """conv3 as _conv_gemm launches it: A = the stem buffer (a real stem output) with lda = s3 * 16 and K = k3 * 16, so
    rows overlap; rows_inner = Tp, valid_inner = T; the k3 * 16 tail past N * Lp * 16 is NaN instead of zeros, so a valid
    output that reads it is NaN.  The generic layout's map (rows (n, t) -> [t][n]) or the tile layout's (-> [tile][t][64]);
    rows t >= T must not be written."""
    monkeypatch.delenv("B200_STEM_IMPL", raising=False)
    T, Tp, Lp, need = engine_geometry(L, k3, s3, pad3)
    if k3 % s3 == 0:
        assert (T - 1) * s3 + k3 == Lp, "the last valid window must end at row Lp - 1"
    if pad3 == 0:
        assert need == pad3 + L > (T - 1) * s3 + k3
    c2, K, tail = 16, k3 * 16, k3 * 16
    g = torch.Generator().manual_seed(H + N + L + s3 + k3)
    weights = [t.cuda() for t in _stem_weights(16, seed=L)]
    stem = torch.full((N * Lp * c2 + tail,), float("nan"), dtype=torch.float16, device="cuda")
    x = _signal(N, L, seed=N + L).cuda()
    bounds = V40 + V40 if act == SWISH_CLAMP else None
    stem_act = SWISH_CLAMP if bounds else SWISH
    native.conv_stem(x, weights[0], weights[1], stem_act, weights[2], weights[3], stem_act, stem, Lp, pad3, bounds=bounds)
    w3 = (torch.randn(H, K, generator=g) * 2.5 / K ** 0.5).half()
    b3 = (torch.randn(H, generator=g) * 0.1).half()
    if layout == "tile":
        TB = native.lstm_tile_chunks(H)                 # the engine's tile: [tile][t][TB chunks]
        rows = dict(stride_inner=TB, group=TB, stride_group=T * TB)
        span = -(-N // TB) * T * TB * H
    else:
        rows = dict(stride_inner=N)
        span = T * N * H
    m = N * Tp
    out_row = gemm_rows(m, Tp, T, rows["stride_inner"], 1, rows.get("group", 0), rows.get("stride_group", 0))
    front = 2 * H + 8
    buf = canary16(front + span + 2 * H + 8)
    native.gemm(stem, s3 * c2, w3.cuda(), b3.cuda(), buf[front:], H, m, H, K, act=act, lo=lo, hi=hi, rows_inner=Tp,
                valid_inner=T, stride_outer=1, impl=native.GEMM_TCGEN05 if impl == "wgmma" else native.GEMM_MMA_SYNC, **rows)
    torch.cuda.synchronize()
    _guard_rows(buf, front, span, H, out_row[out_row >= 0])
    chunks = sorted({0, 1, N // 2, N - 2, N - 1} & set(range(N)))
    s = stem.double().cpu().numpy()
    assert np.isfinite(s[:N * Lp * c2]).all()
    o_lo, o_hi = conv_gemm_reference(s, N, T, Tp, s3, k3, w3, b3, act, lo, hi, chunks)
    r = out_row.reshape(N, Tp)[chunks, :T]
    got = buf[front:front + span].view(-1, H)[torch.as_tensor(r, device="cuda")].double().cpu().numpy()
    what = f"conv GEMM {impl} H={H} N={N} L={L} s3={s3} k3={k3}"
    check_between(got, o_lo, o_hi, what)
    _check_gemm_width(o_lo, o_hi, what)


# ------------------------------------------------------------------------------------------------ engine front end
def _plan(spec):
    from bonito_b200.crf.model import Model
    weights = synth.make_weights(spec, seed=17)
    model = Model(synth.model_config(spec))
    model.load_state_dict(synth.state_dict_from_weights(spec, weights))
    model.use_koi(batchsize=8, chunksize=1000, quantize=False)
    return model.half().eval().to("cuda").native_plan("cuda")


ENGINE_SPECS = [pytest.param(lambda: synth.model_spec("fast", n_lstm=1), 3, 1000, id="fast-generic-layout"),
                pytest.param(lambda: synth.model_spec("hac", n_lstm=1), 3, 995, id="hac-tile-layout"),
                pytest.param(lambda: synth.v40_spec(n_lstm=1), 2, 1995, id="v4.0-clamped-stem-stride5"),
                pytest.param(lambda: synth.old_style_spec(n_lstm=1), 2, 1000, id="r9-v3.1-4-to-16-stem-fma")]


@pytest.mark.parametrize("make_spec,n,L", ENGINE_SPECS)
def test_engine_front_end(native, monkeypatch, make_spec, n, L):
    """forward(return_features=True) of a built plan: the buffers have the geometry the tests above use, feats["stem"] is
    inside the stem interval computed from the plan's own packed weights, activations and bounds, and feats["conv"] is
    inside the conv3 GEMM interval on the zero-padded stem."""
    monkeypatch.delenv("B200_STEM_IMPL", raising=False)
    plan = _plan(make_spec())
    x = _signal(n, L, seed=n + L)
    with torch.inference_mode():
        _, feats = plan.forward(x.cuda(), return_features=True)
    torch.cuda.synchronize()
    (b,) = plan._bufs.values()
    T, Tp, Lp, _ = engine_geometry(L, plan.k3, plan.s3, plan.pad3)
    assert (b["T"], b["Tp"], b["Lp"]) == (T, Tp, Lp)
    bounds = plan.stem_bounds
    w1, b1, w2, b2 = (None if t is None else t.cpu() for t in (plan.w1, plan.b1, plan.w2, plan.b2))
    stem = np.zeros((n, Lp, plan.c2))
    stem[:, plan.pad3:plan.pad3 + L] = feats["stem"].double().cpu().numpy()
    _check_stem(stem, x, (w1, b1, w2, b2), plan.act1, plan.act2, Lp, plan.pad3, bounds, f"engine stem {plan.hidden}")
    flat = np.concatenate([stem.reshape(-1), np.zeros(plan.k3 * plan.c2)])
    o_lo, o_hi = conv_gemm_reference(flat, n, T, Tp, plan.s3, plan.k3, plan.w3.cpu(), plan.b3.cpu(), plan.act3, plan.lo3,
                                     plan.hi3, list(range(n)))
    got = feats["conv"].double().cpu().numpy().transpose(1, 0, 2)                 # [T, N, H] -> [N, T, H]
    check_between(got, o_lo, o_hi, f"engine conv {plan.hidden}")
    _check_gemm_width(o_lo, o_hi, f"engine conv {plan.hidden}")


# ------------------------------------------------------------------------------------------------ quantize_i8
def _quantize_inputs(n, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(n, generator=g) * 2.4 - 1.2).half()
    edges = []
    for v in (126.5 / 127, 127.5 / 127):             # the fp16 values on both sides of the last rounding step and the clamp
        h = np.float16(v)
        edges += [np.nextafter(h, np.float16(0)), h, np.nextafter(h, np.float16(2))]
    special = np.array(edges + [1.0, 0.0, -0.0, 2.0, 1000.0, 65504.0, np.inf, 6e-8, 3e-5, 6.1e-5], dtype=np.float16)
    special = torch.from_numpy(np.concatenate([special, -special]))
    k = min(n, special.numel())
    x[torch.randperm(n, generator=g)[:k]] = special[:k]
    return x


def _i8_reference(x, scale):
    v = np.rint(x.double().numpy() * np.float32(scale))             # numpy rounds half to even
    return np.clip(v, -127, 127).astype(np.int8)


@pytest.mark.parametrize("n8", [1, 255, 256, 257, 3 * 132 * 8 * 256 + 5])
def test_quantize_i8_blocks_and_saturation(native, n8):
    """quantize_i8 (256 threads x 8 elements per block) equals clamp(rint_even(x * 127), -127, 127) bit for bit at one,
    partial and many blocks, with every fp16 value next to 126.5 / 127 and 127.5 / 127, +-1, +-0, subnormals, +-inf and
    large values among the inputs; the 8 bytes before and after the output are untouched."""
    n = 8 * n8
    x = _quantize_inputs(n, seed=n8)
    xbuf = torch.zeros(16 + n, dtype=torch.float16, device="cuda")
    xbuf[16:] = x.cuda()
    buf = torch.full((8 + n + 8,), CANARY8, dtype=torch.uint8, device="cuda")
    native.quantize_i8(xbuf[16:], buf[8:8 + n].view(torch.int8), 127.0)
    torch.cuda.synchronize()
    host = buf.cpu().numpy()
    assert (host[:8] == CANARY8).all() and (host[8 + n:] == CANARY8).all()
    want = _i8_reference(x, 127.0)
    got = host[8:8 + n].view(np.int8)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{bad.size} differ; first x={float(x[bad[0]])} got {got[bad[0]]} want {want[bad[0]]}"


def test_quantize_i8_rounds_ties_to_even(native):
    """With scale 1 the products are exact halves: rint rounds them to even (0.5 -> 0, 1.5 -> 2, -2.5 -> -2)."""
    x = torch.tensor([0.5, 1.5, 2.5, 3.5, -0.5, -1.5, -2.5, 126.5, -126.5, 127.5, 0.25, 0.75], dtype=torch.float16)
    x = torch.cat([x, torch.zeros(4, dtype=torch.float16)])
    out = torch.full((16,), CANARY8, dtype=torch.uint8, device="cuda")
    native.quantize_i8(x.cuda(), out.view(torch.int8), 1.0)
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy().view(np.int8), _i8_reference(x, 1.0))


def test_quantize_i8_refusals_and_empty_input(native):
    """n = 0 writes nothing, also for empty tensors, whose data pointer is null (this was refused as "bad arguments"); n %
    8 != 0 and a misaligned input (16 bytes) or output (8 bytes) are refused before any launch."""
    xbuf = torch.ones(64, dtype=torch.float16, device="cuda")
    buf = torch.full((64,), CANARY8, dtype=torch.uint8, device="cuda")
    native.quantize_i8(xbuf[:0], buf[8:].view(torch.int8), 127.0)
    native.quantize_i8(torch.empty(0, dtype=torch.float16, device="cuda"), torch.empty(0, dtype=torch.int8, device="cuda"))
    for x, out in ((xbuf[:12], buf[8:]), (xbuf[1:9], buf[8:]), (xbuf[:8], buf[9:])):
        with pytest.raises(native.NativeError, match="multiple of 8"):
            native.quantize_i8(x, out.view(torch.int8), 127.0)
    torch.cuda.synchronize()
    assert (buf.cpu().numpy() == CANARY8).all()
