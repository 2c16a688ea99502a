"""
Windowed attention of the transformer (sup) models at its window, tile and grid edges, on both kernels: the wgmma product
path (attention_wgmma.cu, 128-query CTAs) and the mma.sync cross-check (transformer.cu, 64-query CTAs, B200_ATTN_IMPL=mma),
each after rotary_kernel, which rotates q and k of the packed projection in place.  Every call goes through
`native.attention`; the projection and the output carry canary margins (_edges.py), and every element of
out [N][T][NH*64] must be written and nothing else.

Bound of the random-score tests (`attention_interval`).  Both kernels partition the keys into 64-aligned blocks and run
the online softmax block by block: with the running max m_b after block b, key j of block b gets p_j = ex2((s_j - m_b) c),
c = fp32(log2 e) / 8; P_j = rn16(p_j) enters O += P V, the fp32 p_j enters l; earlier blocks are rescaled by
corr = ex2((m_old - m_new) c); out = rn16(o * (1 / l)).  The interval reference follows that in float64:
  * the fp32 tensor-core score is within eps_j = 64 2^-23 sum_d |q_d k_d| of s_j, so the kernel's running max is within
    E_b = max eps over the visible keys of blocks <= b of m_b.  eps_j = 0 where q and k are multiples of 2^-r_q and 2^-r_k
    with sum_d |q_d k_d| < 2^(24 - r_q - r_k): every partial sum, in any order, is then a multiple of 2^-(r_q + r_k)
    below 2^(24 - r_q - r_k), exact in fp32, and so is the score.  Most cases use such inputs (q and k on a 1/16 grid,
    rotary table cos = 1, sin = 0), which leaves P ambiguous only where p itself lies within 2^-21 of an fp16 midpoint;
  * x = (s_j - m_b) c takes two fp32 roundings (2^-22 relative of |x|) and ex2.approx.ftz 2^-22 relative (a result below
    2^-126 may flush to 0), which gives [p_lo, p_hi] and P_j in [rn16(p_lo), rn16(p_hi)];
  * o / l is unchanged when both are multiplied by 2^((M_kernel - M) c), M the row's final max, so in that common frame
    l's weight of key j is 2^((s_j - M) c) within eps_j c + |x| 2^-22 in the exponent and 2^-22 relative (the kernel's m_b
    cancels), while o's weight is P_j 2^((m_b - M) c) with m_b known to +-E_b; the chain of corr factors adds
    2^-22 relative per block and 2^-22 |M - m_b| c ln 2 for the roundings of its arguments, to both;
  * o: the PV dot products and rescales of every block processed, 65 2^-23 sum_j P_j |v_j| per block; l: one 2^-24
    rounding per add, rescale and shuffle (count + 2 blocks + 2), all terms positive;
  * out = o / l over the interval corners, widened by 2^-23 relative (the IEEE reciprocal and the multiply), rounded.
With exact scores most elements admit one or two fp16 values; the widest intervals are those of outputs near 0, where
the absolute accumulation term spans many of the dense small fp16 values.  Each test prints its widest interval and the
share of elements within two values.
"""
import math

import numpy as np
import pytest
import torch

from _edges import CANARY16, bits16, canary16, check_between, check_guarded, fp16_values_admitted, rn16
from oracle import transformer_oracle as TO

HD = 64
C_LOG2 = float(np.float32(1.4426950408889634)) / 8.0      # the kernels' scale_log2e: fp32(log2 e) / sqrtf(64), exact
FRONT, BACK = 4 * HD, 4 * HD + 8                          # canary margins (elements), 16-byte aligned


@pytest.fixture(scope="module")
def native():
    from bonito_b200 import native as nat
    nat.require()
    return nat


@pytest.fixture(params=["wgmma", "mma"])
def impl(request, monkeypatch):
    if request.param == "mma":
        monkeypatch.setenv("B200_ATTN_IMPL", "mma")
    else:
        monkeypatch.delenv("B200_ATTN_IMPL", raising=False)
    return request.param


# ------------------------------------------------------------------------------------------------ references
def _window(T, wl, wr):
    """The kernels' window: a negative side is unlimited."""
    return (T if wl < 0 else wl), (T if wr < 0 else wr)


def _visible(T, wl, wr):
    """[T, Tp] mask of the keys query i sees, keys padded to whole 64-key blocks."""
    wl, wr = _window(T, wl, wr)
    Tp = -(-T // 64) * 64
    i, j = np.arange(T)[:, None], np.arange(Tp)[None, :]
    return (j >= i - wl) & (j <= i + wr) & (j < T)


def _pad_keys(x, Tp):
    out = np.zeros((Tp,) + x.shape[1:])
    out[:x.shape[0]] = x
    return out


def _frac_bits(x):
    """The least r with every value of x a multiple of 2^-r."""
    for r in range(26):
        if (np.floor(x * 2.0 ** r) == x * 2.0 ** r).all():
            return r
    return 99


def attention_interval(q, k, v, wl, wr):
    """q, k, v float64 [N, T, NH, 64] (fp16 values, q and k already rotated) -> lo, hi [N, T, NH, 64]; the bound of the
    module docstring."""
    N, T, NH, _ = q.shape
    vis = _visible(T, wl, wr)
    Tp = vis.shape[1]
    nb = Tp // 64
    wl_, wr_ = _window(T, wl, wr)
    nb_row = min(nb, (min(wl_, T) + min(wr_, T) + 128) // 64 + 2)     # blocks a CTA processes for one of its rows
    count = vis.sum(axis=1)[:, None]
    lo, hi = np.empty((N, T, NH, HD)), np.empty((N, T, NH, HD))
    for n in range(N):
        for h in range(NH):
            qq, kk, vv = q[n, :, h], _pad_keys(k[n, :, h], Tp), _pad_keys(v[n, :, h], Tp)
            S = qq @ kk.T
            A = np.abs(qq) @ np.abs(kk).T
            eps = np.where(A * 2.0 ** (_frac_bits(qq) + _frac_bits(kk)) < 2 ** 24, 0.0, (64 * 2.0 ** -23 + 2.0 ** -40) * A)
            m_run = np.maximum.accumulate(np.where(vis, S, -np.inf).reshape(T, nb, 64).max(-1), axis=1)
            e_run = np.maximum.accumulate(np.where(vis, eps, 0.0).reshape(T, nb, 64).max(-1), axis=1)
            M, E = m_run[:, -1:], e_run[:, -1:]
            mb = np.where(vis, np.repeat(m_run, 64, axis=1), 0.0)
            eb = np.where(vis, np.repeat(e_run, 64, axis=1), 0.0)
            d = np.where(vis, S - mb, 0.0)                              # <= 0 on visible keys
            ed = eps + eb
            x_lo = (d - ed) * C_LOG2 * (1 + 2.0 ** -22)
            x_hi = np.minimum(0.0, (d + ed) * C_LOG2 * (1 - 2.0 ** -22))
            p_lo = np.exp2(x_lo) * (1 - 2.0 ** -22)
            p_lo = np.where(p_lo < 2.0 ** -126, 0.0, p_lo)               # ex2.approx.ftz
            p_hi = np.exp2(x_hi) * (1 + 2.0 ** -22)
            finite = np.isfinite(m_run)                                 # blocks up to the row's first visible key: -inf
            m_safe = np.where(finite, m_run, M)
            gam_b = nb * 2.0 ** -22 + math.log(2) * 2.0 ** -22 * (M - m_safe + E + e_run) * C_LOG2 * 1.01   # [T, nb]
            # o in the frame of the kernel's final max: block b's sum X_b = sum_j P_j v_j times lam_b = 2^((m_b - M) c)
            lam_lo = np.where(finite, np.exp2((m_safe - e_run - M - E) * C_LOG2) * (1 - gam_b), 0.0)
            lam_hi = np.where(finite, np.minimum(1.0, np.exp2((m_safe + e_run - M + E) * C_LOG2)) * (1 + gam_b), 0.0)
            P_lo, P_hi = np.where(vis, rn16(p_lo), 0.0), np.where(vis, rn16(p_hi), 0.0)
            vp, vm = np.maximum(vv, 0.0), np.minimum(vv, 0.0)
            o_lo, o_hi, o_abs = np.zeros((T, HD)), np.zeros((T, HD)), np.zeros((T, HD))
            for b in range(nb):
                sl = slice(64 * b, 64 * b + 64)
                x_l = P_lo[:, sl] @ vp[sl] + P_hi[:, sl] @ vm[sl]
                x_h = P_hi[:, sl] @ vp[sl] + P_lo[:, sl] @ vm[sl]
                ll, lh = lam_lo[:, b:b + 1], lam_hi[:, b:b + 1]
                o_lo += np.minimum(ll * x_l, lh * x_l)
                o_hi += np.maximum(ll * x_h, lh * x_h)
                o_abs += lh * (P_hi[:, sl] @ np.abs(vv[sl]))
            g_o = 65 * nb_row * 2.0 ** -23 * o_abs
            o_lo, o_hi = o_lo - g_o, o_hi + g_o
            # l in the frame of the reference max: the kernel's m_b cancels, the final max leaves a factor F on out
            gam = np.where(vis, np.repeat(gam_b, 64, axis=1), 0.0)
            z = np.where(vis, (S - M) * C_LOG2, -np.inf)
            ez = eps * C_LOG2 + 2.0 ** -22 * (np.abs(d) + ed) * C_LOG2
            wd_lo = np.where(vis & (p_lo > 0), np.exp2(z - ez) * (1 - 2.0 ** -22) * (1 - gam), 0.0)
            wd_hi = np.where(vis, np.exp2(z + ez) * (1 + 2.0 ** -22) * (1 + gam), 0.0)
            l_lo, l_hi = wd_lo.sum(axis=1, keepdims=True), wd_hi.sum(axis=1, keepdims=True)
            g_l = (count + 2 * nb_row + 2) * 2.0 ** -24 * l_hi
            l_lo, l_hi = l_lo - g_l, l_hi + g_l
            f_lo, f_hi = np.exp2(-E * C_LOG2), np.exp2(E * C_LOG2)    # F = 2^((M_kernel - M) c)
            a_, b_ = np.minimum(o_lo / l_lo, o_lo / l_hi), np.maximum(o_hi / l_lo, o_hi / l_hi)
            r_lo, r_hi = np.minimum(f_lo * a_, f_hi * a_), np.maximum(f_lo * b_, f_hi * b_)
            lo[n, :, h] = rn16(r_lo - 2.0 ** -23 * np.abs(r_lo))
            hi[n, :, h] = rn16(r_hi + 2.0 ** -23 * np.abs(r_hi))
    return lo, hi


def attention_point(q, k, v, wl, wr, round_p=True, vis=None):
    """The same block-wise online softmax in float64 without error terms, rounded to fp16: what an exact kernel with these
    rounding points would write.  `round_p=False` skips the fp16 rounding of P; `vis` overrides the window mask."""
    N, T, NH, _ = q.shape
    vis = _visible(T, wl, wr) if vis is None else vis
    Tp = vis.shape[1]
    nb = Tp // 64
    out = np.empty((N, T, NH, HD))
    for n in range(N):
        for h in range(NH):
            qq, kk, vv = q[n, :, h], _pad_keys(k[n, :, h], Tp), _pad_keys(v[n, :, h], Tp)
            S = qq @ kk.T
            m_run = np.maximum.accumulate(np.where(vis, S, -np.inf).reshape(T, nb, 64).max(-1), axis=1)
            M = m_run[:, -1:]
            mb = np.where(vis, np.repeat(m_run, 64, axis=1), 0.0)
            p = np.where(vis, np.exp2((S - mb) * C_LOG2), 0.0)
            P = rn16(p) if round_p else p
            scale = np.where(vis, np.exp2((mb - M) * C_LOG2), 0.0)
            out[n, :, h] = rn16(((P * scale) @ vv) / (p * scale).sum(axis=1, keepdims=True))
    return out


def rotary_reference(x, cs):
    """x [..., T, NH, 64] float64 (fp16 values), cs [T, 64] = [cos 32 | sin 32] -> the kernel's rotated fp16 bits.
    rotary_kernel computes rn16(rn32(a c - b s)) and rn16(rn32(a s + b c)).  Every fp16 value is a multiple of 2^-24, so
    both products are multiples of 2^-48; with |a|, |b| < 16 and |c|, |s| <= 1 the sum or difference is below 32 in
    magnitude, i.e. fits in 53 bits, so float64 holds it exactly, and float64 -> float32 -> float16 repeats the kernel's
    two roundings."""
    c, s = cs[:, None, :32], cs[:, None, 32:]
    a, b = x[..., :32], x[..., 32:]
    assert np.abs(x).max() < 16
    r1 = (a * c - b * s).astype(np.float32).astype(np.float16)
    r2 = (a * s + b * c).astype(np.float32).astype(np.float16)
    return np.concatenate([r1, r2], axis=-1).view(np.int16).astype(np.int64) & 0xFFFF


# ------------------------------------------------------------------------------------------------ running the kernels
def _table(T, identity=False):
    if identity:                                     # cos = 1, sin = 0: rotary leaves q and k as they are
        return torch.cat([torch.ones(T, 32), torch.zeros(T, 32)], dim=1).half()
    cos, sin = TO.rotary_tables(T, HD, fp16=True)
    return torch.cat([cos, sin], dim=1).half()


def _run(native, qkv, cs, wl, wr):
    """One guarded native.attention call.  qkv [N, T, 3, NH, 64] fp16 (host).  Checks that nothing around the projection
    and the output was written and that every output element was; returns the projection after the call (host fp16) and
    the output [N, T, NH, 64] as float64."""
    N, T, _, NH, _ = qkv.shape
    size, osize = qkv.numel(), N * T * NH * HD
    qbuf = canary16(FRONT + size + BACK)
    qbuf[FRONT:FRONT + size] = qkv.reshape(-1).cuda()
    obuf = canary16(FRONT + osize + BACK)
    native.attention(qbuf[FRONT:FRONT + size], cs.cuda(), obuf[FRONT:FRONT + osize], N, T, NH, HD, wl, wr)
    torch.cuda.synchronize()
    qb = bits16(qbuf)
    assert (qb[:FRONT] == CANARY16).all() and (qb[FRONT + size:] == CANARY16).all(), "written outside qkv"
    check_guarded(bits16(obuf), FRONT + np.arange(osize), CANARY16)
    after = qbuf[FRONT:FRONT + size].cpu().view(N, T, 3, NH, HD)
    return after, obuf[FRONT:FRONT + osize].double().cpu().numpy().reshape(N, T, NH, HD)


def _qkv_parts(qkv):
    x = qkv.double().numpy()
    return x[:, :, 0], x[:, :, 1], x[:, :, 2]


def _one_hot_v(N, T, NH):
    j, h, n, d = np.ix_(np.arange(T), np.arange(NH), np.arange(N), np.arange(HD))
    v = ((j + 5 * h + 11 * n) % 64 == d).astype(np.float64)          # [T, NH, N, 64]
    return torch.from_numpy(v.transpose(2, 0, 1, 3)).half()


def _mask_inputs(N, T, NH, seed):
    """q = 0 (every score is exactly 0, every visible key gets P = 1), random k, one-hot v."""
    g = torch.Generator().manual_seed(seed)
    qkv = torch.empty(N, T, 3, NH, HD, dtype=torch.float16)
    qkv[:, :, 0] = 0
    qkv[:, :, 1] = (torch.randn(N, T, NH, HD, generator=g) * 1.5).half()
    qkv[:, :, 2] = _one_hot_v(N, T, NH)
    return qkv


def _random_inputs(N, T, NH, seed, scale=1.5, ramp=0, grid=16):
    """Random q, k, v; q and k rounded to multiples of 1 / `grid` (exact fp32 scores, see the module docstring; 0: plain
    fp16).  `ramp` = +-1 plants a score ramp along the keys (q_0 = 4, k_0 = +-j / 16), so that every row's max lies in its
    last (+1) or first (-1) visible block."""
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(N, T, 3, NH, HD, generator=g) * scale
    if ramp:
        qkv[:, :, :2] *= 0.25
        qkv[:, :, 0, :, 0] = 4.0
        qkv[:, :, 1, :, 0] = ramp * torch.arange(T, dtype=torch.float32)[None, :, None] / 16
    if grid:
        qkv[:, :, :2] = torch.round(qkv[:, :, :2] * grid) / grid
    return qkv.half()


def _report(what, lo, hi):
    widths = fp16_values_admitted(lo, hi)
    print(f"{what}: widest interval {int(widths.max())} fp16 values, {float((widths <= 2).mean()):.4f} of elements "
          f"within 2")


# ------------------------------------------------------------------------------------------------ 1. rotary
@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 63, 65, 1666])
@pytest.mark.parametrize("N", [1, 3])
@pytest.mark.parametrize("NH", [1, 3, 8])
def test_rotary_is_bit_exact(native, impl, NH, N, T):
    """rotary_kernel in place: q and k equal the float64 -> float32 -> float16 emulation bit for bit (see
    `rotary_reference`), v is bitwise unchanged, nothing around the projection is written."""
    g = torch.Generator().manual_seed(100 * T + 10 * N + NH)
    qkv = (torch.randn(N, T, 3, NH, HD, generator=g) * 1.5).clamp(-15, 15).half()
    cs = _table(T)
    after, _ = _run(native, qkv, cs, 127, 128)
    x = qkv.double().numpy()
    csd = cs.double().numpy()
    got = bits16(after)
    for which in (0, 1):
        want = rotary_reference(x[:, :, which], csd)
        bad = got[:, :, which] != want
        assert not bad.any(), f"{'qk'[which]}: {int(bad.sum())} rotated values differ from the emulation"
    assert np.array_equal(got[:, :, 2], bits16(qkv)[:, :, 2]), "v was modified"


# ------------------------------------------------------------------------------------------------ 2. exact mask
def _mask_cases():
    c = [(1, 0, 0, 1, 1, "T=1-self-only"), (1, -1, -1, 8, 3, "T=1-unlimited"),
         (2, 1, 0, 8, 1, "T=2-left-1"), (2, 0, 1, 1, 3, "T=2-right-1"),
         (63, 64, 63, 1, 1, "T=63-window-past-both-ends"), (64, 63, 64, 8, 1, "T=64-one-full-block"),
         (65, 64, 64, 1, 3, "T=65-one-key-in-block-1"), (127, 5, 9, 8, 1, "T=127-last-wgmma-query-row"),
         (128, 65, 0, 1, 3, "T=128-left-65-crosses-block"), (129, 0, 65, 8, 1, "T=129-right-65-one-query-in-tile-2"),
         (191, 63, 64, 8, 3, "T=191-63-64-edges-on-block-boundaries"),
         (193, 64, 63, 1, 1, "T=193-64-63-edges-on-block-boundaries"),
         (255, 64, 64, 8, 1, "T=255-64-64"), (255, 0, 0, 1, 1, "T=255-self-only"),
         (257, 127, 128, 8, 3, "T=257-sup-window"), (257, 128, 127, 1, 1, "T=257-128-127"),
         (257, 129, 129, 8, 1, "T=257-129-129"), (257, 65, 0, 1, 3, "T=257-left-65"), (257, 0, 65, 8, 1, "T=257-right-65"),
         (257, 1, 0, 1, 1, "T=257-left-1"), (257, 0, 1, 1, 1, "T=257-right-1"),
         (1666, 127, 128, 8, 1, "T=1666-sup-window"), (1666, -1, -1, 1, 1, "T=1666-unlimited"),
         (1666, 1673, 1673, 1, 1, "T=1666-window-T+7")]
    return [pytest.param(T, wl, wr, nh, n, id=name) for T, wl, wr, nh, n, name in c]


@pytest.mark.gpu
@pytest.mark.parametrize("T,wl,wr,NH,N", _mask_cases())
def test_attention_mask_is_exact(native, impl, T, wl, wr, NH, N):
    """q = 0 and one-hot v = [(j + 5h + 11n) % 64 == d]: out[n, q, h, d] is the share of the visible keys with that
    residue, counted exactly from [q - wl, q + wr] & [0, T).  The kernel differs from it only by the fp32 sums of
    P = ex2(0) = 1 +- 2^-22 (exactly 1 after the fp16 rounding) and the final division: the interval reference (module
    docstring, here with eps = 0) holds it, and one key more or less at either window edge, or another head's or chunk's
    v, moves some output by about 1 / count, many fp16 values away."""
    qkv = _mask_inputs(N, T, NH, seed=T + wl + 3 * wr)
    after, got = _run(native, qkv, _table(T), wl, wr)
    q, k, v = _qkv_parts(after)
    assert (q == 0).all()
    lo, hi = attention_interval(q, k, v, wl, wr)
    vis = _visible(T, wl, wr)
    share = np.empty_like(got)                                    # count_d / count, exactly
    for n in range(N):
        for h in range(NH):
            share[n, :, h] = (vis[:, :T] @ v[n, :, h]) / vis.sum(axis=1)[:, None]
    check_between(rn16(share), lo, hi, "exact share")             # the reference's own consistency
    check_between(got, lo, hi, f"mask T={T} wl={wl} wr={wr} ({impl})")
    _report(f"mask T={T} ({wl},{wr}) {impl}", lo, hi)


# ------------------------------------------------------------------------------------------------ 3. single-key windows
@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 64, 129, 257])
def test_single_key_window_returns_v_bitwise(native, impl, T):
    """(wl, wr) = (0, 0): each query sees only itself, p = ex2(0) = 1 +- 2^-22, l = p, o = rn16(p) v = v, and
    rn16(v rn32(1 / l)) = v for every fp16 v, so out[q] = v[q] bit for bit."""
    N, NH = 2, 8
    qkv = _random_inputs(N, T, NH, seed=T)
    v = qkv[:, :, 2]
    v[v == 0] = 1.0                                               # the sign of a zero is not part of the contract
    _, got = _run(native, qkv, _table(T), 0, 0)
    want = v.double().numpy()
    assert np.array_equal(got, want), f"{int((got != want).sum())} outputs differ from v"


# ------------------------------------------------------------------------------------------------ 4. random scores
RANDOM_CASES = [
    pytest.param(2, 129, 8, 127, 128, {}, id="sup-window-T=129"),
    pytest.param(1, 257, 8, 127, 128, {}, id="sup-window-T=257"),
    pytest.param(1, 1666, 2, 127, 128, {}, id="sup-window-T=1666"),
    pytest.param(1, 257, 8, 127, 128, dict(grid=0), id="sup-window-rotated-fp16-q-k"),
    pytest.param(2, 257, 8, 0, 128, {}, id="right-only-0-128"),
    pytest.param(2, 257, 8, 127, 0, {}, id="left-only-127-0"),
    pytest.param(3, 257, 8, 5, 9, {}, id="small-window-5-9-warpgroups-skip-blocks"),
    pytest.param(2, 257, 8, 127, 128, dict(ramp=1), id="ramp-max-in-last-visible-block"),
    pytest.param(2, 257, 8, 127, 128, dict(ramp=-1), id="ramp-max-in-first-visible-block"),
    pytest.param(2, 257, 8, 127, 128, dict(scale=6.0, grid=4), id="large-scores-P-underflows-fp16"),
    pytest.param(1, 257, 2, 127, 128, dict(planted=True), id="P-rounds-up-to-the-least-fp16-subnormal"),
]


def _subnormal_p_inputs(N, T, NH, seed):
    """Every 16th key scores 136 (q_0 = 8, k_0 = 17), the others 0: their p = 2^(-136 c) = 0.69 * 2^-24 rounds up to the
    least fp16 subnormal 2^-24 for PV, while l sums the fp32 value.  v = 0 on the high keys and 500 .. 1000 on the others,
    so out ~ 6e-4 is made of the rounded P alone."""
    g = torch.Generator().manual_seed(seed)
    qkv = torch.zeros(N, T, 3, NH, HD)
    hi = torch.arange(T) % 16 == 0
    qkv[:, :, 0, :, 0] = 8.0
    qkv[:, hi, 1, :, 0] = 17.0
    qkv[:, :, 2] = 500.0 + 500.0 * torch.rand(N, T, NH, HD, generator=g)
    qkv[:, hi, 2] = 0.0
    return qkv.half()


def _case_inputs(N, T, NH, seed, kw):
    if kw.get("planted"):
        return _subnormal_p_inputs(N, T, NH, seed)
    return _random_inputs(N, T, NH, seed, **{key: kw[key] for key in ("scale", "ramp", "grid") if key in kw})


@pytest.mark.gpu
@pytest.mark.parametrize("N,T,NH,wl,wr,kw", RANDOM_CASES)
def test_attention_random_scores_in_interval(native, impl, N, T, NH, wl, wr, kw):
    """Random q, k, v against the interval reference of the module docstring, with q and k as the call left them.  Most
    cases keep q and k on a 1/16 grid with the identity rotary table, so that the scores are exact; one runs the real
    table on plain fp16 q and k under the full eps.  The ramps put each row's max in its last or first visible block,
    so the rescale corr is < 1 at every block or = 1 after the first; scale = 6 gives scores of |s| ~ 300, so that many P
    are fp16 subnormals or 0 while l keeps their fp32 values; the planted case makes out a sum of P rounded up to 2^-24."""
    qkv = _case_inputs(N, T, NH, T + wl + wr, kw)
    after, got = _run(native, qkv, _table(T, identity=kw.get("grid", 16) != 0), wl, wr)
    q, k, v = _qkv_parts(after)
    lo, hi = attention_interval(q, k, v, wl, wr)
    check_between(got, lo, hi, f"attention N={N} T={T} ({wl},{wr}) {kw} ({impl})")
    _report(f"random T={T} ({wl},{wr}) {kw} {impl}", lo, hi)


# ------------------------------------------------------------------------------------------------ 5. discriminative power
def _rejects(got, lo, hi):
    try:
        check_between(got, lo, hi, "wrong reference")
    except AssertionError:
        return True
    return False


@pytest.mark.parametrize("T,wl,wr", [pytest.param(257, 127, 128, id="sup-window"), pytest.param(193, 64, 63, id="64-63"),
                                     pytest.param(129, 5, 9, id="5-9")])
def test_mask_check_rejects_wrong_windows_and_heads(T, wl, wr):
    """On the inputs of the exact mask test, the interval check admits the exact emulation and rejects the output of an
    emulation with one key more or less at the left or the right edge, the window shifted by one key either way, or v
    taken from the neighbouring head."""
    N, NH = 2, 3
    q, k, v = _qkv_parts(_mask_inputs(N, T, NH, seed=T))
    lo, hi = attention_interval(q, k, v, wl, wr)
    assert not _rejects(attention_point(q, k, v, wl, wr), lo, hi)
    for wl2, wr2 in ((wl + 1, wr), (wl - 1, wr), (wl, wr + 1), (wl, wr - 1), (wl + 1, wr - 1), (wl - 1, wr + 1)):
        assert _rejects(attention_point(q, k, v, wl2, wr2), lo, hi), (wl2, wr2)
    assert _rejects(attention_point(q, k, np.roll(v, 1, axis=2), wl, wr), lo, hi), "neighbouring head"


@pytest.mark.parametrize("kw", [pytest.param({}, id="random"), pytest.param(dict(ramp=1), id="ramp-up"),
                                pytest.param(dict(ramp=-1), id="ramp-down"),
                                pytest.param(dict(scale=6.0, grid=4), id="large"),
                                pytest.param(dict(planted=True), id="P-subnormal")])
def test_random_check_rejects_wrong_references(kw):
    """On the inputs of the random-score test, the interval check admits the exact emulation and rejects: the mask
    shifted by one key on the left or the right, P not rounded to fp16 before PV, v from the neighbouring head."""
    N, T, NH, wl, wr = 1, 257, 3, 127, 128
    q, k, v = _qkv_parts(_case_inputs(N, T, NH, 5, kw))
    lo, hi = attention_interval(q, k, v, wl, wr)
    assert not _rejects(attention_point(q, k, v, wl, wr), lo, hi)
    vis = _visible(T, wl, wr)
    assert _rejects(attention_point(q, k, v, wl, wr, vis=np.roll(vis, 1, axis=1) & (np.arange(vis.shape[1]) < T)), lo, hi)
    assert _rejects(attention_point(q, k, v, wl, wr, vis=np.roll(vis, -1, axis=1) & (np.arange(vis.shape[1]) < T)), lo, hi)
    assert _rejects(attention_point(q, k, v, wl + 1, wr), lo, hi)
    assert _rejects(attention_point(q, k, v, wl, wr + 1), lo, hi)
    assert _rejects(attention_point(q, k, v, wl, wr, round_p=False), lo, hi), "P not rounded to fp16"
    assert _rejects(attention_point(q, k, np.roll(v, 1, axis=2), wl, wr), lo, hi), "neighbouring head"


# ------------------------------------------------------------------------------------------------ 6. refusals
@pytest.mark.gpu
def test_attention_refuses_head_dim_other_than_64(native, impl):
    qkv = torch.zeros(1, 4, 3, 2, 32, dtype=torch.float16, device="cuda")
    cs = _table(4).cuda()
    out = torch.zeros(1, 4, 64, dtype=torch.float16, device="cuda")
    with pytest.raises(native.NativeError, match="head_dim 32 is not supported"):
        native.attention(qkv, cs, out, 1, 4, 2, 32, 127, 128)
