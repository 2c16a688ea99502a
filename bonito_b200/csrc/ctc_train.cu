// Training kernels of the QuartzNet CTC models (bonito/ctc/model.py in train mode: BatchNorm on batch statistics, Dropout
// after every activation), sm_90a.  Every activation is channels-last fp16 rows [M = N*T][C]; every reduction over the rows
// is split into fixed slices whose fp32 partials are combined in slice order, so no kernel uses atomics and two identical
// calls give bitwise-equal results.  Slice counts depend on the shapes only, never on the device.
//
//   wgrad GEMM      dW[co][k] = sum_r dZ[row(r)][co] X[r][k] over the GEMM rows r of a b200_gemm_fwd_ex row map (overlapping
//                   X rows give the dense k > 1 convolution's gradient in one call): mma.sync m16n8k16 on 128 x 128 output
//                   tiles, both operands staged row-major ([rows][channels], as the forward keeps them) and fed to the
//                   tensor cores through ldmatrix.trans, split-K over row slices into fp32 partials
//   tap wgrads      depthwise dWd[c][k] and the first convolution's dW[c][k] against the raw signal: 32 channels x a
//                   slice of (chunk, 64-frame tile) units per CTA, one fp32 partial per slice
//   bn_stats        per-channel Welford over 512-row slices, merged by Chan's formula in fp64 in slice order
//   bn_act fwd/bwd  BatchNorm (batch statistics) [+ the residual branch's BatchNorm] -> activation -> dropout, and its
//                   gradient: the per-channel sums of g and g * xhat, then dz of both BatchNorm branches; the activation
//                   input is recomputed from the saved pre-BatchNorm tensors
//   head            logits -> fp32 log_softmax, and its gradient (dlogits, dfeat, dW_h, db_h)
//
// Non-finite values pass through: nothing is clamped or skipped, so an inf upstream gradient gives non-finite parameter
// gradients (GradScaler's overflow test).
#include <math.h>

#include <algorithm>

#include "common.cuh"

namespace {

constexpr int SLICE_ROWS = 512;   // rows per partial of the per-channel reductions
constexpr int CH_THREADS = 128;   // per-channel reductions: 2 channels per thread, 256 per CTA

__host__ __device__ inline long long cdiv(long long a, long long b) { return (a + b - 1) / b; }

__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
                 : "r"(addr));
}

// out[i] = sum_{s < S} part[s][i], in slice order
__global__ void sum_partials_kernel(const float* __restrict__ part, int S, long long n, float* __restrict__ out) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        float s = 0.f;
        for (int j = 0; j < S; ++j) s += part[j * n + i];
        out[i] = s;
    }
}

int sum_partials(const float* part, int S, long long n, float* out, cudaStream_t stream) {
    const int grid = (int)std::min<long long>(cdiv(n, 256), 4096);
    sum_partials_kernel<<<grid, 256, 0, stream>>>(part, S, n, out);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------ wgrad GEMM
constexpr int WG_BM = 128, WG_BN = 128, WG_BK = 32, WG_STAGES = 3, WG_PAD = 8, WG_THREADS = 256;
constexpr int WG_LD = WG_BM + WG_PAD;    // 272-byte smem rows: the 8 row addresses of an ldmatrix hit distinct banks

struct WgSmem {
    __half a[WG_STAGES][WG_BK][WG_LD];   // dZ rows [r][co]
    __half b[WG_STAGES][WG_BK][WG_LD];   // X rows  [r][k]
};

struct WgArgs {
    const __half* dz;
    long long ldz, lpz;
    const __half* x;
    long long ldx;
    long long m;          // GEMM rows
    int rows_inner, valid_inner, cout, k;
    int ktiles_per_slice;
};

__global__ void __launch_bounds__(WG_THREADS, 1) wgrad_gemm_kernel(WgArgs p, float* __restrict__ out) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    WgSmem& s = *reinterpret_cast<WgSmem*>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp >> 2, wn = warp & 3;   // 2 x 4 warps, warp tile 64 (co) x 32 (k)
    const int co0 = blockIdx.y * WG_BM, k0 = blockIdx.x * WG_BN;
    const long long ktiles = cdiv(p.m, WG_BK);
    const long long kt0 = (long long)blockIdx.z * p.ktiles_per_slice;
    const int nkt = (int)std::min<long long>(p.ktiles_per_slice, ktiles - kt0);

    auto load_stage = [&](int stage, long long kt) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int chunk = tid + i * WG_THREADS;   // 32 rows x 16 chunks of 16 B per operand
            const int row = chunk >> 4, col = (chunk & 15) * 8;
            const long long r = kt * WG_BK + row;
            bool vr = r < p.m;
            long long outer = 0;
            int inner = 0;
            if (vr) {
                outer = r / p.rows_inner;
                inner = (int)(r - outer * p.rows_inner);
                vr = inner < p.valid_inner;
            }
            const bool va = vr && co0 + col < p.cout;
            cp_async_16(&s.a[stage][row][col], p.dz + (va ? (outer * p.lpz + inner) * p.ldz + co0 + col : 0), va);
            const bool vb = vr && k0 + col < p.k;
            cp_async_16(&s.b[stage][row][col], p.x + (vb ? r * p.ldx + k0 + col : 0), vb);
        }
    };

    float acc[4][4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[i][j][q] = 0.f;

#pragma unroll
    for (int st = 0; st < WG_STAGES - 1; ++st) {
        if (st < nkt) load_stage(st, kt0 + st);
        cp_async_commit();
    }
    const int mi = lane >> 3, mr = lane & 7;
    for (int kt = 0; kt < nkt; ++kt) {
        cp_async_wait<WG_STAGES - 2>();
        __syncthreads();
        {
            const int nk = kt + WG_STAGES - 1;
            if (nk < nkt) load_stage(nk % WG_STAGES, kt0 + nk);
            cp_async_commit();
        }
        const int st = kt % WG_STAGES;
#pragma unroll
        for (int kk = 0; kk < WG_BK; kk += 16) {
            uint32_t af[4][4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {   // A[co][r] = dZ[r][co]: matrices (co 0-7, r 0-7), (co 8-15, r 0-7), (co 0-7, r 8-15), ...
                const int r = kk + mr + (mi >> 1) * 8, c = wm * 64 + i * 16 + (mi & 1) * 8;
                ldmatrix_x4_trans(af[i][0], af[i][1], af[i][2], af[i][3], smem_u32(&s.a[st][r][c]));
            }
            uint32_t bf[4][2];
#pragma unroll
            for (int j = 0; j < 2; ++j) {   // B[r][k] = X[r][k]: matrices (r 0-7, k 0-7), (r 8-15, k 0-7), (r 0-7, k 8-15), ...
                const int r = kk + mr + (mi & 1) * 8, c = wn * 32 + j * 16 + (mi >> 1) * 8;
                ldmatrix_x4_trans(bf[2 * j][0], bf[2 * j][1], bf[2 * j + 1][0], bf[2 * j + 1][1], smem_u32(&s.b[st][r][c]));
            }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) mma_16816(acc[i][j], af[i], bf[j][0], bf[j][1]);
        }
    }
    cp_async_wait<0>();

    float* dst = out + (long long)blockIdx.z * p.cout * p.k;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int co = co0 + wm * 64 + i * 16 + (lane >> 2) + h * 8;
            if (co >= p.cout) continue;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int kc = k0 + wn * 32 + j * 8 + (lane & 3) * 2;   // k is a multiple of 8: kc + 1 < k with kc
                if (kc < p.k)
                    *reinterpret_cast<float2*>(dst + (long long)co * p.k + kc) = make_float2(acc[i][j][2 * h], acc[i][j][2 * h + 1]);
            }
        }
}

// split-K: about two waves of 132 CTAs (a fixed count: the result must not depend on the device), at least 16 row tiles
// (512 rows) per slice, at most 64 slices
int wgrad_slices(long long m, int cout, int k, int* per_slice) {
    const long long ktiles = cdiv(m, WG_BK);
    const long long tiles = cdiv(cout, WG_BM) * cdiv(k, WG_BN);
    long long s = std::min(cdiv(264, tiles), ktiles / 16);
    s = std::max(1LL, std::min(s, 64LL));
    const long long per = cdiv(ktiles, s);
    if (per_slice) *per_slice = (int)per;
    return (int)cdiv(ktiles, per);
}

// ------------------------------------------------------------------------------------------------ tap wgrads
constexpr int TAP_TT = 64, TAP_CH = 32, TAP_THREADS = 256, TAP_GROUPS = TAP_THREADS / TAP_CH;
constexpr int DW_KMAX = 123, FC_KMAX = 33, FC_SMAX = 8;
constexpr int TAP_KJ_MAX = (DW_KMAX + TAP_GROUPS - 1) / TAP_GROUPS;
// rows (depthwise) staged per unit: the last group's window reaches row rows - 1 + TAP_GROUPS * KJ; the signal span
// (TAP_TT - 1) * FC_SMAX + TAP_GROUPS * KJ is smaller
constexpr int TAP_XS = (TAP_TT + TAP_GROUPS * TAP_KJ_MAX) * TAP_CH;

// SIGNAL = false: depthwise, x [N*T rows][ldx] channels-last, out[c][k] += dy[n][t][c] x[n][t + k - K/2][c];
// SIGNAL = true:  first convolution, x [N][L] samples, out[c][k] += dy[n][t][c] x[n][t*stride + k - K/2].
// Thread (group g, channel c) owns the KJ = ceil(K / 8) consecutive taps g*KJ .. g*KJ + KJ - 1 of channel c.  Depthwise:
// its x values for consecutive frames are a sliding window, kept in registers (one shared-memory load per frame).
// Every tap's sum runs over the frames in order, so the result does not depend on KJ.
template <bool SIGNAL, int KJ>
__global__ void __launch_bounds__(TAP_THREADS) tap_wgrad_kernel(const __half* __restrict__ dy, long long ldy,
                                                                 const __half* __restrict__ x, long long ldx, int N, int T,
                                                                 int L, int C, int K, int stride, int units_per_slice,
                                                                 float* __restrict__ out) {
    __shared__ float xs[TAP_XS];
    __shared__ float ys[TAP_TT * TAP_CH];
    const int tid = threadIdx.x, cc = tid % TAP_CH, grp = tid / TAP_CH;
    const int c0 = blockIdx.x * TAP_CH, c = c0 + cc, k0 = grp * KJ;
    const int tiles = (int)cdiv(T, TAP_TT);
    const long long units = (long long)N * tiles;
    const long long u0 = (long long)blockIdx.y * units_per_slice;
    const long long u1 = std::min<long long>(units, u0 + units_per_slice);
    const int h = K / 2;
    float acc[KJ];
#pragma unroll
    for (int j = 0; j < KJ; ++j) acc[j] = 0.f;

    for (long long u = u0; u < u1; ++u) {
        const int n = (int)(u / tiles), t0 = (int)(u % tiles) * TAP_TT;
        const int rows = min(TAP_TT, T - t0);
        for (int i = tid; i < TAP_TT * TAP_CH; i += TAP_THREADS) {
            const int tt = i / TAP_CH, ci = c0 + i % TAP_CH;
            ys[i] = (tt < rows && ci < C) ? __half2float(dy[((long long)n * T + t0 + tt) * ldy + ci]) : 0.f;
        }
        if (SIGNAL) {
            const int span = (rows - 1) * stride + TAP_GROUPS * KJ;
            for (int i = tid; i < span; i += TAP_THREADS) {
                const long long pos = (long long)t0 * stride - h + i;
                xs[i] = (i < (rows - 1) * stride + K && pos >= 0 && pos < L) ? __half2float(x[(long long)n * ldx + pos]) : 0.f;
            }
        } else {
            const int span = (rows + TAP_GROUPS * KJ) * TAP_CH;
            for (int i = tid; i < span; i += TAP_THREADS) {
                const int r = i / TAP_CH, tt = t0 - h + r, ci = c0 + i % TAP_CH;
                xs[i] = (r < rows + K - 1 && tt >= 0 && tt < T && ci < C) ? __half2float(x[((long long)n * T + tt) * ldx + ci])
                                                                           : 0.f;
            }
        }
        __syncthreads();
        if (k0 < K) {
            if (SIGNAL) {
                for (int tt = 0; tt < rows; ++tt) {
                    const float g = ys[tt * TAP_CH + cc];
#pragma unroll
                    for (int j = 0; j < KJ; ++j) acc[j] = fmaf(g, xs[tt * stride + k0 + j], acc[j]);
                }
            } else {
                float w[KJ];
#pragma unroll
                for (int j = 0; j < KJ; ++j) w[j] = xs[(k0 + j) * TAP_CH + cc];
                for (int tt = 0; tt < rows; ++tt) {
                    const float g = ys[tt * TAP_CH + cc];
#pragma unroll
                    for (int j = 0; j < KJ; ++j) acc[j] = fmaf(g, w[j], acc[j]);
#pragma unroll
                    for (int j = 0; j + 1 < KJ; ++j) w[j] = w[j + 1];
                    w[KJ - 1] = xs[(tt + k0 + KJ) * TAP_CH + cc];
                }
            }
        }
        __syncthreads();
    }
    if (c < C) {
        float* dst = out + ((long long)blockIdx.y * C + c) * K;
#pragma unroll
        for (int j = 0; j < KJ; ++j)
            if (k0 + j < K) dst[k0 + j] = acc[j];
    }
}

template <bool SIGNAL, int KJ>
void launch_tap_kj(int kj, dim3 grid, cudaStream_t st, const __half* dy, long long ldy, const __half* x, long long ldx, int n,
                   int t, int l, int c, int k, int stride, int per, float* out) {
    if constexpr (KJ > 0) {
        if (kj == KJ) {
            tap_wgrad_kernel<SIGNAL, KJ><<<grid, TAP_THREADS, 0, st>>>(dy, ldy, x, ldx, n, t, l, c, k, stride, per, out);
            return;
        }
        launch_tap_kj<SIGNAL, KJ - 1>(kj, grid, st, dy, ldy, x, ldx, n, t, l, c, k, stride, per, out);
    }
}

int tap_slices(int n, int t, int* per_slice) {
    const long long units = (long long)n * cdiv(t, TAP_TT);
    const long long s = std::max(1LL, std::min(units, 128LL));
    const long long per = cdiv(units, s);
    if (per_slice) *per_slice = (int)per;
    return (int)cdiv(units, per);
}

// ------------------------------------------------------------------------------------------------ BatchNorm statistics
__global__ void __launch_bounds__(CH_THREADS) bn_stats_partial_kernel(const __half* __restrict__ z, long long ldz, long long M,
                                                                       int C, float* __restrict__ pmean, float* __restrict__ pm2) {
    const int c = blockIdx.x * 2 * CH_THREADS + 2 * threadIdx.x;
    if (c >= C) return;
    const long long r0 = (long long)blockIdx.y * SLICE_ROWS, r1 = std::min<long long>(M, r0 + SLICE_ROWS);
    float m0 = 0.f, m1 = 0.f, q0 = 0.f, q1 = 0.f;
    for (long long r = r0; r < r1; ++r) {   // Welford
        const float2 v = __half22float2(*reinterpret_cast<const __half2*>(z + r * ldz + c));
        const float inv = 1.f / (float)(r - r0 + 1);
        const float d0 = v.x - m0, d1 = v.y - m1;
        m0 = fmaf(d0, inv, m0);
        m1 = fmaf(d1, inv, m1);
        q0 = fmaf(d0, v.x - m0, q0);
        q1 = fmaf(d1, v.y - m1, q1);
    }
    const long long o = (long long)blockIdx.y * C + c;
    pmean[o] = m0;
    pmean[o + 1] = m1;
    pm2[o] = q0;
    pm2[o + 1] = q1;
}

__global__ void bn_stats_final_kernel(const float* __restrict__ pmean, const float* __restrict__ pm2, int S, long long M, int C,
                                      float eps, float momentum, float* __restrict__ mean, float* __restrict__ invstd,
                                      float* __restrict__ running_mean, float* __restrict__ running_var) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double n = 0.0, mu = 0.0, m2 = 0.0;
    for (int s = 0; s < S; ++s) {   // Chan et al.: merge (n, mu, m2) with the slice's (nb, mb, qb)
        const double nb = (double)std::min<long long>(SLICE_ROWS, M - (long long)s * SLICE_ROWS);
        const double mb = pmean[(long long)s * C + c], qb = pm2[(long long)s * C + c];
        const double nn = n + nb, d = mb - mu;
        mu += d * nb / nn;
        m2 += qb + d * d * n * nb / nn;
        n = nn;
    }
    const double var = m2 / (double)M;
    mean[c] = (float)mu;
    invstd[c] = (float)(1.0 / sqrt(var + (double)eps));
    if (running_mean) {
        running_mean[c] = (float)((1.0 - momentum) * running_mean[c] + momentum * mu);
        running_var[c] = (float)((1.0 - momentum) * running_var[c] + momentum * (m2 / (double)(M - 1)));
    }
}

// ------------------------------------------------------------------------------------------------ BatchNorm + act + dropout
struct Bn {
    long long m;
    int c, t, act;
    float p;
    unsigned long long seed;
    int unit;
    const __half* z;
    long long ldz;
    const float *mean, *invstd, *gamma, *beta;
    const __half* zr;
    long long ldzr;
    const float *mean_r, *invstd_r, *gamma_r, *beta_r;
    uint8_t* mask;
};

// counter-based keep decision of element (row, channel) of dropout `unit`: splitmix64 of (seed, unit, index)
__device__ __forceinline__ bool keep_elem(unsigned long long seed, int unit, long long idx, uint32_t threshold) {
    unsigned long long z = seed + 0xD1B54A32D192ED03ull * (unsigned long long)(unit + 1) +
                           0x9E3779B97F4A7C15ull * (unsigned long long)(idx + 1);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z ^= z >> 31;
    return (uint32_t)(z >> 40) >= threshold;
}

__device__ __forceinline__ float sigmoid_acc(float x) { return 1.f / (1.f + expf(-x)); }

// fp16 activation input of element j of the 8-channel chunk starting at channel c of row m: the BatchNorm output rounded
// to fp16, plus the residual branch's (each rounded, then their sum), as the module tree rounds under autocast
struct Pre {
    float s[8], xh[8], xr[8];
};

__device__ __forceinline__ void load8(const __half* p, float (&v)[8]) {
    const uint4 u = *reinterpret_cast<const uint4*>(p);
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(h[j]);
        v[2 * j] = f.x;
        v[2 * j + 1] = f.y;
    }
}

__device__ __forceinline__ void pre_act(const Bn& a, long long m, int c, Pre& q) {
    float z[8];
    load8(a.z + m * a.ldz + c, z);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        q.xh[j] = (z[j] - a.mean[c + j]) * a.invstd[c + j];
        q.s[j] = round_f16(fmaf(a.gamma[c + j], q.xh[j], a.beta[c + j]));
    }
    if (a.zr) {
        load8(a.zr + m * a.ldzr + c, z);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            q.xr[j] = (z[j] - a.mean_r[c + j]) * a.invstd_r[c + j];
            q.s[j] = round_f16(q.s[j] + round_f16(fmaf(a.gamma_r[c + j], q.xr[j], a.beta_r[c + j])));
        }
    }
}

__device__ __forceinline__ float act_fwd(float s, int act) {
    return act == B200_ACT_RELU ? fmaxf(s, 0.f) : act == B200_ACT_SWISH ? round_f16(s * sigmoid_acc(s)) : s;
}
// g * act'(s); relu selects (0 where s <= 0), as torch's threshold_backward does
__device__ __forceinline__ float act_bwd(float g, float s, int act) {
    if (act == B200_ACT_RELU) return s > 0.f ? g : 0.f;
    if (act == B200_ACT_SWISH) {
        const float sg = sigmoid_acc(s);
        return g * (sg * (1.f + s * (1.f - sg)));
    }
    return g;
}

__device__ __forceinline__ uint32_t drop_threshold(float p) { return (uint32_t)fminf(p * 16777216.f, 16777216.f); }

__global__ void bn_act_fwd_kernel(Bn a, __half* __restrict__ out, long long ldo, long long lpo) {
    const int cw = a.c / 8;
    const long long n8 = a.m * cw;
    const uint32_t thr = drop_threshold(a.p);
    const float scale = 1.f / (1.f - a.p);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
        const long long m = i / cw;
        const int c = (int)(i - m * cw) * 8;
        Pre q;
        pre_act(a, m, c, q);
        uint32_t bits = 0;
        __align__(16) __half o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float v = act_fwd(q.s[j], a.act);
            if (a.mask) {
                const bool k = keep_elem(a.seed, a.unit, m * a.c + c + j, thr);
                bits |= (uint32_t)k << j;
                v = k ? round_f16(v * scale) : 0.f;
            }
            o[j] = __float2half_rn(v);
        }
        if (a.mask) a.mask[i] = (uint8_t)bits;
        const long long n = m / a.t;
        *reinterpret_cast<uint4*>(out + (n * lpo + (m - n * a.t)) * ldo + c) = *reinterpret_cast<const uint4*>(o);
    }
}

// gradient at the activation input: dy (+ dy2) through dropout and the activation
__device__ __forceinline__ void grad_pre(const Bn& a, const __half* dy, long long ldy, const __half* dy2, long long ldy2,
                                         long long m, int c, const Pre& q, float (&g)[8]) {
    load8(dy + m * ldy + c, g);
    if (dy2) {
        float g2[8];
        load8(dy2 + m * ldy2 + c, g2);
#pragma unroll
        for (int j = 0; j < 8; ++j) g[j] += g2[j];
    }
    const uint32_t bits = a.mask ? a.mask[m * (a.c / 8) + c / 8] : 0xffu;
    const float scale = a.mask ? 1.f / (1.f - a.p) : 1.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) g[j] = act_bwd((bits >> j) & 1u ? g[j] * scale : 0.f, q.s[j], a.act);
}

struct BnGrad {
    const __half *dy, *dy2;
    long long ldy, ldy2;
};

// per-slice sums of g, g * xhat and g * xhat_r: 8 channels per thread, 32 threads across 256 channels, BWD_PHASES row
// phases (one warp each), combined in phase order
constexpr int BWD_PHASES = 8;
__global__ void __launch_bounds__(BWD_PHASES * 32) bn_act_bwd_sums_kernel(Bn a, BnGrad d, float* __restrict__ part) {
    __shared__ float red[3][BWD_PHASES][256];
    const int lanec = threadIdx.x % 32, phase = threadIdx.x / 32;
    const int c = blockIdx.x * 256 + lanec * 8;
    const long long r0 = (long long)blockIdx.y * SLICE_ROWS, r1 = std::min<long long>(a.m, r0 + SLICE_ROWS);
    float sg[8], sx[8], sr[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) sg[j] = sx[j] = sr[j] = 0.f;
    if (c < a.c) {
        for (long long m = r0 + phase; m < r1; m += BWD_PHASES) {
            Pre q;
            pre_act(a, m, c, q);
            float g[8];
            grad_pre(a, d.dy, d.ldy, d.dy2, d.ldy2, m, c, q, g);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                sg[j] += g[j];
                sx[j] = fmaf(g[j], q.xh[j], sx[j]);
                if (a.zr) sr[j] = fmaf(g[j], q.xr[j], sr[j]);
            }
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        red[0][phase][lanec * 8 + j] = sg[j];
        red[1][phase][lanec * 8 + j] = sx[j];
        red[2][phase][lanec * 8 + j] = sr[j];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 3 * 256; i += BWD_PHASES * 32) {
        const int w = i / 256, cc = i % 256;
        if (blockIdx.x * 256 + cc >= a.c) continue;
        float v = red[w][0][cc];
        for (int ph = 1; ph < BWD_PHASES; ++ph) v += red[w][ph][cc];
        part[((long long)w * gridDim.y + blockIdx.y) * a.c + blockIdx.x * 256 + cc] = v;
    }
}

// coef [3][C] = sum g / M, sum g xhat / M, sum g xhat_r / M; dgamma, dbeta (and the residual branch's)
__global__ void bn_act_bwd_final_kernel(const float* __restrict__ part, int S, long long M, int C, float* __restrict__ coef,
                                        float* __restrict__ dgamma, float* __restrict__ dbeta, float* __restrict__ dgamma_r,
                                        float* __restrict__ dbeta_r) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double s[3];
    for (int w = 0; w < 3; ++w) {
        double v = 0.0;
        for (int j = 0; j < S; ++j) v += part[((long long)w * S + j) * C + c];
        s[w] = v;
    }
    dbeta[c] = (float)s[0];
    dgamma[c] = (float)s[1];
    if (dgamma_r) {
        dbeta_r[c] = (float)s[0];
        dgamma_r[c] = (float)s[2];
    }
    for (int w = 0; w < 3; ++w) coef[(long long)w * C + c] = (float)(s[w] / (double)M);
}

__global__ void bn_act_bwd_dz_kernel(Bn a, BnGrad d, const float* __restrict__ coef, __half* __restrict__ dz,
                                     __half* __restrict__ dzr, long long ldo, long long lpo) {
    const int cw = a.c / 8;
    const long long n8 = a.m * cw;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
        const long long m = i / cw;
        const int c = (int)(i - m * cw) * 8;
        Pre q;
        pre_act(a, m, c, q);
        float g[8];
        grad_pre(a, d.dy, d.ldy, d.dy2, d.ldy2, m, c, q, g);
        const long long n = m / a.t;
        const long long o = (n * lpo + (m - n * a.t)) * ldo + c;
        __align__(16) __half v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float sg = coef[c + j], sx = coef[a.c + c + j];
            v[j] = __float2half_rn(a.gamma[c + j] * a.invstd[c + j] * (g[j] - sg - q.xh[j] * sx));
        }
        *reinterpret_cast<uint4*>(dz + o) = *reinterpret_cast<const uint4*>(v);
        if (dzr) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float sg = coef[c + j], sr = coef[2 * a.c + c + j];
                v[j] = __float2half_rn(a.gamma_r[c + j] * a.invstd_r[c + j] * (g[j] - sg - q.xr[j] * sr));
            }
            *reinterpret_cast<uint4*>(dzr + o) = *reinterpret_cast<const uint4*>(v);
        }
    }
}

// ------------------------------------------------------------------------------------------------ head
constexpr int NCLS = 5, HEAD_WARPS = 8;

// warp per row: lanes take 8-feature chunks, partial dot products combined by a fixed xor butterfly
__device__ __forceinline__ void head_logits(const __half* x, long long row, int F, const float* ws, int lane, float (&l)[NCLS]) {
#pragma unroll
    for (int c = 0; c < NCLS; ++c) l[c] = 0.f;
    for (int f = lane * 8; f < F; f += 256) {
        float v[8];
        load8(x + row * F + f, v);
#pragma unroll
        for (int c = 0; c < NCLS; ++c)
#pragma unroll
            for (int j = 0; j < 8; ++j) l[c] = fmaf(v[j], ws[c * F + f + j], l[c]);
    }
#pragma unroll
    for (int c = 0; c < NCLS; ++c)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) l[c] += __shfl_xor_sync(0xffffffffu, l[c], o);
}

__global__ void __launch_bounds__(HEAD_WARPS * 32) head_fwd_kernel(const __half* __restrict__ x, long long M, int F,
                                                                    const __half* __restrict__ w, const __half* __restrict__ bias,
                                                                    float* __restrict__ logp) {
    extern __shared__ float ws[];   // [5][F]
    for (int i = threadIdx.x; i < NCLS * F; i += blockDim.x) ws[i] = __half2float(w[i]);
    __syncthreads();
    const int lane = threadIdx.x & 31;
    for (long long row = (long long)blockIdx.x * HEAD_WARPS + threadIdx.x / 32; row < M; row += (long long)gridDim.x * HEAD_WARPS) {
        float l[NCLS];
        head_logits(x, row, F, ws, lane, l);
        float mx = -INFINITY;
#pragma unroll
        for (int c = 0; c < NCLS; ++c) {
            l[c] = round_f16(l[c] + (bias ? __half2float(bias[c]) : 0.f));   // the fp16 logits of the autocast convolution
            mx = fmaxf(mx, l[c]);
        }
        float se = 0.f;
#pragma unroll
        for (int c = 0; c < NCLS; ++c) se += expf(l[c] - mx);
        const float lse = mx + logf(se);
        if (lane < NCLS) {
            float v = l[0];
#pragma unroll
            for (int c = 1; c < NCLS; ++c)
                if (lane == c) v = l[c];
            logp[row * NCLS + lane] = v - lse;
        }
    }
}

// dlogits = g - softmax * sum_c g; dx = dlogits W (fp16); dlogits kept [M][8] fp32 for the weight gradient
__global__ void __launch_bounds__(HEAD_WARPS * 32) head_bwd_dx_kernel(long long M, int F, const __half* __restrict__ w,
                                                                       const float* __restrict__ logp, const float* __restrict__ g,
                                                                       float* __restrict__ dl, __half* __restrict__ dx) {
    extern __shared__ float ws[];
    for (int i = threadIdx.x; i < NCLS * F; i += blockDim.x) ws[i] = __half2float(w[i]);
    __syncthreads();
    const int lane = threadIdx.x & 31;
    for (long long row = (long long)blockIdx.x * HEAD_WARPS + threadIdx.x / 32; row < M; row += (long long)gridDim.x * HEAD_WARPS) {
        float gs = 0.f, d[NCLS];
#pragma unroll
        for (int c = 0; c < NCLS; ++c) gs += g[row * NCLS + c];
#pragma unroll
        for (int c = 0; c < NCLS; ++c) d[c] = g[row * NCLS + c] - expf(logp[row * NCLS + c]) * gs;
        if (lane < 8) {
            float v = 0.f;
#pragma unroll
            for (int c = 0; c < NCLS; ++c)
                if (lane == c) v = d[c];
            dl[row * 8 + lane] = v;
        }
        for (int f = lane * 8; f < F; f += 256) {
            __align__(16) __half v[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float s = 0.f;
#pragma unroll
                for (int c = 0; c < NCLS; ++c) s = fmaf(d[c], ws[c * F + f + j], s);
                v[j] = __float2half_rn(s);
            }
            *reinterpret_cast<uint4*>(dx + row * F + f) = *reinterpret_cast<const uint4*>(v);
        }
    }
}

// per-slice partials [S][5][F + 1] of dW_h (columns < F) and db_h (column F): thread per column, loop over the slice
__global__ void __launch_bounds__(256) head_bwd_w_kernel(const __half* __restrict__ x, long long M, int F,
                                                          const float* __restrict__ dl, float* __restrict__ part) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f > F) return;
    const long long r0 = (long long)blockIdx.y * SLICE_ROWS, r1 = std::min<long long>(M, r0 + SLICE_ROWS);
    float acc[NCLS] = {0.f, 0.f, 0.f, 0.f, 0.f};
    for (long long r = r0; r < r1; ++r) {
        const float v = f < F ? __half2float(x[r * F + f]) : 1.f;
        const float4 d0 = *reinterpret_cast<const float4*>(dl + r * 8);
        const float d4 = dl[r * 8 + 4];
        acc[0] = fmaf(d0.x, v, acc[0]);
        acc[1] = fmaf(d0.y, v, acc[1]);
        acc[2] = fmaf(d0.z, v, acc[2]);
        acc[3] = fmaf(d0.w, v, acc[3]);
        acc[4] = fmaf(d4, v, acc[4]);
    }
#pragma unroll
    for (int c = 0; c < NCLS; ++c) part[((long long)blockIdx.y * NCLS + c) * (F + 1) + f] = acc[c];
}

__global__ void head_bwd_w_final_kernel(const float* __restrict__ part, int S, int F, float* __restrict__ dw, float* __restrict__ db) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= NCLS * (F + 1)) return;
    float s = 0.f;
    for (int j = 0; j < S; ++j) s += part[(long long)j * NCLS * (F + 1) + i];
    const int c = i / (F + 1), f = i % (F + 1);
    if (f < F) dw[c * F + f] = s;
    else if (db) db[c] = s;
}

inline size_t align256(size_t x) { return (x + 255) / 256 * 256; }
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

int check_bn(const b200_bn_act* a) {
    B200_REQUIRE(a, "bn_act: null argument struct");
    B200_REQUIRE(a->m > 1 && a->t > 0 && a->m % a->t == 0, "bn_act: need m > 1 rows, a multiple of t (m=%lld t=%d)", a->m, a->t);
    B200_REQUIRE(a->c > 0 && a->c % 8 == 0 && a->c <= 4096, "bn_act: c must be a multiple of 8 in [8, 4096] (c=%d)", a->c);
    B200_REQUIRE(a->act == B200_ACT_NONE || a->act == B200_ACT_RELU || a->act == B200_ACT_SWISH,
                 "bn_act: activation %d is not supported (none, relu, swish)", a->act);
    B200_REQUIRE(a->p >= 0.f && a->p < 1.f, "bn_act: dropout p must be in [0, 1) (p=%g)", (double)a->p);
    B200_REQUIRE(a->z && a->mean && a->invstd && a->gamma && a->beta, "bn_act: null pointer argument");
    B200_REQUIRE(a->ldz >= a->c && a->ldz % 8 == 0 && aligned16(a->z), "bn_act: z needs ldz %% 8 == 0, ldz >= c, 16-byte alignment");
    if (a->zr) {
        B200_REQUIRE(a->mean_r && a->invstd_r && a->gamma_r && a->beta_r, "bn_act: null residual BatchNorm argument");
        B200_REQUIRE(a->ldzr >= a->c && a->ldzr % 8 == 0 && aligned16(a->zr),
                     "bn_act: zr needs ldzr %% 8 == 0, ldzr >= c, 16-byte alignment");
    }
    B200_REQUIRE(a->p == 0.f || a->mask, "bn_act: dropout p > 0 needs a mask buffer");
    return 0;
}

Bn to_bn(const b200_bn_act* a) {
    Bn b;
    b.m = a->m;
    b.c = a->c;
    b.t = a->t;
    b.act = a->act;
    b.p = a->p;
    b.seed = a->seed;
    b.unit = a->unit;
    b.z = (const __half*)a->z;
    b.ldz = a->ldz;
    b.mean = a->mean;
    b.invstd = a->invstd;
    b.gamma = a->gamma;
    b.beta = a->beta;
    b.zr = (const __half*)a->zr;
    b.ldzr = a->ldzr;
    b.mean_r = a->mean_r;
    b.invstd_r = a->invstd_r;
    b.gamma_r = a->gamma_r;
    b.beta_r = a->beta_r;
    b.mask = a->p > 0.f ? (uint8_t*)a->mask : nullptr;
    return b;
}

int elementwise_grid(long long n8) { return (int)std::max(1LL, std::min(cdiv(n8, 256), 132LL * 16)); }

}  // namespace

extern "C" {

size_t b200_wgrad_gemm_workspace_bytes(long long m, int cout, int k) {
    if (m <= 0 || cout <= 0 || k <= 0) return 0;
    const int s = wgrad_slices(m, cout, k, nullptr);
    return s > 1 ? (size_t)s * cout * k * sizeof(float) : 0;
}

int b200_wgrad_gemm(const void* dz, long long ldz, long long lpz, const void* x, long long ldx, long long m, int cout, int k,
                    int rows_inner, int valid_inner, void* workspace, void* dw, void* stream) {
    B200_REQUIRE(dz && x && dw, "wgrad_gemm: null pointer argument");
    B200_REQUIRE(m > 0 && cout > 0 && k > 0, "wgrad_gemm: bad sizes m=%lld cout=%d k=%d", m, cout, k);
    B200_REQUIRE(cout % 8 == 0 && k % 8 == 0 && ldz % 8 == 0 && ldx % 8 == 0 && ldz >= cout && ldx > 0,
                 "wgrad_gemm: cout (%d), k (%d), ldz (%lld), ldx (%lld) must be multiples of 8, ldz >= cout", cout, k, ldz, ldx);
    B200_REQUIRE(aligned16(dz) && aligned16(x), "wgrad_gemm: dz and x must be 16-byte aligned");
    B200_REQUIRE(rows_inner > 0 && valid_inner > 0 && valid_inner <= rows_inner && m % rows_inner == 0 && lpz >= valid_inner,
                 "wgrad_gemm: bad row map m=%lld rows_inner=%d valid_inner=%d lpz=%lld", m, rows_inner, valid_inner, lpz);
    B200_REQUIRE(cdiv(cout, WG_BM) <= 65535, "wgrad_gemm: cout %d too large", cout);
    int per = 0;
    const int s = wgrad_slices(m, cout, k, &per);
    B200_REQUIRE(s == 1 || workspace, "wgrad_gemm: %d slices need b200_wgrad_gemm_workspace_bytes() of workspace", s);
    cudaStream_t st = (cudaStream_t)stream;
    B200_CHECK_CUDA(cudaFuncSetAttribute(wgrad_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(WgSmem)));
    WgArgs p{(const __half*)dz, ldz, lpz, (const __half*)x, ldx, m, rows_inner, valid_inner, cout, k, per};
    dim3 grid((unsigned)cdiv(k, WG_BN), (unsigned)cdiv(cout, WG_BM), (unsigned)s);
    float* out = s > 1 ? (float*)workspace : (float*)dw;
    wgrad_gemm_kernel<<<grid, WG_THREADS, sizeof(WgSmem), st>>>(p, out);
    B200_CHECK_CUDA(cudaGetLastError());
    if (s > 1) return sum_partials(out, s, (long long)cout * k, (float*)dw, st);
    return 0;
}

size_t b200_depthwise_wgrad_workspace_bytes(int n, int t, int c, int k) {
    if (n <= 0 || t <= 0 || c <= 0 || k <= 0) return 0;
    return (size_t)tap_slices(n, t, nullptr) * c * k * sizeof(float);
}

int b200_depthwise_wgrad(const void* dy, long long ldy, const void* x, long long ldx, int n, int t, int c, int k, void* workspace,
                         void* dw, void* stream) {
    B200_REQUIRE(dy && x && dw && workspace, "depthwise_wgrad: null pointer argument");
    B200_REQUIRE(n > 0 && t > 0, "depthwise_wgrad: bad sizes n=%d t=%d", n, t);
    B200_REQUIRE(c >= 256 && c <= 512 && c % 8 == 0 && k % 2 == 1 && k <= DW_KMAX,
                 "depthwise_wgrad: c must be a multiple of 8 in [256, 512] and k odd <= %d (c=%d k=%d)", DW_KMAX, c, k);
    B200_REQUIRE(ldy >= c && ldx >= c, "depthwise_wgrad: ldy (%lld) and ldx (%lld) must be >= c", ldy, ldx);
    int per = 0;
    const int s = tap_slices(n, t, &per);
    dim3 grid((unsigned)cdiv(c, TAP_CH), (unsigned)s);
    launch_tap_kj<false, TAP_KJ_MAX>((int)cdiv(k, TAP_GROUPS), grid, (cudaStream_t)stream, (const __half*)dy, ldy,
                                     (const __half*)x, ldx, n, t, 0, c, k, 1, per, (float*)workspace);
    B200_CHECK_CUDA(cudaGetLastError());
    return sum_partials((const float*)workspace, s, (long long)c * k, (float*)dw, (cudaStream_t)stream);
}

size_t b200_conv_first_wgrad_workspace_bytes(int n, int t, int c, int k) { return b200_depthwise_wgrad_workspace_bytes(n, t, c, k); }

int b200_conv_first_wgrad(const void* dz, long long ldz, const void* x, int n, int l, int c, int k, int stride, void* workspace,
                          void* dw, void* stream) {
    B200_REQUIRE(dz && x && dw && workspace, "conv_first_wgrad: null pointer argument");
    B200_REQUIRE(n > 0 && l > 0, "conv_first_wgrad: bad sizes n=%d l=%d", n, l);
    B200_REQUIRE(c > 0 && c <= 512 && c % 8 == 0 && k % 2 == 1 && k <= FC_KMAX && stride >= 1 && stride <= FC_SMAX && ldz >= c,
                 "conv_first_wgrad: needs c %% 8 == 0 <= 512, odd k <= %d, 1 <= stride <= %d, ldz >= c (c=%d k=%d stride=%d)",
                 FC_KMAX, FC_SMAX, c, k, stride);
    const int t = (l - 1) / stride + 1;
    int per = 0;
    const int s = tap_slices(n, t, &per);
    dim3 grid((unsigned)cdiv(c, TAP_CH), (unsigned)s);
    launch_tap_kj<true, (FC_KMAX + TAP_GROUPS - 1) / TAP_GROUPS>((int)cdiv(k, TAP_GROUPS), grid, (cudaStream_t)stream,
                                                                 (const __half*)dz, ldz, (const __half*)x, l, n, t, l, c, k,
                                                                 stride, per, (float*)workspace);
    B200_CHECK_CUDA(cudaGetLastError());
    return sum_partials((const float*)workspace, s, (long long)c * k, (float*)dw, (cudaStream_t)stream);
}

size_t b200_bn_stats_workspace_bytes(long long m, int c) {
    if (m <= 0 || c <= 0) return 0;
    return 2 * align256((size_t)cdiv(m, SLICE_ROWS) * c * sizeof(float));
}

int b200_bn_stats(const void* z, long long ldz, long long m, int c, float eps, float momentum, void* workspace, void* mean,
                  void* invstd, void* running_mean, void* running_var, void* stream) {
    B200_REQUIRE(z && workspace && mean && invstd, "bn_stats: null pointer argument");
    B200_REQUIRE(m > 1 && c > 0 && c % 2 == 0 && ldz >= c && ldz % 2 == 0, "bn_stats: bad sizes m=%lld c=%d ldz=%lld", m, c, ldz);
    B200_REQUIRE((reinterpret_cast<uintptr_t>(z) & 3) == 0, "bn_stats: z must be 4-byte aligned (it is read as half2)");
    B200_REQUIRE((running_mean == nullptr) == (running_var == nullptr), "bn_stats: running_mean and running_var go together");
    B200_REQUIRE(cdiv(m, SLICE_ROWS) <= 65535, "bn_stats: at most %d rows", 65535 * SLICE_ROWS);
    const int s = (int)cdiv(m, SLICE_ROWS);
    float* pmean = (float*)workspace;
    float* pm2 = (float*)((unsigned char*)workspace + align256((size_t)s * c * sizeof(float)));
    cudaStream_t st = (cudaStream_t)stream;
    bn_stats_partial_kernel<<<dim3((unsigned)cdiv(c, 2 * CH_THREADS), (unsigned)s), CH_THREADS, 0, st>>>((const __half*)z, ldz, m, c,
                                                                                                      pmean, pm2);
    B200_CHECK_CUDA(cudaGetLastError());
    bn_stats_final_kernel<<<(unsigned)cdiv(c, 128), 128, 0, st>>>(pmean, pm2, s, m, c, eps, momentum, (float*)mean, (float*)invstd,
                                                                  (float*)running_mean, (float*)running_var);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int b200_bn_act_fwd(const b200_bn_act* args, void* out, long long ldo, long long lpo, void* stream) {
    if (int rc = check_bn(args)) return rc;
    B200_REQUIRE(out && ldo >= args->c && ldo % 8 == 0 && aligned16(out) && lpo >= args->t,
                 "bn_act_fwd: out needs ldo %% 8 == 0, ldo >= c, lpo >= t, 16-byte alignment");
    const Bn a = to_bn(args);
    const long long n8 = a.m * (a.c / 8);
    bn_act_fwd_kernel<<<elementwise_grid(n8), 256, 0, (cudaStream_t)stream>>>(a, (__half*)out, ldo, lpo);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

size_t b200_bn_act_bwd_workspace_bytes(long long m, int c) {
    if (m <= 0 || c <= 0) return 0;
    return align256((size_t)3 * cdiv(m, SLICE_ROWS) * c * sizeof(float)) + align256((size_t)3 * c * sizeof(float));
}

int b200_bn_act_bwd(const b200_bn_act* args, const void* dy, long long ldy, const void* dy2, long long ldy2, void* workspace,
                    void* dgamma, void* dbeta, void* dgamma_r, void* dbeta_r, void* dz, void* dzr, long long ldo, long long lpo,
                    void* stream) {
    if (int rc = check_bn(args)) return rc;
    B200_REQUIRE(dy && workspace && dgamma && dbeta && dz, "bn_act_bwd: null pointer argument");
    B200_REQUIRE(ldy >= args->c && ldy % 8 == 0 && aligned16(dy), "bn_act_bwd: dy needs ldy %% 8 == 0, ldy >= c, 16-byte alignment");
    B200_REQUIRE(!dy2 || (ldy2 >= args->c && ldy2 % 8 == 0 && aligned16(dy2)),
                 "bn_act_bwd: dy2 needs ldy2 %% 8 == 0, ldy2 >= c, 16-byte alignment");
    B200_REQUIRE(!args->zr || (dgamma_r && dbeta_r && dzr), "bn_act_bwd: the residual branch needs dgamma_r, dbeta_r and dzr");
    B200_REQUIRE(ldo >= args->c && ldo % 8 == 0 && lpo >= args->t && aligned16(dz) && (!dzr || aligned16(dzr)),
                 "bn_act_bwd: dz needs ldo %% 8 == 0, ldo >= c, lpo >= t, 16-byte alignment");
    B200_REQUIRE(cdiv(args->m, SLICE_ROWS) <= 65535, "bn_act_bwd: at most %d rows", 65535 * SLICE_ROWS);
    const Bn a = to_bn(args);
    const BnGrad d{(const __half*)dy, (const __half*)dy2, ldy, ldy2};
    const int s = (int)cdiv(a.m, SLICE_ROWS);
    float* part = (float*)workspace;
    float* coef = (float*)((unsigned char*)workspace + align256((size_t)3 * s * a.c * sizeof(float)));
    cudaStream_t st = (cudaStream_t)stream;
    bn_act_bwd_sums_kernel<<<dim3((unsigned)cdiv(a.c, 256), (unsigned)s), BWD_PHASES * 32, 0, st>>>(a, d, part);
    B200_CHECK_CUDA(cudaGetLastError());
    bn_act_bwd_final_kernel<<<(unsigned)cdiv(a.c, 128), 128, 0, st>>>(part, s, a.m, a.c, coef, (float*)dgamma, (float*)dbeta,
                                                                      a.zr ? (float*)dgamma_r : nullptr, (float*)dbeta_r);
    B200_CHECK_CUDA(cudaGetLastError());
    bn_act_bwd_dz_kernel<<<elementwise_grid(a.m * (a.c / 8)), 256, 0, st>>>(a, d, coef, (__half*)dz, a.zr ? (__half*)dzr : nullptr,
                                                                            ldo, lpo);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int b200_ctc_head_train_fwd(const void* x, long long m, int f, const void* w, const void* bias, void* logp, void* stream) {
    B200_REQUIRE(x && w && logp, "ctc_head_train_fwd: null pointer argument");
    B200_REQUIRE(m > 0 && f >= 8 && f <= 2048 && f % 8 == 0 && aligned16(x),
                 "ctc_head_train_fwd: m > 0, f a multiple of 8 in [8, 2048], x 16-byte aligned (m=%lld f=%d)", m, f);
    const unsigned grid = (unsigned)std::min<long long>(cdiv(m, HEAD_WARPS), 132LL * 8);
    head_fwd_kernel<<<grid, HEAD_WARPS * 32, NCLS * f * sizeof(float), (cudaStream_t)stream>>>(
        (const __half*)x, m, f, (const __half*)w, (const __half*)bias, (float*)logp);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

size_t b200_ctc_head_bwd_workspace_bytes(long long m, int f) {
    if (m <= 0 || f <= 0) return 0;
    return align256((size_t)m * 8 * sizeof(float)) + align256((size_t)cdiv(m, SLICE_ROWS) * NCLS * (f + 1) * sizeof(float));
}

int b200_ctc_head_bwd(const void* x, long long m, int f, const void* w, const void* logp, const void* g, void* workspace, void* dw,
                      void* db, void* dx, void* stream) {
    B200_REQUIRE(x && w && logp && g && workspace && dw && dx, "ctc_head_bwd: null pointer argument");
    B200_REQUIRE(m > 0 && f >= 8 && f <= 2048 && f % 8 == 0 && aligned16(x) && aligned16(dx),
                 "ctc_head_bwd: m > 0, f a multiple of 8 in [8, 2048], x and dx 16-byte aligned (m=%lld f=%d)", m, f);
    B200_REQUIRE(cdiv(m, SLICE_ROWS) <= 65535, "ctc_head_bwd: at most %d rows", 65535 * SLICE_ROWS);
    float* dl = (float*)workspace;
    float* part = (float*)((unsigned char*)workspace + align256((size_t)m * 8 * sizeof(float)));
    const int s = (int)cdiv(m, SLICE_ROWS);
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned grid = (unsigned)std::min<long long>(cdiv(m, HEAD_WARPS), 132LL * 8);
    head_bwd_dx_kernel<<<grid, HEAD_WARPS * 32, NCLS * f * sizeof(float), st>>>(m, f, (const __half*)w, (const float*)logp,
                                                                                (const float*)g, dl, (__half*)dx);
    B200_CHECK_CUDA(cudaGetLastError());
    head_bwd_w_kernel<<<dim3((unsigned)cdiv(f + 1, 256), (unsigned)s), 256, 0, st>>>((const __half*)x, m, f, dl, part);
    B200_CHECK_CUDA(cudaGetLastError());
    head_bwd_w_final_kernel<<<(unsigned)cdiv(NCLS * (f + 1), 128), 128, 0, st>>>(part, s, f, (float*)dw, (float*)db);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // extern "C"
