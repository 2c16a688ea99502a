// Fused conv stem of the LSTM-CRF encoder: Conv1d(1->C1,k=K1,'same') + act, then
// Conv1d(C1->C2,k=K2,'same') + act, written channels-last into a zero-padded buffer
//     out[n][PADL + l][c]   (l in [0,L), c in [0,C2)), Lp rows per chunk
// so that the strided conv that follows (k19 s6 in hac) is a plain GEMM over overlapping rows.
// The 164 MB (hac, batch 512) conv1 activation of the reference never reaches HBM.
// Reference semantics: bonito/nn.py:221-241 (Conv1d -> folded BN -> activation); the fp16
// rounding points of the reference's half-precision path are kept (conv output, then activation).
#include <stdlib.h>

#include "common.cuh"

namespace {

constexpr int TL = 256;  // output positions per CTA

template <int C1, int K1, int C2, int K2>
__global__ void __launch_bounds__(TL)
conv_stem_kernel(const __half* __restrict__ x, int L, const __half* __restrict__ w1, const __half* __restrict__ b1,
                 int act1, const __half* __restrict__ w2, const __half* __restrict__ b2, int act2,
                 __half* __restrict__ out, int Lp, int padl, float lo1, float hi1, float lo2, float hi2) {
    constexpr int P1 = K1 / 2, P2 = K2 / 2;
    constexpr int NA1 = TL + K2 - 1;        // conv1 outputs needed by this tile
    constexpr int NX = NA1 + K1 - 1;        // input samples needed
    __shared__ float xs[NX];
    __shared__ float a1s[C1][NA1];
    __shared__ __align__(16) float w2s[C1 * K2][C2];
    __shared__ float w1s[K1][C1];
    __shared__ float b1s[C1], b2s[C2];

    const int tid = threadIdx.x;
    const int n = blockIdx.y;
    const int p0 = blockIdx.x * TL;   // first padded position of the tile
    const int l0 = p0 - padl;         // its signal coordinate
    const __half* xn = x + (long long)n * L;

    for (int i = tid; i < NX; i += TL) {
        int l = l0 - P2 - P1 + i;
        xs[i] = (l >= 0 && l < L) ? __half2float(xn[l]) : 0.f;
    }
    for (int i = tid; i < C1 * K2 * C2; i += TL) {
        int co = i % C2, ck = i / C2;  // ck = cin*K2 + tap
        int cin = ck / K2, tap = ck % K2;
        w2s[ck][co] = __half2float(w2[(co * C1 + cin) * K2 + tap]);
    }
    for (int i = tid; i < K1 * C1; i += TL) {
        int c = i % C1, k = i / C1;
        w1s[k][c] = __half2float(w1[c * K1 + k]);
    }
    if (tid < C1) b1s[tid] = b1 ? __half2float(b1[tid]) : 0.f;
    if (tid < C2) b2s[tid] = b2 ? __half2float(b2[tid]) : 0.f;
    __syncthreads();

    for (int i = tid; i < NA1; i += TL) {
        int l = l0 - P2 + i;
        bool in = (l >= 0 && l < L);
        float xv[K1];
#pragma unroll
        for (int k = 0; k < K1; ++k) xv[k] = xs[i + k];
#pragma unroll
        for (int c = 0; c < C1; ++c) {
            float acc = b1s[c];
#pragma unroll
            for (int k = 0; k < K1; ++k) acc = fmaf(w1s[k][c], xv[k], acc);
            a1s[c][i] = in ? apply_act_f16(acc, act1, lo1, hi1) : 0.f;
        }
    }
    __syncthreads();

    const int p = p0 + tid;
    if (p >= Lp) return;
    const int l = p - padl;
    __half* dst = out + ((long long)n * Lp + p) * C2;
    if (l < 0 || l >= L) {
#pragma unroll
        for (int c = 0; c < C2; c += 8) *reinterpret_cast<uint4*>(dst + c) = make_uint4(0, 0, 0, 0);
        return;
    }
    float acc[C2];
#pragma unroll
    for (int c = 0; c < C2; ++c) acc[c] = b2s[c];
#pragma unroll 4
    for (int cin = 0; cin < C1; ++cin) {
#pragma unroll
        for (int tap = 0; tap < K2; ++tap) {
            float v = a1s[cin][tid + tap];
            const float4* wrow = reinterpret_cast<const float4*>(w2s[cin * K2 + tap]);
#pragma unroll
            for (int q = 0; q < C2 / 4; ++q) {
                float4 w = wrow[q];
                acc[4 * q + 0] = fmaf(w.x, v, acc[4 * q + 0]);
                acc[4 * q + 1] = fmaf(w.y, v, acc[4 * q + 1]);
                acc[4 * q + 2] = fmaf(w.z, v, acc[4 * q + 2]);
                acc[4 * q + 3] = fmaf(w.w, v, acc[4 * q + 3]);
            }
        }
    }
#pragma unroll
    for (int c = 0; c < C2; c += 8) {
        __half2 h[4];
#pragma unroll
        for (int q = 0; q < 4; ++q)
            h[q] = __floats2half2_rn(apply_act_f16(acc[c + 2 * q], act2, lo2, hi2),
                                     apply_act_f16(acc[c + 2 * q + 1], act2, lo2, hi2));
        *reinterpret_cast<uint4*>(dst + c) = *reinterpret_cast<uint4*>(h);
    }
}

// ---- tensor-core variant for the 16 -> 16 (k5) second convolution ---------------------------------------------------
// conv2 is 94 % of the stem's arithmetic (16 x 5 x 16 FMAs per position).  Here it is an implicit GEMM on mma.sync
// (m16n8k16, fp16 x fp16 -> fp32): the conv1 activations of the tile are kept channels-last in shared memory, so the A
// fragment of tap k for 16 consecutive positions is one ldmatrix.x4 of rows p+k .. p+k+15 (48-byte row pitch: conflict
// free), and the ten B fragments (5 taps x 2 halves of the output channels) live in registers.  Same rounding points as
// the FMA kernel (conv1 output and activation rounded to fp16, conv2 accumulates in fp32, output rounded, activation,
// rounded); the accumulation order differs, as it does in any GEMM.
constexpr int A1_PITCH = 24;   // halfs per conv1 position in shared memory (16 used)
constexpr int TC_THREADS = TL + 32;   // eight GEMM warps + one more so that the TL + 4 conv1 positions take a single pass

__global__ void __launch_bounds__(TC_THREADS, 2)
conv_stem_tc_kernel(const __half* __restrict__ x, int L, const __half* __restrict__ w1, const __half* __restrict__ b1,
                    int act1, const __half* __restrict__ w2, const __half* __restrict__ b2, int act2,
                    __half* __restrict__ out, int Lp, int padl, float lo1, float hi1, float lo2, float hi2) {
    constexpr int C1 = 16, K1 = 5, C2 = 16, K2 = 5, P1 = K1 / 2, P2 = K2 / 2;
    constexpr int NA1 = TL + K2 - 1, NX = NA1 + K1 - 1;
    __shared__ float xs[NX];
    __shared__ float w1s[K1][C1];
    __shared__ float b1s[C1];
    __shared__ __align__(16) __half a1h[NA1][A1_PITCH];
    __shared__ __align__(16) __half stage[TL / 32][32][C2];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = blockIdx.y;
    const int p0 = blockIdx.x * TL;
    const int l0 = p0 - padl;
    const __half* xn = x + (long long)n * L;

    for (int i = tid; i < NX; i += TC_THREADS) {
        const int l = l0 - P2 - P1 + i;
        xs[i] = (l >= 0 && l < L) ? __half2float(xn[l]) : 0.f;
    }
    for (int i = tid; i < K1 * C1; i += TC_THREADS) w1s[i / C1][i % C1] = __half2float(w1[(i % C1) * K1 + i / C1]);
    if (tid < C1) b1s[tid] = b1 ? __half2float(b1[tid]) : 0.f;

    __syncthreads();

    // conv1 (1 -> 16, k5) + activation, channels-last fp16
    for (int i = tid; i < NA1; i += TC_THREADS) {
        const int l = l0 - P2 + i;
        const bool in = (l >= 0 && l < L);
        float xv[K1];
#pragma unroll
        for (int k = 0; k < K1; ++k) xv[k] = xs[i + k];
        __half2 h[C1 / 2];
#pragma unroll
        for (int c = 0; c < C1; c += 2) {
            float acc0 = b1s[c], acc1 = b1s[c + 1];
#pragma unroll
            for (int k = 0; k < K1; ++k) {
                acc0 = fmaf(w1s[k][c], xv[k], acc0);
                acc1 = fmaf(w1s[k][c + 1], xv[k], acc1);
            }
            h[c / 2] = in ? __floats2half2_rn(apply_act_f16(acc0, act1, lo1, hi1), apply_act_f16(acc1, act1, lo1, hi1))
                          : __floats2half2_rn(0.f, 0.f);
        }
        *reinterpret_cast<uint4*>(&a1h[i][0]) = *reinterpret_cast<const uint4*>(&h[0]);
        *reinterpret_cast<uint4*>(&a1h[i][8]) = *reinterpret_cast<const uint4*>(&h[4]);
    }
    // B fragments: B[k = cin][n = cout] = w2[cout][cin][tap]; b0 holds k = 2q, 2q+1, b1 holds k = 2q+8, 2q+9 for n = g
    const int g = lane >> 2, q = lane & 3;
    uint32_t bfrag[K2][2][2];
#pragma unroll
    for (int tap = 0; tap < K2; ++tap)
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
            const __half* wr = w2 + (size_t)(nt * 8 + g) * C1 * K2 + tap;
#pragma unroll
            for (int hk = 0; hk < 2; ++hk) {
                const __half2 v = __halves2half2(wr[(2 * q + 8 * hk) * K2], wr[(2 * q + 8 * hk + 1) * K2]);
                bfrag[tap][nt][hk] = *reinterpret_cast<const uint32_t*>(&v);
            }
        }
    float bias[2][2];
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
        bias[nt][0] = b2 ? __half2float(b2[nt * 8 + 2 * q]) : 0.f;
        bias[nt][1] = b2 ? __half2float(b2[nt * 8 + 2 * q + 1]) : 0.f;
    }
    __syncthreads();

    // conv2 as implicit GEMM: warp w owns output positions [32w, 32w + 32) of the tile
    if (warp >= TL / 32) return;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
        const int pb = warp * 32 + mt * 16;
        float acc[2][4];
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
            acc[nt][0] = acc[nt][2] = bias[nt][0];
            acc[nt][1] = acc[nt][3] = bias[nt][1];
        }
#pragma unroll
        for (int tap = 0; tap < K2; ++tap) {
            uint32_t a[4];
            ldmatrix_x4(a[0], a[1], a[2], a[3],
                        smem_u32(&a1h[pb + tap + (lane & 7) + 8 * ((lane >> 3) & 1)][8 * (lane >> 4)]));
            mma_16816(acc[0], a, bfrag[tap][0][0], bfrag[tap][0][1]);
            mma_16816(acc[1], a, bfrag[tap][1][0], bfrag[tap][1][1]);
        }
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
            const __half2 lo = __floats2half2_rn(apply_act_f16(acc[nt][0], act2, lo2, hi2), apply_act_f16(acc[nt][1], act2, lo2, hi2));
            const __half2 hi = __floats2half2_rn(apply_act_f16(acc[nt][2], act2, lo2, hi2), apply_act_f16(acc[nt][3], act2, lo2, hi2));
            *reinterpret_cast<__half2*>(&stage[warp][mt * 16 + g][nt * 8 + 2 * q]) = lo;
            *reinterpret_cast<__half2*>(&stage[warp][mt * 16 + g + 8][nt * 8 + 2 * q]) = hi;
        }
    }
    __syncwarp();
    // 32 positions x 32 B of this warp, contiguous in the output: two 16-byte pieces per lane
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int idx = lane + 32 * i, pos = idx >> 1, half = idx & 1;
        const int p = p0 + warp * 32 + pos;
        if (p < Lp) {
            const int l = p - padl;
            uint4 v = make_uint4(0, 0, 0, 0);
            if (l >= 0 && l < L) v = *reinterpret_cast<const uint4*>(&stage[warp][pos][half * 8]);
            *reinterpret_cast<uint4*>(out + ((long long)n * Lp + p) * C2 + half * 8) = v;
        }
    }
}

}  // namespace

int launch_conv_stem(const __half* x, int N, int L, int C1, int K1, const __half* w1, const __half* b1, int act1,
                     int C2, int K2, const __half* w2, const __half* b2, int act2, __half* out, int Lp, int padl,
                     float lo1, float hi1, float lo2, float hi2, cudaStream_t stream) {
    B200_REQUIRE(N <= 65535, "conv_stem: at most 65535 chunks per call (n=%d): the chunk index is gridDim.y", N);
    dim3 grid((Lp + TL - 1) / TL, N);
    const char* impl = getenv("B200_STEM_IMPL");   // "fma": the CUDA-core kernel for every shape
    if (C1 == 16 && K1 == 5 && C2 == 16 && K2 == 5 && !(impl && impl[0] == 'f')) {
        conv_stem_tc_kernel<<<grid, TC_THREADS, 0, stream>>>(x, L, w1, b1, act1, w2, b2, act2, out, Lp, padl, lo1, hi1, lo2, hi2);
        B200_CHECK_CUDA(cudaGetLastError());
        return 0;
    }
#define STEM_CASE(c1, k1, c2, k2)                                                                         \
    if (C1 == c1 && K1 == k1 && C2 == c2 && K2 == k2) {                                                   \
        conv_stem_kernel<c1, k1, c2, k2><<<grid, TL, 0, stream>>>(x, L, w1, b1, act1, w2, b2, act2, out,  \
                                                                  Lp, padl, lo1, hi1, lo2, hi2);          \
        B200_CHECK_CUDA(cudaGetLastError());                                                              \
        return 0;                                                                                         \
    }
    STEM_CASE(16, 5, 16, 5)  // v4.x / v5.x fast, hac, sup LSTM models
    STEM_CASE(4, 5, 16, 5)   // old-style rnn_encoder (bonito/crf/model.py:150-162)
#undef STEM_CASE
    b200_set_error("conv_stem: unsupported shape 1->%d (k%d) -> %d (k%d)", C1, K1, C2, K2);
    return -2;
}
