// Depthwise Conv1d of the QuartzNet CTC models (TCSConv1d.depthwise, bonito/ctc/model.py:90-121): per channel c,
//     y[n][t][c] = sum_k w[c][k] * x[n][t + k - K/2][c]      (stride 1, dilation 1, zero padding at each chunk's ends)
// on channels-last fp16 rows with row pitches, so the kernel reads from and writes into column ranges of wider buffers
// (the [depthwise out | block input] operand of a residual block's fused pointwise + residual GEMM).  Accumulation is fp32,
// rounded once to fp16: the rounding point of the reference's half Conv1d.
//
// One CTA computes DW_TT frames x DW_CC channels of one chunk.  The (DW_TT + KP) x DW_CC input tile is staged in shared
// memory with zero-filling cp.async (rows outside the chunk and channels past C read as zeros, so the inner loop has no
// halo rows and no bounds branches); the taps are padded with zero weights to KP, a multiple of DW_F.  A thread owns one
// channel pair and DW_F consecutive frames and slides a register window over the rows: per block of DW_F taps it loads
// DW_F new rows (one half2 each) and DW_F weight pairs for 2 * DW_F * DW_F FMAs.
#include "common.cuh"

namespace {

constexpr int DW_THREADS = 256;           // 8 warps
constexpr int DW_CC = 64;                 // channels per CTA: one warp covers 32 channel pairs
constexpr int DW_F = 8;                   // frames per thread (register window) and taps per unrolled block
constexpr int DW_TT = (DW_THREADS / 32) * DW_F;   // frames per CTA

__global__ void __launch_bounds__(DW_THREADS)
depthwise_kernel(const __half* __restrict__ x, long long ldx, const __half* __restrict__ w, __half* __restrict__ y,
                 long long ldy, int T, int C, int K, int KP) {
    extern __shared__ __align__(16) unsigned char dw_smem[];
    float2* ws = reinterpret_cast<float2*>(dw_smem);                          // [KP][DW_CC / 2]
    __half2* xs = reinterpret_cast<__half2*>(ws + KP * (DW_CC / 2));         // [DW_TT + KP][DW_CC / 2]
    const int rows = DW_TT + KP;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int t0 = blockIdx.x * DW_TT, c0 = blockIdx.y * DW_CC, n = blockIdx.z;
    const int P = K / 2;

    // input tile: row r holds frame t0 - P + r; 8 channels (16 bytes) per cp.async
    const __half* xn = x + (long long)n * T * ldx;
    for (int i = tid; i < rows * (DW_CC / 8); i += DW_THREADS) {
        const int r = i >> 3, q = i & 7;
        const int t = t0 - P + r, c = c0 + 8 * q;
        const bool valid = t >= 0 && t < T && c < C;
        const __half* src = valid ? xn + (long long)t * ldx + c : x;
        cp_async_16(reinterpret_cast<__half*>(xs + r * (DW_CC / 2)) + 8 * q, src, valid);
    }
    cp_async_commit();
    for (int i = tid; i < KP * (DW_CC / 2); i += DW_THREADS) {
        const int k = i / (DW_CC / 2), p = i % (DW_CC / 2), c = c0 + 2 * p;
        float2 v = make_float2(0.f, 0.f);
        if (k < K && c < C) v = make_float2(__half2float(w[(long long)c * K + k]), __half2float(w[(long long)(c + 1) * K + k]));
        ws[i] = v;
    }
    cp_async_wait<0>();
    __syncthreads();

    const int f0 = warp * DW_F;
    const __half2* xc = xs + lane;
    const float2* wc = ws + lane;
    float2 acc[DW_F], win[DW_F];
#pragma unroll
    for (int j = 0; j < DW_F; ++j) {
        acc[j] = make_float2(0.f, 0.f);
        win[j] = __half22float2(xc[(f0 + j) * (DW_CC / 2)]);
    }
#pragma unroll 2
    for (int kb = 0; kb < KP; kb += DW_F) {
        float2 nxt[DW_F];
#pragma unroll
        for (int j = 0; j < DW_F; ++j) nxt[j] = __half22float2(xc[(f0 + kb + DW_F + j) * (DW_CC / 2)]);
#pragma unroll
        for (int d = 0; d < DW_F; ++d) {
            const float2 wv = wc[(kb + d) * (DW_CC / 2)];
#pragma unroll
            for (int j = 0; j < DW_F; ++j) {
                const float2 xv = (j + d < DW_F) ? win[j + d] : nxt[j + d - DW_F];
                acc[j].x = fmaf(wv.x, xv.x, acc[j].x);
                acc[j].y = fmaf(wv.y, xv.y, acc[j].y);
            }
        }
#pragma unroll
        for (int j = 0; j < DW_F; ++j) win[j] = nxt[j];
    }

    const int c = c0 + 2 * lane;
    if (c >= C) return;
    __half* yn = y + (long long)n * T * ldy + c;
#pragma unroll
    for (int j = 0; j < DW_F; ++j) {
        const int t = t0 + f0 + j;
        if (t < T) *reinterpret_cast<__half2*>(yn + (long long)t * ldy) = __floats2half2_rn(acc[j].x, acc[j].y);
    }
}

bool supported_taps(int K) {
    switch (K) {
        case 5: case 9: case 31: case 33: case 39: case 51: case 63: case 67: case 75: case 87: case 115: case 123: return true;
        default: return false;
    }
}

}  // namespace

int launch_depthwise(const __half* x, long long ldx, const __half* w, __half* y, long long ldy, int N, int T, int C, int K,
                     cudaStream_t stream) {
    B200_REQUIRE(supported_taps(K) && C >= 256 && C <= 512 && C % 8 == 0,
                 "depthwise: unsupported shape C=%d K=%d (C in [256, 512], C %% 8 == 0; K one of 5, 9, 31, 33, 39, 51, 63, "
                 "67, 75, 87, 115, 123)", C, K);
    B200_REQUIRE(ldx % 8 == 0 && ldy % 8 == 0 && ldx >= C && ldy >= C && ((uintptr_t)x & 15) == 0 && ((uintptr_t)y & 3) == 0,
                 "depthwise: pitches must be multiples of 8 and >= C, x 16-byte aligned (ldx=%lld ldy=%lld)", ldx, ldy);
    const int KP = (K + DW_F - 1) / DW_F * DW_F;
    const size_t smem = (size_t)KP * (DW_CC / 2) * sizeof(float2) + (size_t)(DW_TT + KP) * (DW_CC / 2) * sizeof(__half2);
    // the largest tile (K = 123) needs 56 KB; the attribute belongs to the current device, so it is set on every launch
    B200_CHECK_CUDA(cudaFuncSetAttribute(depthwise_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    dim3 grid((T + DW_TT - 1) / DW_TT, (C + DW_CC - 1) / DW_CC, N);
    depthwise_kernel<<<grid, DW_THREADS, smem, stream>>>(x, ldx, w, y, ldy, T, C, K, KP);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}
