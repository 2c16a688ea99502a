// Kernels of the QuartzNet CTC models (bonito/ctc/model.py) that are not depthwise convolutions or GEMMs:
//   conv_first_ex   the C1 block: Conv1d(1 -> C, k, stride s, pad k/2) with its BatchNorm folded in + activation, written
//                   channels-last with a row pitch (straight into the right-hand columns of the next block's
//                   [depthwise out | block input] buffer)
//   ctc_head        Decoder: Conv1d(F -> 5, k1, bias) -> log_softmax, plus the per-frame argmax of the greedy decode
#include "common.cuh"

namespace {

// ------------------------------------------------------------------------------------------------ conv_first_ex
constexpr int CFX_THREADS = 128;   // output rows per CTA
constexpr int CFX_CC = 64;         // channels per CTA

__global__ void __launch_bounds__(CFX_THREADS)
conv_first_ex_kernel(const __half* __restrict__ x, int L, const __half* __restrict__ w, const __half* __restrict__ bias,
                     int C, int K, int S, int T, int act, float lo, float hi, __half* __restrict__ out, long long ldo, int Lp,
                     int padl) {
    extern __shared__ float cfx_smem[];
    float* ws = cfx_smem;                 // [K][CFX_CC]
    float* bs = ws + K * CFX_CC;          // [CFX_CC]
    float* xs = bs + CFX_CC;              // [(CFX_THREADS - 1) * S + K]
    const int tid = threadIdx.x, n = blockIdx.z, c0 = blockIdx.y * CFX_CC;
    const int p0 = blockIdx.x * CFX_THREADS, P = K / 2;
    const int nc = min(CFX_CC, C - c0);
    for (int i = tid; i < K * CFX_CC; i += CFX_THREADS) {
        const int k = i / CFX_CC, c = i % CFX_CC;
        ws[i] = c < nc ? __half2float(w[(c0 + c) * K + k]) : 0.f;
    }
    for (int i = tid; i < CFX_CC; i += CFX_THREADS) bs[i] = (bias && i < nc) ? __half2float(bias[c0 + i]) : 0.f;
    // sample of row p, tap k: (p - padl) * S - P + k
    const int nx = (CFX_THREADS - 1) * S + K;
    const long long l0 = (long long)(p0 - padl) * S - P;
    for (int i = tid; i < nx; i += CFX_THREADS) {
        const long long l = l0 + i;
        xs[i] = (l >= 0 && l < L) ? __half2float(x[(size_t)n * L + l]) : 0.f;
    }
    __syncthreads();
    const int p = p0 + tid;
    if (p >= Lp) return;
    const int t = p - padl;
    const bool in = t >= 0 && t < T;
    __half* dst = out + ((size_t)n * Lp + p) * ldo + c0;
    const float* xv = xs + tid * S;
    for (int cg = 0; cg < nc; cg += 8) {
        float acc[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = bs[cg + e];
        for (int k = 0; k < K; ++k) {
            const float v = xv[k];
            const float* wk = ws + k * CFX_CC + cg;
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[e] = fmaf(wk[e], v, acc[e]);
        }
        __half2 h[4];
#pragma unroll
        for (int q = 0; q < 4; ++q)
            h[q] = in ? __floats2half2_rn(apply_act_f16(acc[2 * q], act, lo, hi), apply_act_f16(acc[2 * q + 1], act, lo, hi))
                      : __floats2half2_rn(0.f, 0.f);
        *reinterpret_cast<uint4*>(dst + cg) = *reinterpret_cast<const uint4*>(h);
    }
}

// ------------------------------------------------------------------------------------------------ ctc_head
constexpr int HEAD_THREADS = 256;
constexpr int NCLS = 5;

// LPR lanes per row, 32 / LPR rows per warp and step; lane `sub` of a row reads the 8-feature groups sub, sub + LPR, ...
template <int LPR>
__global__ void __launch_bounds__(HEAD_THREADS)
ctc_head_kernel(const __half* __restrict__ x, long long M, int F, const __half* __restrict__ w, const __half* __restrict__ bias,
                __half* __restrict__ logp, uint8_t* __restrict__ labels, float* __restrict__ probs) {
    extern __shared__ float head_smem[];   // [F / 8][NCLS][8]
    const int tid = threadIdx.x, lane = tid & 31, sub = lane % LPR;
    for (int i = tid; i < NCLS * F; i += HEAD_THREADS) {
        const int c = i / F, f = i % F;
        head_smem[((f >> 3) * NCLS + c) * 8 + (f & 7)] = __half2float(w[i]);
    }
    float b[NCLS];
#pragma unroll
    for (int c = 0; c < NCLS; ++c) b[c] = bias ? __half2float(bias[c]) : 0.f;
    __syncthreads();
    constexpr int RPW = 32 / LPR;
    const long long warps = (long long)gridDim.x * (HEAD_THREADS / 32);
    const int G = F / 8;
    for (long long base = ((long long)blockIdx.x * (HEAD_THREADS / 32) + (tid >> 5)) * RPW; base < M; base += warps * RPW) {
        const long long row = base + lane / LPR;
        const bool valid = row < M;
        float acc[NCLS] = {0.f, 0.f, 0.f, 0.f, 0.f};
        if (valid) {
            const uint4* xr = reinterpret_cast<const uint4*>(x + row * F);
            for (int g = sub; g < G; g += LPR) {
                const uint4 v = xr[g];
                const __half2* h = reinterpret_cast<const __half2*>(&v);
                float xf[8];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float2 f2 = __half22float2(h[q]);
                    xf[2 * q] = f2.x;
                    xf[2 * q + 1] = f2.y;
                }
                const float4* wg = reinterpret_cast<const float4*>(head_smem + g * NCLS * 8);
#pragma unroll
                for (int c = 0; c < NCLS; ++c) {
                    const float4 wa = wg[2 * c], wb = wg[2 * c + 1];
                    acc[c] = fmaf(wa.x, xf[0], acc[c]);
                    acc[c] = fmaf(wa.y, xf[1], acc[c]);
                    acc[c] = fmaf(wa.z, xf[2], acc[c]);
                    acc[c] = fmaf(wa.w, xf[3], acc[c]);
                    acc[c] = fmaf(wb.x, xf[4], acc[c]);
                    acc[c] = fmaf(wb.y, xf[5], acc[c]);
                    acc[c] = fmaf(wb.z, xf[6], acc[c]);
                    acc[c] = fmaf(wb.w, xf[7], acc[c]);
                }
            }
        }
#pragma unroll
        for (int off = LPR / 2; off > 0; off >>= 1)
#pragma unroll
            for (int c = 0; c < NCLS; ++c) acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], off);
        if (!valid || sub != 0) continue;
        // logits rounded to fp16 (the half Conv1d), log_softmax in fp32 rounded to fp16 (the half log_softmax)
        float l[NCLS], m = -INFINITY;
#pragma unroll
        for (int c = 0; c < NCLS; ++c) {
            l[c] = round_f16(acc[c] + b[c]);
            m = fmaxf(m, l[c]);
        }
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < NCLS; ++c) s += expf(l[c] - m);
        const float lse = m + logf(s);
        int best = 0;
        float lp[NCLS], top = -INFINITY;
#pragma unroll
        for (int c = 0; c < NCLS; ++c) {
            lp[c] = round_f16(l[c] - lse);
            if (lp[c] >= top) {                  // equal log-probs: the highest index wins
                top = lp[c];
                best = c;
            }
        }
        if (logp) {
#pragma unroll
            for (int c = 0; c < NCLS; ++c) logp[row * NCLS + c] = __float2half_rn(lp[c]);
        }
        labels[row] = (uint8_t)best;
        probs[row] = expf(top);
    }
}

}  // namespace

int launch_conv_first_ex(const __half* x, int N, int L, int C, int K, int S, const __half* w, const __half* bias, int act,
                         float lo, float hi, __half* out, long long ldo, int Lp, int padl, cudaStream_t stream) {
    B200_REQUIRE(C % 8 == 0 && C > 0 && C <= 512 && K % 2 == 1 && K <= 33 && S >= 1 && S <= 8,
                 "conv_first_ex: unsupported shape 1->%d (k%d, stride %d)", C, K, S);
    B200_REQUIRE(ldo % 8 == 0 && ldo >= C && ((uintptr_t)out & 15) == 0,
                 "conv_first_ex: ldo must be a multiple of 8 and >= C, out 16-byte aligned (ldo=%lld)", ldo);
    const int T = (L - 1) / S + 1;    // (L + 2 (K/2) - K) / S + 1 for odd K
    B200_REQUIRE(Lp >= padl + T, "conv_first_ex: lp=%d < padl + frames (%d + %d)", Lp, padl, T);
    dim3 grid((Lp + CFX_THREADS - 1) / CFX_THREADS, (C + CFX_CC - 1) / CFX_CC, N);
    const size_t smem = (size_t)(K * CFX_CC + CFX_CC + (CFX_THREADS - 1) * S + K) * sizeof(float);
    conv_first_ex_kernel<<<grid, CFX_THREADS, smem, stream>>>(x, L, w, bias, C, K, S, T, act, lo, hi, out, ldo, Lp, padl);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int launch_ctc_head(const __half* x, long long M, int F, const __half* w, const __half* bias, __half* logp, uint8_t* labels,
                    float* probs, cudaStream_t stream) {
    B200_REQUIRE(F % 8 == 0 && F > 0 && F <= 2048 && ((uintptr_t)x & 15) == 0,
                 "ctc_head: features must be a multiple of 8 in [8, 2048] and x 16-byte aligned (F=%d)", F);
    const size_t smem = (size_t)NCLS * F * sizeof(float);
    int dev = 0, sms = 0;
    B200_CHECK_CUDA(cudaGetDevice(&dev));
    B200_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const int G = F / 8;
    const int lpr = G >= 32 ? 32 : G > 8 ? 16 : G > 4 ? 8 : G > 2 ? 4 : G > 1 ? 2 : 1;
    const long long rows_per_cta = (long long)(HEAD_THREADS / 32) * (32 / lpr);
    const unsigned grid = (unsigned)std::min<long long>((M + rows_per_cta - 1) / rows_per_cta, (long long)sms * 8);
    switch (lpr) {
#define HEAD_CASE(v) \
        case v: ctc_head_kernel<v><<<grid, HEAD_THREADS, smem, stream>>>(x, M, F, w, bias, logp, labels, probs); break;
        HEAD_CASE(1) HEAD_CASE(2) HEAD_CASE(4) HEAD_CASE(8) HEAD_CASE(16) HEAD_CASE(32)
#undef HEAD_CASE
    }
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}
