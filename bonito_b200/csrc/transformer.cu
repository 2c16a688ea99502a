// Kernels of the transformer (sup v5) path that are not GEMMs.  Reference semantics:
//   conv_first      bonito/nn.py:221-241  Convolution(1 -> C, k, 'same') + Swish, written channels-last + zero halo so
//                   that every following Convolution is a wgmma GEMM over overlapping rows (gemm_wgmma.cu)
//   attention       bonito/transformer/model.py:42-79  rotary (flash_attn/layers/rotary.py, NeoX half rotation, fp16 cos/sin)
//                   + flash_attn_qkvpacked_func(window_size=(wl, wr)), non-causal, softmax scale 1/sqrt(head_dim)
//   rmsnorm         bonito/transformer/model.py:126-127  x = RMSNorm(sublayer(x), residual = alpha * x)
//                   (flash_attn/ops/triton/layer_norm.py: add and normalise in fp32, one rounding on store; alpha*x is an
//                   fp16 multiply in the reference because deepnorm_alpha is a half buffer)
//   swiglu          flash_attn/ops/activations.py:107-111  float(gate) * float(y) / (1 + exp(-gate)), rounded once
// First correct versions: attention runs on the legacy mma.sync path (it is ~6 % of the layer's FLOPs because of the
// 256-wide window); the GEMMs are the wgmma kernels.
#include <stdlib.h>

#include "common.cuh"

namespace {

// ------------------------------------------------------------------------------------------------ conv_first
constexpr int CF_THREADS = 128;

__global__ void __launch_bounds__(CF_THREADS)
conv_first_kernel(const __half* __restrict__ x, int L, const __half* __restrict__ w, const __half* __restrict__ bias,
                  int C, int K, int act, __half* __restrict__ out, int Lp, int padl) {
    extern __shared__ float cf_smem[];
    float* ws = cf_smem;                 // [K][C]
    float* bs = ws + K * C;              // [C]
    float* xs = bs + C;                  // [CF_THREADS + K - 1]
    const int tid = threadIdx.x, n = blockIdx.y;
    const int p0 = blockIdx.x * CF_THREADS, l0 = p0 - padl, P = K / 2;
    for (int i = tid; i < K * C; i += CF_THREADS) ws[i] = __half2float(w[(i % C) * K + i / C]);
    for (int i = tid; i < C; i += CF_THREADS) bs[i] = bias ? __half2float(bias[i]) : 0.f;
    for (int i = tid; i < CF_THREADS + K - 1; i += CF_THREADS) {
        const int l = l0 - P + i;
        xs[i] = (l >= 0 && l < L) ? __half2float(x[(size_t)n * L + l]) : 0.f;
    }
    __syncthreads();
    const int p = p0 + tid;
    if (p >= Lp) return;
    const int l = p - padl;
    __half* dst = out + ((size_t)n * Lp + p) * C;
    const bool in = l >= 0 && l < L;
    for (int c0 = 0; c0 < C; c0 += 8) {
        __half2 h[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            float v[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int c = c0 + 2 * q + e;
                float acc = bs[c];
                for (int k = 0; k < K; ++k) acc = fmaf(ws[k * C + c], xs[tid + k], acc);
                v[e] = in ? apply_act_f16(acc, act, 0.f, 0.f) : 0.f;
            }
            h[q] = __floats2half2_rn(v[0], v[1]);
        }
        *reinterpret_cast<uint4*>(dst + c0) = *reinterpret_cast<uint4*>(h);
    }
}

// ------------------------------------------------------------------------------------------------ rmsnorm
// out[r] = rmsnorm(a[r] + fp16(alpha * x[r])) * w ; one warp per row, D = 32 * 8 * VEC elements
template <int D>
__global__ void __launch_bounds__(256)
rmsnorm_residual_kernel(const __half* __restrict__ a, const __half* __restrict__ x, const __half* __restrict__ w,
                        float alpha, float eps, __half* __restrict__ out, long long M) {
    constexpr int VEC = D / 256;  // uint4 (8 halves) per lane
    const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= M) return;
    float s[VEC][8];
    float ss = 0.f;
#pragma unroll
    for (int v = 0; v < VEC; ++v) {
        const int col = (v * 32 + lane) * 8;
        const uint4 ra = *reinterpret_cast<const uint4*>(a + row * D + col);
        const uint4 rx = *reinterpret_cast<const uint4*>(x + row * D + col);
        const __half2* ha = reinterpret_cast<const __half2*>(&ra);
        const __half2* hx = reinterpret_cast<const __half2*>(&rx);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float2 fa = __half22float2(ha[q]), fx = __half22float2(hx[q]);
            s[v][2 * q] = fa.x + round_f16(alpha * fx.x);
            s[v][2 * q + 1] = fa.y + round_f16(alpha * fx.y);
            ss += s[v][2 * q] * s[v][2 * q] + s[v][2 * q + 1] * s[v][2 * q + 1];
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float rstd = rsqrtf(ss / D + eps);
#pragma unroll
    for (int v = 0; v < VEC; ++v) {
        const int col = (v * 32 + lane) * 8;
        const uint4 rw = *reinterpret_cast<const uint4*>(w + col);
        const __half2* hw = reinterpret_cast<const __half2*>(&rw);
        __half2 o[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float2 fw = __half22float2(hw[q]);
            o[q] = __floats2half2_rn(s[v][2 * q] * rstd * fw.x, s[v][2 * q + 1] * rstd * fw.y);
        }
        *reinterpret_cast<uint4*>(out + row * D + col) = *reinterpret_cast<uint4*>(o);
    }
}

// ------------------------------------------------------------------------------------------------ swiglu
// h [M][2F]: y = h[:, :F], gate = h[:, F:]  ->  out[M][F] = gate * y / (1 + exp(-gate))
__global__ void __launch_bounds__(256)
swiglu_kernel(const __half* __restrict__ h, __half* __restrict__ out, long long M, int F) {
    const long long i = ((long long)blockIdx.x * 256 + threadIdx.x) * 8;
    if (i >= M * F) return;
    const long long row = i / F;
    const int col = (int)(i - row * F);
    const uint4 ry = *reinterpret_cast<const uint4*>(h + row * 2 * F + col);
    const uint4 rg = *reinterpret_cast<const uint4*>(h + row * 2 * F + F + col);
    const __half2* hy = reinterpret_cast<const __half2*>(&ry);
    const __half2* hg = reinterpret_cast<const __half2*>(&rg);
    __half2 o[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const float2 y = __half22float2(hy[q]), g = __half22float2(hg[q]);
        o[q] = __floats2half2_rn(g.x * y.x / (1.0f + __expf(-g.x)), g.y * y.y / (1.0f + __expf(-g.y)));
    }
    *reinterpret_cast<uint4*>(out + i) = *reinterpret_cast<uint4*>(o);
}

// ------------------------------------------------------------------------------------------------ attention
// qkv [N][T][3][NH][64] fp16; rotary on q and k; keys j with q - wl <= j <= q + wr; out [N][T][NH*64].
// One CTA = 64 queries of one (chunk, head), 4 warps x 16 query rows, flash-style online softmax over 64-key blocks
// streamed through a cp.async double buffer.
constexpr int HD = 64, AQ = 64, AK = 64, LDT = HD + 8;

__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
                 : "r"(addr));
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}

// Rotary embedding applied once, in place, to the q and k parts of the packed projection (the attention kernel then
// only copies tiles; rotating inside its loader repeated the work for each of the ~5 query tiles that read a key block).
// One thread per (token, q|k, head, 8-element group of the first half): rotates (x[d], x[d+32]) for 8 d.
__global__ void __launch_bounds__(256)
rotary_kernel(__half* __restrict__ qkv, const __half* __restrict__ cs, long long tokens, int T, int NH) {
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    const long long total = tokens * 2 * NH * 4;
    if (i >= total) return;
    const int grp = (int)(i & 3);
    const int head = (int)((i >> 2) % NH);
    const int which = (int)((i / (4LL * NH)) & 1);
    const long long tok = i / (8LL * NH);
    const int t = (int)(tok % T);
    __half* p = qkv + ((tok * 3 + which) * NH + head) * HD + grp * 8;
    const __half* c = cs + (size_t)t * 64 + grp * 8;
    uint4 lo = *reinterpret_cast<uint4*>(p), hi = *reinterpret_cast<uint4*>(p + 32);
    const uint4 cc = *reinterpret_cast<const uint4*>(c), ss = *reinterpret_cast<const uint4*>(c + 32);
    __half* x1 = reinterpret_cast<__half*>(&lo);
    __half* x2 = reinterpret_cast<__half*>(&hi);
    const __half* co = reinterpret_cast<const __half*>(&cc);
    const __half* si = reinterpret_cast<const __half*>(&ss);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        const float a = __half2float(x1[e]), b = __half2float(x2[e]), cf = __half2float(co[e]), sf = __half2float(si[e]);
        x1[e] = __float2half_rn(a * cf - b * sf);
        x2[e] = __float2half_rn(a * sf + b * cf);
    }
    *reinterpret_cast<uint4*>(p) = lo;
    *reinterpret_cast<uint4*>(p + 32) = hi;
}

// load 64 rows x 64 dims of q or k (which = 0/1) or v (2) starting at token t0 into smem [64][LDT]; `cs` != nullptr
// applies the rotary embedding to q / k on the fly (used when the projection has not been rotated in place)
__device__ __forceinline__ void load_tile(__half (*dst)[LDT], const __half* __restrict__ qkv, const __half* __restrict__ cs,
                                          int n, int T, int NH, int head, int which, int t0, int tid) {
    const int row = tid >> 1, half16 = (tid & 1) * 16;  // dims [half16, half16+16) and the same + 32
    const int t = t0 + row;
    uint4 lo[2], hi[2];
    if (t >= 0 && t < T) {
        const __half* src = qkv + ((((size_t)n * T + t) * 3 + which) * NH + head) * HD;
        lo[0] = *reinterpret_cast<const uint4*>(src + half16);
        lo[1] = *reinterpret_cast<const uint4*>(src + half16 + 8);
        hi[0] = *reinterpret_cast<const uint4*>(src + 32 + half16);
        hi[1] = *reinterpret_cast<const uint4*>(src + 32 + half16 + 8);
        if (which < 2 && cs != nullptr) {
            const __half* c = cs + (size_t)t * 64 + half16;   // cos [T][32] then sin at +32
            const __half* x1 = reinterpret_cast<const __half*>(lo);
            const __half* x2 = reinterpret_cast<const __half*>(hi);
            __half o1[16], o2[16];
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const float co = __half2float(c[i]), si = __half2float(c[32 + i]);
                const float a = __half2float(x1[i]), b = __half2float(x2[i]);
                o1[i] = __float2half_rn(a * co - b * si);
                o2[i] = __float2half_rn(a * si + b * co);
            }
            lo[0] = reinterpret_cast<uint4*>(o1)[0]; lo[1] = reinterpret_cast<uint4*>(o1)[1];
            hi[0] = reinterpret_cast<uint4*>(o2)[0]; hi[1] = reinterpret_cast<uint4*>(o2)[1];
        }
    } else {
        lo[0] = lo[1] = hi[0] = hi[1] = make_uint4(0, 0, 0, 0);
    }
    *reinterpret_cast<uint4*>(&dst[row][half16]) = lo[0];
    *reinterpret_cast<uint4*>(&dst[row][half16 + 8]) = lo[1];
    *reinterpret_cast<uint4*>(&dst[row][32 + half16]) = hi[0];
    *reinterpret_cast<uint4*>(&dst[row][32 + half16 + 8]) = hi[1];
}

// the same tile through cp.async (16-byte pieces, rows outside [0, T) zero-filled): used for the double-buffered K / V stream
__device__ __forceinline__ void load_tile_async(__half (*dst)[LDT], const __half* __restrict__ qkv, int n, int T, int NH,
                                                int head, int which, int t0, int tid) {
    const int row = tid >> 1, half16 = (tid & 1) * 16;
    const int t = t0 + row;
    const bool ok = t >= 0 && t < T;
    const __half* src = ok ? qkv + ((((size_t)n * T + t) * 3 + which) * NH + head) * HD : qkv;
    cp_async_16(&dst[row][half16], src + half16, ok);
    cp_async_16(&dst[row][half16 + 8], src + half16 + 8, ok);
    cp_async_16(&dst[row][32 + half16], src + 32 + half16, ok);
    cp_async_16(&dst[row][32 + half16 + 8], src + 32 + half16 + 8, ok);
}

__global__ void __launch_bounds__(128)
attention_kernel(const __half* __restrict__ qkv, const __half* __restrict__ cs, __half* __restrict__ out, int T, int NH,
                 int wl, int wr, float scale_log2e) {
    __shared__ __align__(16) __half Qs[AQ][LDT];
    __shared__ __align__(16) __half Kb[2][AK][LDT];   // double-buffered: block i+1 streams in while block i is consumed
    __shared__ __align__(16) __half Vb[2][AK][LDT];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int q0 = blockIdx.x * AQ, head = blockIdx.y, n = blockIdx.z;
    const int g = lane >> 2, qd = lane & 3;

    load_tile(Qs, qkv, cs, n, T, NH, head, 0, q0, tid);
    __syncthreads();
    uint32_t qf[4][4];   // A fragments of this warp's 16 query rows, 4 k-steps over the 64 dims
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
        const int row = warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
        ldmatrix_x4(qf[kk][0], qf[kk][1], qf[kk][2], qf[kk][3], smem_u32(&Qs[row][kk * 16 + (lane >> 4) * 8]));
    }
    float o[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    const int qrow[2] = {q0 + warp * 16 + g, q0 + warp * 16 + g + 8};

    int k_lo = q0 - wl; if (k_lo < 0) k_lo = 0;
    int k_hi = q0 + AQ - 1 + wr + 1; if (k_hi > T) k_hi = T;
    const int kb0 = (k_lo / AK) * AK;
    if (kb0 < k_hi) {
        load_tile_async(Kb[0], qkv, n, T, NH, head, 1, kb0, tid);
        load_tile_async(Vb[0], qkv, n, T, NH, head, 2, kb0, tid);
    }
    cp_async_commit();
    int buf = 0;
    for (int kb = kb0; kb < k_hi; kb += AK, buf ^= 1) {
        if (kb + AK < k_hi) {   // the other buffer was released by the barrier that ended the previous iteration
            load_tile_async(Kb[buf ^ 1], qkv, n, T, NH, head, 1, kb + AK, tid);
            load_tile_async(Vb[buf ^ 1], qkv, n, T, NH, head, 2, kb + AK, tid);
        }
        cp_async_commit();
        cp_async_wait<1>();   // everything but the group just committed: this block's tiles have landed
        __syncthreads();
        __half (*Ks)[LDT] = Kb[buf];
        __half (*Vs)[LDT] = Vb[buf];
        // S = Q K^T  (16 x 64 per warp)
        float s[8][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
            for (int jp = 0; jp < 4; ++jp) {
                uint32_t b0, b1, b2, b3;
                const int row = jp * 16 + (lane & 7) + (lane >> 4) * 8;
                ldmatrix_x4(b0, b1, b2, b3, smem_u32(&Ks[row][kk * 16 + ((lane >> 3) & 1) * 8]));
                mma_16816(s[2 * jp], qf[kk], b0, b1);
                mma_16816(s[2 * jp + 1], qf[kk], b2, b3);
            }
        }
        // mask + online softmax (rows g and g+8; a row is shared by the 4 lanes of a quad)
        float m_new[2] = {m_run[0], m_run[1]};
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int r = e >> 1, key = kb + j * 8 + 2 * qd + (e & 1), q = qrow[r];
                const bool ok = key < T && q < T && key >= q - wl && key <= q + wr;
                s[j][e] = ok ? s[j][e] : -INFINITY;
                m_new[r] = fmaxf(m_new[r], s[j][e]);
            }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            m_new[r] = fmaxf(m_new[r], __shfl_xor_sync(0xffffffffu, m_new[r], 1));
            m_new[r] = fmaxf(m_new[r], __shfl_xor_sync(0xffffffffu, m_new[r], 2));
        }
        float corr[2], msafe[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            msafe[r] = (m_new[r] == -INFINITY) ? 0.f : m_new[r];
            corr[r] = ex2_approx((m_run[r] - msafe[r]) * scale_log2e);   // ex2(-inf) = 0 for the first block
            m_run[r] = m_new[r];
            l_run[r] *= corr[r];
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            o[j][0] *= corr[0]; o[j][1] *= corr[0]; o[j][2] *= corr[1]; o[j][3] *= corr[1];
        }
        uint32_t pf[4][4];   // P as A fragments: k-step kk covers keys 16kk .. 16kk+15 = score tiles 2kk, 2kk+1
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float p[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                p[e] = ex2_approx((s[j][e] - msafe[e >> 1]) * scale_log2e);
                l_run[e >> 1] += p[e];
            }
            pf[j >> 1][(j & 1) * 2 + 0] = pack_h2(p[0], p[1]);
            pf[j >> 1][(j & 1) * 2 + 1] = pack_h2(p[2], p[3]);
        }
        // O += P V   (V^T fragments through ldmatrix.trans)
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
            for (int dp = 0; dp < 4; ++dp) {
                uint32_t b0, b1, b2, b3;
                const int row = kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;   // key
                const int col = dp * 16 + (lane >> 4) * 8;                       // dim
                ldmatrix_x4_trans(b0, b1, b2, b3, smem_u32(&Vs[row][col]));
                mma_16816(o[2 * dp], pf[kk], b0, b1);
                mma_16816(o[2 * dp + 1], pf[kk], b2, b3);
            }
        }
        __syncthreads();   // this buffer is refilled by the loads issued at the top of the next iteration but one
    }
    // normalise and store
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
        l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int q = qrow[r];
        if (q >= T) continue;
        const float inv = 1.0f / l_run[r];
        __half* dst = out + ((size_t)n * T + q) * NH * HD + head * HD;
#pragma unroll
        for (int j = 0; j < 8; ++j)
            *reinterpret_cast<__half2*>(dst + j * 8 + 2 * qd) = __floats2half2_rn(o[j][2 * r] * inv, o[j][2 * r + 1] * inv);
    }
}

}  // namespace

int launch_conv_first(const __half* x, int N, int L, int C, int K, const __half* w, const __half* bias, int act,
                      __half* out, int Lp, int padl, cudaStream_t stream) {
    B200_REQUIRE(C % 8 == 0 && C <= 128 && K % 2 == 1 && K <= 15, "conv_first: unsupported shape 1->%d (k%d)", C, K);
    B200_REQUIRE(N <= 65535, "conv_first: at most 65535 chunks per call (n=%d): the chunk index is gridDim.y", N);
    dim3 grid((Lp + CF_THREADS - 1) / CF_THREADS, N);
    const size_t smem = (size_t)(K * C + C + CF_THREADS + K) * sizeof(float);
    conv_first_kernel<<<grid, CF_THREADS, smem, stream>>>(x, L, w, bias, C, K, act, out, Lp, padl);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int launch_rmsnorm_residual(const __half* a, const __half* x, const __half* w, float alpha, float eps, __half* out,
                            long long M, int D, cudaStream_t stream) {
    const unsigned grid = (unsigned)((M + 7) / 8);
    if (D == 512) rmsnorm_residual_kernel<512><<<grid, 256, 0, stream>>>(a, x, w, alpha, eps, out, M);
    else if (D == 256) rmsnorm_residual_kernel<256><<<grid, 256, 0, stream>>>(a, x, w, alpha, eps, out, M);
    else if (D == 768) rmsnorm_residual_kernel<768><<<grid, 256, 0, stream>>>(a, x, w, alpha, eps, out, M);
    else if (D == 1024) rmsnorm_residual_kernel<1024><<<grid, 256, 0, stream>>>(a, x, w, alpha, eps, out, M);
    else { b200_set_error("rmsnorm: d_model %d is not supported (256, 512, 768, 1024)", D); return -2; }
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int launch_swiglu(const __half* h, __half* out, long long M, int F, cudaStream_t stream) {
    B200_REQUIRE(F % 8 == 0, "swiglu: hidden size %d must be a multiple of 8", F);
    const long long vecs = M * F / 8;
    swiglu_kernel<<<(unsigned)((vecs + 255) / 256), 256, 0, stream>>>(h, out, M, F);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int launch_attention_wgmma(const __half* qkv, __half* out, int N, int T, int NH, int wl, int wr, cudaStream_t stream);

int launch_attention(__half* qkv, const __half* cos_sin, __half* out, int N, int T, int NH, int head_dim, int wl,
                     int wr, cudaStream_t stream) {
    B200_REQUIRE(head_dim == HD, "attention: head_dim %d is not supported (64)", head_dim);
    const long long tokens = (long long)N * T, work = tokens * 2 * NH * 4;
    rotary_kernel<<<(unsigned)((work + 255) / 256), 256, 0, stream>>>(qkv, cos_sin, tokens, T, NH);
    // product path: the wgmma kernel (attention_wgmma.cu); B200_ATTN_IMPL=mma runs the mma.sync kernel below (on-device
    // cross-check)
    const char* impl = getenv("B200_ATTN_IMPL");
    if (!(impl && impl[0] == 'm')) {
        B200_CHECK_CUDA(cudaGetLastError());
        return launch_attention_wgmma(qkv, out, N, T, NH, wl, wr, stream);
    }
    if (wl < 0) wl = T;
    if (wr < 0) wr = T;
    dim3 grid((T + AQ - 1) / AQ, NH, N);
    const float scale_log2e = 1.4426950408889634f / sqrtf((float)head_dim);
    attention_kernel<<<grid, 128, 0, stream>>>(qkv, nullptr, out, T, NH, wl, wr, scale_log2e);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}
