// C[M,N] = epilogue(A[M,K] * B[N,K]^T) on the Hopper tensor cores (wgmma, sm_90a): the product GEMM of every
// convolution-as-GEMM, LSTM input projection, CRF head and transformer projection.
//
//   * CTA tile 128 x 128, two warpgroups of 64 rows each issue wgmma.mma_async m64n128 (fp16: k16, int8: k32) with both
//     operands in shared memory, fp32 / s32 accumulators in registers (64 per thread);
//   * a 3-deep cp.async ring of 128-byte K slices (64 fp16 or 128 int8 per row) per operand, stored K-major without
//     swizzle as 8-row x 16-byte core matrices ([16-byte k-chunk][row][16 B]); two CTAs per SM (96 KB each), so one
//     CTA's epilogue overlaps the other's main loop;
//   * the epilogue works on the accumulator fragment in registers (thread = rows lane/4 and lane/4 + 8 of its warp's
//     16 rows, columns 8j + 2(lane%4) + {0,1}): bias, fp16 rounding, activation, the row / column-block maps of
//     GemmEpilogue, and the fused SwiGLU (a 64-column group [32 y | 32 gate] lies in one thread's columns).
//
// A rows may overlap (lda < K): the strided convolutions run as GEMMs over the channels-last, zero-padded stem output
// (reference: bonito/nn.py:235-241, Conv1d k19 s6).
#include <type_traits>

#include "tc_common.cuh"

namespace {

constexpr int BM = 128, BN = 128, KB = 128;          // KB: bytes of K per stage and row
constexpr int KC = KB / 16;                          // 16-byte k-chunks per stage
constexpr int STAGES = 3, THREADS = 256;
constexpr uint32_t OP_BYTES = BM * KB;               // one operand slice: 16 KB
constexpr uint32_t STAGE_BYTES = 2 * OP_BYTES;
constexpr uint32_t SMEM_BYTES = STAGES * STAGE_BYTES;   // 96 KB

template <bool I8>
__global__ void __launch_bounds__(THREADS, 2)
gemm_wgmma_kernel(const unsigned char* __restrict__ A, long long lda_bytes, const unsigned char* __restrict__ B,
                  const float* __restrict__ col_scale, __half* __restrict__ C, long long ldc, int M, int N, int K_bytes,
                  GemmEpilogue ep) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const uint32_t base = smem_u32(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wg = warp >> 2, wq = warp & 3;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
    const int ktiles = (K_bytes + KB - 1) / KB;

    // 2 x 1024 16-byte chunks per stage; chunk c: k-chunk c % KC of row c / KC (a warp reads 4 rows x 128 contiguous bytes)
    auto load_stage = [&](int stage, int kt) {
        const int k0 = kt * KB;
        unsigned char* sa = smem_raw + stage * STAGE_BYTES;
#pragma unroll
        for (int i = 0; i < (BM * KC) / THREADS; ++i) {
            const int c = tid + i * THREADS, row = c / KC, kc = c % KC;
            const bool kin = k0 + kc * 16 < K_bytes;
            const int gm = m0 + row, gn = n0 + row;
            const bool va = kin && gm < M, vb = kin && gn < N;
            const uint32_t off = (uint32_t)kc * (BM * 16) + (uint32_t)row * 16;
            cp_async_16(sa + off, A + (va ? (long long)gm * lda_bytes + k0 + kc * 16 : 0), va);
            cp_async_16(sa + OP_BYTES + off, B + (vb ? (long long)gn * K_bytes + k0 + kc * 16 : 0), vb);
        }
    };

    using Acc = typename std::conditional<I8, int, float>::type;
    Acc acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0;

#pragma unroll
    for (int st = 0; st < STAGES - 1; ++st) {
        if (st < ktiles) load_stage(st, st);
        cp_async_commit();
    }
    for (int kt = 0; kt < ktiles; ++kt) {
        cp_async_wait<STAGES - 2>();
        fence_proxy_async_smem();   // cp.async writes (generic proxy) -> visible to wgmma (async proxy)
        __syncthreads();            // also: every warpgroup is done with the stage refilled below
        {
            const int nk = kt + STAGES - 1;
            if (nk < ktiles) load_stage(nk % STAGES, nk);
            cp_async_commit();
        }
        const uint32_t sa = base + (uint32_t)(kt % STAGES) * STAGE_BYTES + (uint32_t)wg * (64 * 16);
        const uint32_t sb = base + (uint32_t)(kt % STAGES) * STAGE_BYTES + OP_BYTES;
        wg_fence_regs(acc);
        wg_fence();
#pragma unroll
        for (int ks = 0; ks < KC / 2; ++ks) {   // one wgmma consumes two k-chunks (32 bytes of K)
            const uint64_t da = wg_desc_noswz(sa + (uint32_t)ks * 2 * (BM * 16), BM * 16, 128);
            const uint64_t db = wg_desc_noswz(sb + (uint32_t)ks * 2 * (BN * 16), BN * 16, 128);
            if constexpr (I8) wgmma_m64n128k32_s8(acc, da, db, 1);
            else wgmma_m64n128k16_f16(acc, da, db, 1);
        }
        wg_commit();
        wg_wait<0>();
        wg_fence_regs(acc);
    }
    cp_async_wait<0>();

    const int r0 = m0 + wg * 64 + wq * 16 + (lane >> 2), cq = 2 * (lane & 3);
    if (!I8 && ep.act == B200_ACT_SWIGLU) {
        // 64-column group G of the tile: y = columns 8j' + cq + e, gate = 32 + the same; output column (n0 + 64G) / 2 + ...
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int gm = r0 + 8 * h;
            if (gm >= M) continue;
            const long long orow = map_row(ep.map, gm);
            if (orow < 0) continue;
#pragma unroll
            for (int G = 0; G < 2; ++G) {
                if (n0 + 64 * G >= N) continue;
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) {
                    const int jy = 8 * G + jj, jg = jy + 4;
                    const float y0 = round_f16((float)acc[jy * 4 + h * 2]), y1 = round_f16((float)acc[jy * 4 + h * 2 + 1]);
                    const float g0 = round_f16((float)acc[jg * 4 + h * 2]), g1 = round_f16((float)acc[jg * 4 + h * 2 + 1]);
                    const int oc = (n0 + 64 * G) / 2 + 8 * jj + cq;
                    *reinterpret_cast<__half2*>(C + orow * ldc + oc) =
                        __floats2half2_rn(g0 * y0 * rcp_approx(1.0f + __expf(-g0)), g1 * y1 * rcp_approx(1.0f + __expf(-g1)));
                }
            }
        }
        return;
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int gm = r0 + 8 * h;
        if (gm >= M) continue;
        const long long orow = map_row(ep.map, gm);
        if (orow < 0) continue;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const int gn = n0 + 8 * j + cq;   // N % 8 == 0: the pair (gn, gn + 1) is in range together
            if (gn >= N) continue;
            float v0, v1;
            if constexpr (I8) {
                const float b0 = ep.bias ? __half2float(ep.bias[gn]) : 0.f, b1 = ep.bias ? __half2float(ep.bias[gn + 1]) : 0.f;
                v0 = fmaf((float)acc[j * 4 + h * 2], col_scale[gn], b0);
                v1 = fmaf((float)acc[j * 4 + h * 2 + 1], col_scale[gn + 1], b1);
            } else {
                v0 = acc[j * 4 + h * 2];
                v1 = acc[j * 4 + h * 2 + 1];
                if (ep.bias) {
                    v0 += __half2float(ep.bias[gn]);
                    v1 += __half2float(ep.bias[gn + 1]);
                }
            }
            v0 = apply_act_f16(v0, ep.act, ep.lo, ep.hi);
            v1 = apply_act_f16(v1, ep.act, ep.lo, ep.hi);
            long long drow = orow;
            int dcol = gn;
            if (ep.cb_width > 0) {   // column-block remap (cb_width is even: a pair never straddles two blocks)
                const int cb = gn / ep.cb_width;
                drow += (long long)cb * ep.cb_rows;
                dcol = gn - cb * ep.cb_width;
            }
            *reinterpret_cast<__half2*>(C + drow * ldc + dcol) = __floats2half2_rn(v0, v1);
        }
    }
}

template <bool I8>
int launch(const void* A, long long lda_bytes, const void* B, const float* col_scale, __half* C, long long ldc, int M, int N,
           int K_bytes, const GemmEpilogue& ep, cudaStream_t stream) {
    static bool configured = false;
    if (!configured) {
        B200_CHECK_CUDA(cudaFuncSetAttribute(gemm_wgmma_kernel<I8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
        configured = true;
    }
    dim3 grid((N + BN - 1) / BN, (M + BM - 1) / BM);
    B200_REQUIRE(grid.y <= 65535, "gemm: M = %d needs more than 65535 row blocks", M);
    gemm_wgmma_kernel<I8><<<grid, THREADS, SMEM_BYTES, stream>>>((const unsigned char*)A, lda_bytes, (const unsigned char*)B,
                                                                 col_scale, C, ldc, M, N, K_bytes, ep);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace

// max_ctas is accepted for the ABI and not needed here: the kernel is not persistent, its CTAs leave as they finish and
// the block scheduler hands the SMs to whatever else is queued.
int launch_gemm_tc(const __half* A, long long lda, const __half* B, __half* C, long long ldc, int M, int N, int K,
                   const GemmEpilogue& ep, int max_ctas, cudaStream_t stream) {
    (void)max_ctas;
    B200_REQUIRE(((uintptr_t)A % 16) == 0 && ((uintptr_t)B % 16) == 0 && ((uintptr_t)C % 16) == 0,
                 "gemm: operands must be 16-byte aligned");
    return launch<false>(A, lda * 2, B, nullptr, C, ldc, M, N, K * 2, ep, stream);
}

// C = act(scale[col] * (A_i8 B_i8^T) + bias): int8 operands (A [M][K] row stride lda bytes, B [N][K]), exact s32
// accumulation on the int8 tensor cores.
int launch_gemm_i8(const int8_t* A, long long lda, const int8_t* B, const float* col_scale, __half* C, long long ldc, int M,
                   int N, int K, const GemmEpilogue& ep, int max_ctas, cudaStream_t stream) {
    (void)max_ctas;
    B200_REQUIRE(((uintptr_t)A % 16) == 0 && ((uintptr_t)B % 16) == 0 && ((uintptr_t)C % 16) == 0 && col_scale != nullptr,
                 "gemm_i8: operands must be 16-byte aligned and a column scale is required");
    B200_REQUIRE(K % 16 == 0 && lda % 16 == 0 && ep.act != B200_ACT_SWIGLU,
                 "gemm_i8: K (%d) and lda (%lld) must be multiples of 16 bytes, no SwiGLU", K, lda);
    return launch<true>(A, lda, B, col_scale, C, ldc, M, N, K, ep, stream);
}
