// C[M,N] = epilogue(A[M,K] * B[N,K]^T) on the Hopper tensor cores (wgmma, sm_90a): the product GEMM of every
// convolution-as-GEMM, LSTM input projection, CRF head and transformer projection.
//
//   * a CTA owns one 128-row block of A and sweeps a run of 128-column tiles of N (all of them when the grid is large
//     enough), so that one CTA streams tile after tile through one pipeline: while it rounds and stores tile j, the next
//     tile's operands are already arriving;
//   * one producer warp fills a 3-deep ring of stages with TMA copies (128-byte K slices -- 64 fp16 or 128 int8 -- of 128
//     rows of A and of B, 128-byte swizzle), signalling through mbarriers ("full": bytes landed, "empty": every consumer
//     warp is done with the stage);
//   * two consumer warpgroups of 64 rows each issue wgmma.mma_async m64n128 (fp16: k16, int8: k32) with both operands in
//     shared memory, fp32 / s32 accumulators in registers (64 per thread), keeping one stage's MMAs in flight while the
//     next one is issued (wgmma.wait_group 1).  Every accumulator sums its K steps in ascending order;
//   * two CTAs per SM (97 KB of shared memory each), so one CTA's epilogue overlaps the other's MMAs;
//   * the epilogue works on the accumulator fragment in registers (thread = rows lane/4 and lane/4 + 8 of its warp's
//     16 rows, columns 8j + 2(lane%4) + {0,1}): bias, fp16 rounding, activation, the row / column-block maps of
//     GemmEpilogue, and the fused SwiGLU (a 64-column group [32 y | 32 gate] lies in one thread's columns).
//
// A rows may overlap (lda < K): the strided convolutions run as GEMMs over the channels-last, zero-padded stem output
// (reference: bonito/nn.py:235-241, Conv1d k19 s6).  TMA zero-fills the rows / columns of a partial tile.
#include <cuda.h>
#include <cudaTypedefs.h>

#include <type_traits>

#include "tc_common.cuh"

namespace {

constexpr int BM = 128, BN = 128, KB = 128;          // KB: bytes of K per stage and row (one 128-byte swizzle row)
constexpr int STAGES = 3;
constexpr int CONSUMERS = 256, THREADS = CONSUMERS + 32;   // two consumer warpgroups + one producer warp
constexpr uint32_t OP_BYTES = BM * KB;               // one operand slice: 16 KB
constexpr uint32_t STAGE_BYTES = 2 * OP_BYTES;
constexpr uint32_t SMEM_BYTES = 1024 + STAGES * STAGE_BYTES + 64;   // alignment slack + ring + 2 x STAGES mbarriers

template <bool I8>
__global__ void __launch_bounds__(THREADS, 2)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
                  const float* __restrict__ col_scale, __half* __restrict__ C, long long ldc, int M, int N, int K_bytes,
                  int tiles_per_cta, GemmEpilogue ep) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;   // the 128-byte swizzle repeats every 1024 bytes
    const uint32_t bar_full = base + STAGES * STAGE_BYTES, bar_empty = bar_full + 8 * STAGES;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int m0 = blockIdx.x * BM;
    const int ntiles = (N + BN - 1) / BN;
    const int nt0 = blockIdx.y * tiles_per_cta, nt1 = min(ntiles, nt0 + tiles_per_cta);
    const int ktiles = (K_bytes + KB - 1) / KB;

    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(bar_full + 8 * s, 1);
            mbar_init(bar_empty + 8 * s, CONSUMERS / 32);
        }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp == CONSUMERS / 32) {   // producer
        if (elect_one_sync()) {
            int it = 0;
            for (int nt = nt0; nt < nt1; ++nt) {
                for (int kt = 0; kt < ktiles; ++kt, ++it) {
                    const int s = it % STAGES;
                    mbar_wait(bar_empty + 8 * s, ((it / STAGES) & 1) ^ 1);
                    const uint32_t sa = base + (uint32_t)s * STAGE_BYTES, full = bar_full + 8 * s;
                    mbar_expect_tx(full, STAGE_BYTES);
                    const int k0 = kt * (I8 ? KB : KB / 2);   // in elements
                    tma_load_2d(sa, &tma_a, k0, m0, full);
                    tma_load_2d(sa + OP_BYTES, &tma_b, k0, nt * BN, full);
                }
            }
        }
        return;
    }

    const int wg = warp >> 2, wq = warp & 3;
    using Acc = typename std::conditional<I8, int, float>::type;
    Acc acc[64];
    int it = 0;
    for (int nt = nt0; nt < nt1; ++nt) {
        const int n0 = nt * BN;
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = 0;
        for (int kt = 0; kt < ktiles; ++kt, ++it) {
            const int s = it % STAGES;
            mbar_wait(bar_full + 8 * s, (it / STAGES) & 1);
            const uint32_t sa = base + (uint32_t)s * STAGE_BYTES + (uint32_t)wg * (64 * KB);
            const uint32_t sb = base + (uint32_t)s * STAGE_BYTES + OP_BYTES;
            wg_fence_regs(acc);
            wg_fence();
#pragma unroll
            for (int ks = 0; ks < KB / 32; ++ks) {   // one wgmma consumes 32 bytes of K
                const uint64_t da = wg_desc_sw128(sa + 32 * ks), db = wg_desc_sw128(sb + 32 * ks);
                if constexpr (I8) wgmma_m64n128k32_s8(acc, da, db, 1);
                else wgmma_m64n128k16_f16(acc, da, db, 1);
            }
            wg_commit();
            if (kt > 0) {   // the previous stage's MMAs are done: hand its buffers back to the producer
                wg_wait<1>();
                if (lane == 0) mbar_arrive(bar_empty + 8 * ((it - 1) % STAGES));
            }
        }
        wg_wait<0>();
        wg_fence_regs(acc);
        if (lane == 0) mbar_arrive(bar_empty + 8 * ((it - 1) % STAGES));

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
            continue;
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
}

// 2-D tensor map of a K-major operand: `rows` rows of `k` elements, `ld_bytes` apart (rows may overlap), boxes of one
// 128-byte K slice x 128 rows, 128-byte swizzle, zero fill outside the tensor
int make_tma(CUtensorMap* map, const void* ptr, bool i8, long long k, long long rows, long long ld_bytes) {
    static PFN_cuTensorMapEncodeTiled_v12000 encode = nullptr;
    if (!encode) {
        cudaDriverEntryPointQueryResult q;
        void* fn = nullptr;
        B200_CHECK_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
        B200_REQUIRE(q == cudaDriverEntryPointSuccess && fn, "gemm: cuTensorMapEncodeTiled is not available");
        encode = (PFN_cuTensorMapEncodeTiled_v12000)fn;
    }
    const cuuint64_t dims[2] = {(cuuint64_t)k, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)ld_bytes};
    const cuuint32_t box[2] = {(cuuint32_t)(i8 ? KB : KB / 2), (cuuint32_t)BM};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = encode(map, i8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr),
                              dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    B200_REQUIRE(r == CUDA_SUCCESS, "gemm: cuTensorMapEncodeTiled failed (%d) for k=%lld rows=%lld ld=%lld bytes", (int)r, k,
                 rows, ld_bytes);
    return 0;
}

template <bool I8>
int launch(const void* A, long long lda_bytes, const void* B, const float* col_scale, __half* C, long long ldc, int M, int N,
           int K_bytes, const GemmEpilogue& ep, cudaStream_t stream) {
    static bool configured = false;
    static int sms = 0;
    if (!configured) {
        B200_CHECK_CUDA(cudaFuncSetAttribute(gemm_wgmma_kernel<I8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
        int dev = 0;
        B200_CHECK_CUDA(cudaGetDevice(&dev));
        B200_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        configured = true;
    }
    const int es = I8 ? 1 : 2;
    CUtensorMap ta, tb;
    int rc = make_tma(&ta, A, I8, K_bytes / es, M, lda_bytes);
    if (rc) return rc;
    rc = make_tma(&tb, B, I8, K_bytes / es, N, K_bytes);
    if (rc) return rc;
    // a CTA sweeps all column tiles of its row block unless that leaves fewer than ~4 waves of CTAs (small M): then the
    // column tiles are split into runs over blockIdx.y
    const int mblocks = (M + BM - 1) / BM, ntiles = (N + BN - 1) / BN;
    int per = ntiles;
    while (per > 1 && (long long)mblocks * ((ntiles + per - 1) / per) < 8LL * sms) per = (per + 1) / 2;
    dim3 grid(mblocks, (ntiles + per - 1) / per);
    gemm_wgmma_kernel<I8><<<grid, THREADS, SMEM_BYTES, stream>>>(ta, tb, col_scale, C, ldc, M, N, K_bytes, per, ep);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace

// max_ctas is accepted for the ABI and not needed here: the kernel is not persistent, a CTA leaves once its row block's
// column tiles are done and the block scheduler hands the SMs to whatever else is queued.  For the hac input projection
// (12 column tiles per CTA) that is about 0.28 ms on average: 7.0 ms alone on an H100 80GB HBM3 (700 W) for 6664 CTAs,
// 2 x 132 resident at a time.  scripts/step_timeline.py shows no steady-state recurrent launch of the two-batch hac step
// starting later after its input projection than with the previous one-tile-per-CTA kernel (both within 0.01 ms).
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
