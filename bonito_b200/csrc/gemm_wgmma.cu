// C[M,N] = epilogue(A[M,K] * B[N,K]^T) on the Hopper tensor cores (wgmma, sm_90a): the product GEMM of every
// convolution-as-GEMM, LSTM input projection, CRF head and transformer projection.
//
//   * a CTA owns one 128-row block of A and sweeps a run of up to MAX_RUN 128-column tiles of N through one pipeline:
//     while it rounds and stores tile j, the next tile's operands are already arriving.  The runs of a row block are
//     consecutive CTAs, so they are resident together: they read the same A rows from L2 and write neighbouring parts
//     of the same output rows;
//   * one producer warp fills a 3-deep ring of stages with TMA copies (128-byte K slices -- 64 fp16 or 128 int8 -- of 128
//     rows of A and of B, 128-byte swizzle), signalling through mbarriers ("full": bytes landed, "empty": every consumer
//     warp is done with the stage);
//   * two consumer warpgroups of 64 rows each issue wgmma.mma_async m64n128 (fp16: k16, int8: k32) with both operands in
//     shared memory, fp32 / s32 accumulators in registers (64 per thread), keeping one stage's MMAs in flight while the
//     next one is issued (wgmma.wait_group 1).  Every accumulator sums its K steps in ascending order;
//   * two CTAs per SM (105 KB of shared memory each), so one CTA's epilogue overlaps the other's MMAs;
//   * the epilogue computes on the accumulator fragment in registers (thread = rows lane/4 and lane/4 + 8 of its warp's
//     16 rows, columns 8j + 2(lane%4) + {0,1}): bias, fp16 rounding, activation and the fused SwiGLU (a 64-column
//     group [32 y | 32 gate] lies in one thread's columns); it stores through a 1 KB buffer per warp, 16 rows x 32
//     columns at a time, in 16-byte row segments placed by the row / column-block maps of GemmEpilogue (store_block).
//
// Measured alone on an H100 80GB HBM3 (700 W), the shapes with large outputs reach 22-32 % of their HBM floor (hac CRF
// head 2.77 ms against 0.72 ms, strided conv 1.09 against 0.24, sup CRF head 5.69 against 1.81).  The rest of their time
// has not been broken down; every column tile still re-reads its CTA's A row block from L2.
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
// column tiles per CTA at most.  Runs of 2 were faster alone than runs of all the tiles of a row block on every large
// shape of the benchmarked workloads (H100 80GB HBM3, 700 W: hac CRF head 2.76 against 2.87 ms, sup fc2 1.04 against
// 1.31 ms, sup CRF head 6.33 against 6.69 ms), and than runs of 1 or 4 on most of them.
constexpr int MAX_RUN = 2;
constexpr int CONSUMERS = 256, THREADS = CONSUMERS + 32;   // two consumer warpgroups + one producer warp
constexpr uint32_t OP_BYTES = BM * KB;               // one operand slice: 16 KB
constexpr uint32_t STAGE_BYTES = 2 * OP_BYTES;
constexpr uint32_t EPI_BYTES = 16 * 32 * 2;          // a consumer warp's epilogue buffer: 16 rows x 32 fp16 columns
// alignment slack + ring + 2 x STAGES mbarriers + the epilogue buffers.  Two CTAs fit on an SM (2 x (105 KB + 1 KB
// reserved) of 228 KB); 16 KB of buffers (64 columns per warp) would leave one.
constexpr uint32_t SMEM_BYTES = 1024 + STAGES * STAGE_BYTES + 64 + (CONSUMERS / 32) * EPI_BYTES;

__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
    const __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<const uint32_t*>(&h);
}

// Writes a 16-row x 32-column block of the warp's results to output columns c0 .. c0 + 31 (those below n_out) of its
// rows; orow[h]: output row of row lane/4 + 8h (-1: not written).  v[2 jj + h] is the lane's accumulator-fragment pair
// (row lane/4 + 8h, columns 8 jj + 2(lane%4), +1).  The pairs pass through the warp's buffer `buf` (64-byte rows, 16-byte
// chunk c of row r at chunk c ^ (r/2 % 4), so that neither stmatrix nor the read-back has bank conflicts) and come back
// as one 16-byte chunk per lane: each store instruction writes 8 rows x 64 contiguous bytes, whole 32-byte sectors,
// where a store of the fragment itself writes 8 rows x 16 bytes.  A column block (cb_width, a multiple of 32) never
// splits the 32 columns.
__device__ __forceinline__ void store_block(const uint32_t (&v)[8], uint32_t buf, int lane, const long long (&orow)[2], int c0,
                                            int n_out, __half* C, long long ldc, const GemmEpilogue& ep) {
    __syncwarp();   // every lane has read the previous block out of the buffer
    {
        const int q = lane >> 3, row = 8 * (q & 1) + (lane & 7), sw = (row >> 1) & 3;   // matrix q: (jj = 2k + q/2, h = q%2)
#pragma unroll
        for (int k = 0; k < 2; ++k)
            stmatrix_x4(buf + row * 64 + 16 * ((2 * k + (q >> 1)) ^ sw), v[4 * k], v[4 * k + 1], v[4 * k + 2], v[4 * k + 3]);
    }
    __syncwarp();
    const int c = lane & 3, col = c0 + 8 * c;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int row = 8 * h + (lane >> 2);
        const uint4 d = ld_shared_v4(buf + row * 64 + 16 * (c ^ ((row >> 1) & 3)));
        if (orow[h] < 0 || col >= n_out) continue;
        long long drow = orow[h];
        int dcol = col;
        if (ep.cb_width > 0) {   // column-block remap
            const int cb = col / ep.cb_width;
            drow += (long long)cb * ep.cb_rows;
            dcol = col - cb * ep.cb_width;
        }
        *reinterpret_cast<uint4*>(C + drow * ldc + dcol) = d;
    }
}

template <bool I8>
__global__ void __launch_bounds__(THREADS, 2)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
                  const float* __restrict__ col_scale, __half* __restrict__ C, long long ldc, int M, int N, int K_bytes,
                  int tiles_per_cta, GemmEpilogue ep) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;   // the 128-byte swizzle repeats every 1024 bytes
    const uint32_t bar_full = base + STAGES * STAGE_BYTES, bar_empty = bar_full + 8 * STAGES;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nruns = (N + BN * tiles_per_cta - 1) / (BN * tiles_per_cta);
    const int m0 = (int)(blockIdx.x / nruns) * BM;
    const int ntiles = (N + BN - 1) / BN;
    const int nt0 = (int)(blockIdx.x % nruns) * tiles_per_cta, nt1 = min(ntiles, nt0 + tiles_per_cta);
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
    const uint32_t stage = bar_full + 64 + (uint32_t)warp * EPI_BYTES;
    const int cq = 2 * (lane & 3);
    long long orow[2];   // output rows of the lane's two rows (the same for every column tile)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int gm = m0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
        orow[h] = gm < M ? map_row(ep.map, gm) : -1;
    }
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

        // 32-column blocks of the tile (SwiGLU: one per 64-column group, 32 outputs), each rounded into fp16 pairs
        // v[2 jj + h] = (row lane/4 + 8h, columns 8 jj + cq, +1 of the block) and written by store_block
        if (!I8 && ep.act == B200_ACT_SWIGLU) {
            // 64-column group G of the tile: y = columns 8j' + cq + e, gate = 32 + the same; output column (n0 + 64G) / 2 + ...
#pragma unroll
            for (int G = 0; G < 2; ++G) {
                const int c0 = (n0 + 64 * G) / 2;
                if (c0 >= N / 2) continue;
                uint32_t v[8];
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) {
                    const int jy = 8 * G + jj, jg = jy + 4;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const float y0 = round_f16((float)acc[jy * 4 + h * 2]), y1 = round_f16((float)acc[jy * 4 + h * 2 + 1]);
                        const float g0 = round_f16((float)acc[jg * 4 + h * 2]), g1 = round_f16((float)acc[jg * 4 + h * 2 + 1]);
                        v[2 * jj + h] = pack_half2(g0 * y0 * rcp_approx(1.0f + __expf(-g0)), g1 * y1 * rcp_approx(1.0f + __expf(-g1)));
                    }
                }
                store_block(v, stage, lane, orow, c0, N / 2, C, ldc, ep);
            }
            continue;
        }
#pragma unroll
        for (int p = 0; p < 4; ++p) {
            const int c0 = n0 + 32 * p;
            if (c0 >= N) continue;
            uint32_t v[8];
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
                const int j = 4 * p + jj;
                const int gn = n0 + 8 * j + cq;   // N % 8 == 0: the pair (gn, gn + 1) is in range together
                const bool in = gn < N;           // pairs past N are computed from zeros and never stored
                float s0 = 0.f, s1 = 0.f, b0 = 0.f, b1 = 0.f;
                if (in && ep.bias) {
                    b0 = __half2float(ep.bias[gn]);
                    b1 = __half2float(ep.bias[gn + 1]);
                }
                if constexpr (I8) {
                    if (in) {
                        s0 = col_scale[gn];
                        s1 = col_scale[gn + 1];
                    }
                }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float v0, v1;
                    if constexpr (I8) {
                        v0 = fmaf((float)acc[j * 4 + h * 2], s0, b0);
                        v1 = fmaf((float)acc[j * 4 + h * 2 + 1], s1, b1);
                    } else {
                        v0 = acc[j * 4 + h * 2];
                        v1 = acc[j * 4 + h * 2 + 1];
                        if (ep.bias) {
                            v0 += b0;
                            v1 += b1;
                        }
                    }
                    v[2 * jj + h] = pack_half2(apply_act_f16(v0, ep.act, ep.lo, ep.hi), apply_act_f16(v1, ep.act, ep.lo, ep.hi));
                }
            }
            store_block(v, stage, lane, orow, c0, N, C, ldc, ep);
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
    // runs of MAX_RUN column tiles, shorter when that leaves fewer than ~4 waves of CTAs (small M); CTA b takes run
    // b % runs of row block b / runs
    const int mblocks = (M + BM - 1) / BM, ntiles = (N + BN - 1) / BN;
    int per = ntiles < MAX_RUN ? ntiles : MAX_RUN;
    while (per > 1 && (long long)mblocks * ((ntiles + per - 1) / per) < 8LL * sms) per = (per + 1) / 2;
    dim3 grid(mblocks * ((ntiles + per - 1) / per));
    gemm_wgmma_kernel<I8><<<grid, THREADS, SMEM_BYTES, stream>>>(ta, tb, col_scale, C, ldc, M, N, K_bytes, per, ep);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace

// max_ctas is accepted for the ABI and not needed here: the kernel is not persistent, a CTA leaves once its run of
// column tiles is done and the block scheduler hands the SMs to whatever else is queued.
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
