// One whole LSTM layer of width 384 (hac) on the Hopper tensor cores, tile layout: the input projection x_t W_ih^T + b is
// computed inside the persistent recurrence instead of by a GEMM ahead of it, so the gate pre-activations never go to HBM.
// Reference semantics: bonito/nn.py:353-415 (torch.nn.LSTM, gate order i,f,g,o, zero initial state, optional time reversal).
//
// Decomposition (as lstm_rec_tile.cu): a cluster of CS = 8 CTAs owns one batch tile of NB = 64 chunks for all T steps;
// CTA `rank` owns hidden units [48 rank, 48 rank + 48) = 192 gate rows, and the h all-gather (staging block in global
// memory, one multicast bulk copy per CTA, single-buffered h tile guarded by a cluster barrier) is the same protocol.
// What differs is the orientation and where the operands live:
//   * gates [192 rows x 64 chunks] = W . [x_t | h_{t-1}]^T, three warpgroups of 64 gate rows, wgmma m64n64k16 with the
//     weights as A and the activation tile as B (K-major, N = chunks).  The h tile [k-chunk][chunk][16 B] is a valid
//     no-swizzle K-major B operand, so the exchange writes it exactly as before;
//   * W_hh (this warpgroup's 64 rows x 384) stays in registers as A fragments for the whole kernel: 24 k16 steps x 4;
//   * W_ih (192 x 384 = 144 KB) stays in shared memory as a no-swizzle K-major A operand;
//   * x_t comes from the previous layer's output [tile][T][64][H] by TMA: six 64-chunk x 64-column boxes (8 KB, 128-byte
//     swizzle) per step through a ring of RING boxes that the MMAs of the x product release one by one.  The ring holds
//     half a step, so each step's last three boxes are loaded while its first three are consumed; the cluster pulls
//     every box into L2 PREFETCH steps ahead, so that those loads wait on L2 and not on HBM;
//   * A row m of warpgroup wg is unit 16 wg + 4 (m/16) + (m%8)/2 (CTA-local), gate 2 (m%2) + (m%16)/8: the two rows a thread
//     holds are (i, f) of a unit in even quads and (g, o) of the same unit in the odd quad next to it.  One __shfl_xor(4)
//     per value pair then gives every thread all four gates of 8 cells (even quads take the even chunk of each column pair,
//     odd quads the odd one).
// Schedule of a step: the x product of step t (its operands do not depend on h), bias and fp16 rounding of it -- exactly
// the GEMM epilogue, so the gate pre-activations are bit-identical to b200_gemm_fwd_ex + lstm_rec_tile -- then the wait
// for h_{t-1}, the W_hh product from zero, and acc + float(gx) per gate as lstm_rec_tile does.  The x product runs while
// the peers' blocks of h_{t-1} are still in flight.  y of step t-1 is written from this CTA's block of h_{t-1} in the h
// tile while the W_hh product runs; only the last step writes y from the staging block.
//
// Operands: x [tiles][T][64][H] fp16; wih [4H][H] and bias [4H] rows in [unit][gate] order (the gx column order of the
// unfused path); whh [4H][H] rows [unit/8][gate][unit%8]; y [tiles][T][64][H].
#include <cuda.h>
#include <cudaTypedefs.h>

#include "tc_common.cuh"

namespace {

constexpr int H = 384, CS = 8, UPC = H / CS, ROWS = 4 * UPC, NB = 64;
constexpr int THREADS = 384;                         // three warpgroups x 64 gate rows (16 units)
constexpr int KCH = H / 8;                           // 48 k-chunks of 16 bytes
constexpr int KS = H / 16;                           // 24 k16 steps
constexpr int XBOX = H / 64;                         // x boxes per step: 64 columns (128 bytes) x 64 chunks
constexpr int RING = 3;
constexpr int PREFETCH = 2;                          // steps of x pulled into L2 ahead of the step that reads them
constexpr uint32_t XBOX_BYTES = NB * 128;            // 8192
constexpr uint32_t W_BYTES = KCH * ROWS * 16;        // 147456
constexpr uint32_t HT_BYTES = KCH * NB * 16;         // 49152
constexpr uint32_t BLK_BYTES = (UPC / 8) * NB * 16;  // 6144: this CTA's block of the h tile
constexpr uint32_t OFF_X = 0, OFF_W = OFF_X + RING * XBOX_BYTES, OFF_H = OFF_W + W_BYTES, OFF_ST = OFF_H + HT_BYTES,
                   OFF_BAR = OFF_ST + BLK_BYTES;     // barriers: h, full[RING], empty[RING]
constexpr uint32_t SMEM_BYTES = 1024 + OFF_BAR + 8 * (1 + 2 * RING);   // + slack to align the x ring to 1024 bytes
static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget");

__device__ __forceinline__ void bulk_multicast(uint32_t dst, const void* gsrc, uint32_t bytes, uint32_t bar, uint16_t mask) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;\n" ::
            "r"(dst), "l"(gsrc), "r"(bytes), "r"(bar), "h"(mask)
        : "memory");
}
// pull a box of the tensor into L2 ahead of its TMA load (no shared memory, no completion to wait for)
__device__ __forceinline__ void tma_prefetch_l2_2d(const void* tmap, int c0, int c1) {
    asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];\n" ::"l"(reinterpret_cast<uint64_t>(tmap)),
                 "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;\n" ::: "memory"); }
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;\n" ::: "memory"); }

// A row m (0..191) of this CTA -> (CTA-local unit, gate)
__device__ __forceinline__ void row_unit_gate(int m, int& ul, int& gate) {
    const int r = m % 16;
    ul = (m / 64) * 16 + (m % 64) / 16 * 4 + (r % 8) / 2;
    gate = 2 * (r % 2) + r / 8;
}

__global__ void __cluster_dims__(CS, 1, 1) __launch_bounds__(THREADS, 1)
lstm_fused_tile_kernel(const __grid_constant__ CUtensorMap tma_x, const __half* __restrict__ wih,
                       const __half* __restrict__ bias, const __half* __restrict__ whh, __half* __restrict__ y,
                       unsigned char* __restrict__ hx, int T, int N, int reverse) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    const uint32_t raw = smem_u32(smem_raw), base = (raw + 1023u) & ~1023u;   // the 128-byte swizzle repeats every 1 KB
    unsigned char* smem = smem_raw + (base - raw);
    const uint32_t hbar = base + OFF_BAR, full = hbar + 8, empty = full + 8 * RING;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wg = warp >> 2, wq = warp & 3, q = lane & 3;
    const int odd = (lane >> 2) & 1;
    const uint32_t rank = cluster_ctarank();
    const int tile = blockIdx.x / CS;
    const int nb = min(NB, N - tile * NB);   // valid chunks of this tile
    const int xrow0 = tile * T * NB;         // first x row of this tile
    const int boxes = T * XBOX;
    y += (size_t)tile * T * (NB * H);
    hx += (size_t)(tile * CS + (int)rank) * 2 * BLK_BYTES;   // this CTA's exchange staging: [parity][6 KB]

    auto issue_box = [&](int li) {   // box li = (step li / XBOX, columns 64 (li % XBOX)) into ring slot li % RING
        const int step = li / XBOX, t = reverse ? (T - 1 - step) : step, s = li % RING;
        mbar_expect_tx(full + 8 * s, XBOX_BYTES);
        tma_load_2d(base + OFF_X + (uint32_t)s * XBOX_BYTES, &tma_x, (li % XBOX) * 64, xrow0 + t * NB, full + 8 * s);
    };
    // every warp is done with box li: once all twelve are, thread 0 refills its slot with box li + RING
    auto release_box = [&](int li) {
        const uint32_t e = empty + 8 * (li % RING);
        if (lane == 0) mbar_arrive(e);
        if (tid == 0 && li + RING < boxes) {
            mbar_wait(e, (uint32_t)((li / RING) & 1));
            issue_box(li + RING);
        }
    };
    if (tid == 0) {
        mbar_init(hbar, 1);
        for (int s = 0; s < RING; ++s) {
            mbar_init(full + 8 * s, 1);
            mbar_init(empty + 8 * s, THREADS / 32);
        }
        mbar_fence_init();
        for (int li = 0; li < min(RING, boxes); ++li) issue_box(li);
    }
    // resident W_ih slice: [k-chunk][row][16 B]
    for (int i = tid; i < ROWS * KCH; i += THREADS) {
        const int m = i % ROWS, kc = i / ROWS;
        int ul, gate;
        row_unit_gate(m, ul, gate);
        const int src_row = ((int)rank * UPC + ul) * 4 + gate;
        cp_async_16(smem + OFF_W + (uint32_t)kc * (ROWS * 16) + (uint32_t)m * 16, wih + (size_t)src_row * H + kc * 8, true);
    }
    cp_async_commit();
    // resident W_hh rows of this thread (A fragment rows lane/4 and lane/4 + 8 of the warp's 16), bias of the same rows
    const int m0 = wg * 64 + wq * 16 + (lane >> 2);
    int ul0, gate0, ul1, gate1;
    row_unit_gate(m0, ul0, gate0);
    row_unit_gate(m0 + 8, ul1, gate1);
    const int unit = (int)rank * UPC + ul0;   // ul1 == ul0
    const __half* w0 = whh + (size_t)((unit >> 3) * 32 + gate0 * 8 + (unit & 7)) * H + 2 * q;
    const __half* w1 = whh + (size_t)((unit >> 3) * 32 + gate1 * 8 + (unit & 7)) * H + 2 * q;
    uint32_t wa[KS][4];
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
        wa[ks][0] = __ldg(reinterpret_cast<const unsigned int*>(w0 + ks * 16));
        wa[ks][1] = __ldg(reinterpret_cast<const unsigned int*>(w1 + ks * 16));
        wa[ks][2] = __ldg(reinterpret_cast<const unsigned int*>(w0 + ks * 16 + 8));
        wa[ks][3] = __ldg(reinterpret_cast<const unsigned int*>(w1 + ks * 16 + 8));
    }
    const float bias0 = __half2float(bias[unit * 4 + gate0]), bias1 = __half2float(bias[unit * 4 + gate1]);
    cp_async_wait<0>();
    fence_proxy_async_smem();
    __syncthreads();
    cluster_sync_all();   // every CTA's barrier is initialised before any peer's copy can land

    // this thread's cells: unit ul0 (CTA-local), chunks 8j + 2q + odd
    float c_state[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) c_state[j] = 0.f;
    const uint64_t da_x = wg_desc_noswz(base + OFF_W + (uint32_t)wg * (64 * 16), ROWS * 16, 128);
    const uint64_t db_h = wg_desc_noswz(base + OFF_H, NB * 16, 128);
    float acc[32];
    for (int step = 0; step < T; ++step) {
        const int t = reverse ? (T - 1 - step) : step;
        const int par = step & 1;
        // L2 prefetch of x (see the header): CTA `rank` < XBOX pulls box `rank` of step + PREFETCH
        if (tid == 32 && (int)rank < XBOX && step + PREFETCH < T) {
            const int sp = step + PREFETCH;
            tma_prefetch_l2_2d(&tma_x, (int)rank * 64, xrow0 + (reverse ? (T - 1 - sp) : sp) * NB);
        }
        // x product: acc = W_ih rows . x_t^T, k ascending like the GEMM
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[i] = 0.f;
        wg_fence_regs(acc);
        wg_fence();
#pragma unroll
        for (int kb = 0; kb < XBOX; ++kb) {
            const int li = step * XBOX + kb, s = li % RING;
            mbar_wait(full + 8 * s, (uint32_t)((li / RING) & 1));
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
                wgmma_m64n64k16_f16(acc, da_x + (uint64_t)((kb * 8 + kk * 2) * ROWS * 16 / 16),
                                    wg_desc_sw128(base + OFF_X + (uint32_t)s * XBOX_BYTES + 32 * kk), 1);
            wg_commit();
            if (kb > 0) {   // the MMAs of the previous box are done
                wg_wait<1>();
                release_box(li - 1);
            }
        }
        wg_wait<0>();
        wg_fence_regs(acc);
        release_box(step * XBOX + XBOX - 1);
        // gate pre-activations of the step, rounded as the GEMM epilogue rounds them: gx[j][h] = rows h, chunks 8j + 2q + {0,1}
        __half2 gx[8][2];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            gx[j][0] = __floats2half2_rn(acc[j * 4] + bias0, acc[j * 4 + 1] + bias0);
            gx[j][1] = __floats2half2_rn(acc[j * 4 + 2] + bias1, acc[j * 4 + 3] + bias1);
        }

#pragma unroll
        for (int i = 0; i < 32; ++i) acc[i] = 0.f;
        if (step > 0) {   // h_{-1} = 0: nothing to multiply at step 0
            mbar_wait(hbar, (uint32_t)((step - 1) & 1));
            wg_fence_regs(acc);
            wg_fence();
#pragma unroll
            for (int ks = 0; ks < KS; ++ks)   // one k16 step = two k-chunks
                wgmma_m64n64k16_f16_rs(acc, wa[ks], db_h + (uint64_t)(ks * 2 * NB * 16 / 16));
            wg_commit();
            // while the MMAs run: y of the previous step from this CTA's own block of h_{t-1} in the h tile, so that
            // these stores are not in front of the fence that releases the staged block of h_t to its bulk copy
            const int tp = reverse ? (T - step) : (step - 1);
            for (int i = tid; i < (int)(BLK_BYTES / 16); i += THREADS) {
                const int kc = i / NB, chunk = i % NB;
                if (chunk < nb)
                    *reinterpret_cast<uint4*>(y + ((size_t)tp * NB + chunk) * H + rank * UPC + kc * 8) =
                        *reinterpret_cast<const uint4*>(smem + OFF_H + rank * BLK_BYTES + (uint32_t)i * 16);
            }
            wg_wait<0>();
            wg_fence_regs(acc);
        }
        if (step + 1 < T) cluster_arrive();   // this CTA is done reading h_{t-1}

        const int ul = ul0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float keep[2], recv[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const float a0 = acc[j * 4 + h * 2] + __low2float(gx[j][h]);
                const float a1 = acc[j * 4 + h * 2 + 1] + __high2float(gx[j][h]);
                keep[h] = odd ? a1 : a0;
                recv[h] = __shfl_xor_sync(0xffffffffu, odd ? a0 : a1, 4);
            }
            const float ai = odd ? recv[0] : keep[0], af = odd ? recv[1] : keep[1];
            const float ag = odd ? keep[0] : recv[0], ao = odd ? keep[1] : recv[1];
            float si, sf, tg, so;
            gate_activations(ai, af, ag, ao, si, sf, tg, so);
            const float c = fmaf(sf, c_state[j], si * tg);
            c_state[j] = c;
            const int chunk = 8 * j + 2 * q + odd;
            *reinterpret_cast<__half*>(smem + OFF_ST + (uint32_t)(ul >> 3) * (NB * 16) + (uint32_t)chunk * 16 +
                                       (uint32_t)(ul & 7) * 2) = __float2half_rn(so * tanh_f(c));
        }
        __syncthreads();   // the block of h_t is staged
        unsigned char* stg = hx + (size_t)par * BLK_BYTES;
        for (int i = tid; i < (int)(BLK_BYTES / 16); i += THREADS) {
            const uint4 v = *reinterpret_cast<const uint4*>(smem + OFF_ST + (uint32_t)i * 16);
            if (step + 1 < T) {
                reinterpret_cast<uint4*>(stg)[i] = v;
            } else {   // the last step's h_t is not exchanged: y straight from the staged block
                const int kc = i / NB, chunk = i % NB;
                if (chunk < nb) *reinterpret_cast<uint4*>(y + ((size_t)t * NB + chunk) * H + rank * UPC + kc * 8) = v;
            }
        }
        if (step + 1 == T) break;
        fence_proxy_async_global();   // the staged block (generic stores) -> visible to the bulk copy (async proxy)
        __syncthreads();
        cluster_wait();               // every CTA of the cluster has drained its reads of h_{t-1}
        if (tid == 0) {
            mbar_expect_tx(hbar, HT_BYTES);   // the eight blocks of h_t
            bulk_multicast(base + OFF_H + rank * BLK_BYTES, stg, BLK_BYTES, hbar, (uint16_t)((1u << CS) - 1u));
        }
    }
    cluster_sync_all();   // nobody leaves while a peer may still address this CTA's shared memory
}

// x viewed as rows [tiles * T * 64][H]: boxes of 64 columns (128 bytes) x 64 rows, 128-byte swizzle
int make_x_map(CUtensorMap* map, const __half* x, long long rows) {
    static PFN_cuTensorMapEncodeTiled_v12000 encode = nullptr;
    if (!encode) {
        cudaDriverEntryPointQueryResult qr;
        void* fn = nullptr;
        B200_CHECK_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr));
        B200_REQUIRE(qr == cudaDriverEntryPointSuccess && fn, "lstm_fused_tile: cuTensorMapEncodeTiled is not available");
        encode = (PFN_cuTensorMapEncodeTiled_v12000)fn;
    }
    const cuuint64_t dims[2] = {(cuuint64_t)H, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)H * 2};
    const cuuint32_t box[2] = {64, (cuuint32_t)NB};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(x), dims, strides, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    B200_REQUIRE(r == CUDA_SUCCESS, "lstm_fused_tile: cuTensorMapEncodeTiled failed (%d) for %lld rows", (int)r, rows);
    return 0;
}

}  // namespace

// x [tiles][T][64][H] (rows of chunks >= N are read, their results dropped), y [tiles][T][64][H]; tiles = ceil(N / 64);
// workspace: lstm_rec_tile_workspace_bytes(N) bytes of exchange staging (contents irrelevant)
int launch_lstm_fused_tile(const __half* x, const __half* wih, const __half* bias, const __half* whh, __half* y,
                           void* workspace, int T, int N, int hidden, int reverse, cudaStream_t stream) {
    B200_REQUIRE(hidden == H, "lstm_fused_tile: hidden size %d is not supported (384)", hidden);
    B200_REQUIRE(((uintptr_t)x % 16) == 0 && ((uintptr_t)y % 16) == 0 && ((uintptr_t)wih % 16) == 0 &&
                     ((uintptr_t)whh % 16) == 0 && ((uintptr_t)workspace % 16) == 0,
                 "lstm_fused_tile: operands must be 16-byte aligned");
    if (T == 0 || N == 0) return 0;
    static bool configured = false;
    if (!configured) {
        B200_CHECK_CUDA(cudaFuncSetAttribute(lstm_fused_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
        configured = true;
    }
    const int tiles = (N + NB - 1) / NB;
    CUtensorMap tx;
    const int rc = make_x_map(&tx, x, (long long)tiles * T * NB);
    if (rc) return rc;
    lstm_fused_tile_kernel<<<tiles * CS, THREADS, SMEM_BYTES, stream>>>(tx, wih, bias, whh, y, (unsigned char*)workspace, T,
                                                                         N, reverse);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}
