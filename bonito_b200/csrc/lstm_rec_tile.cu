// Persistent recurrent part of one LSTM layer on the Hopper tensor cores (hac: H = 384), tile layout.
// Reference semantics: bonito/nn.py:353-415 (torch.nn.LSTM, gate order i,f,g,o, zero initial state, optional
// time reversal), the span `Model.use_koi` hands to koi.lstm (bonito/crf/model.py:240-246).
//
// Decomposition:
//   * a cluster of CS = 8 CTAs owns one batch tile of NB = 64 chunks for all T steps; CTA `rank` owns hidden units
//     [48 rank, 48 rank + 48) = 192 gate columns.  Its slice of W_hh (192 x 384 fp16 = 144 KB) stays in shared memory
//     for the whole kernel, next to the h tile of the step (64 chunks x 384 = 48 KB): 8 CTAs is the smallest cluster
//     whose slice and h tile fit the 227 KB an H100 CTA may have.
//   * per step the gate pre-activations are ONE product per warpgroup, gates^T = h_{t-1} [64 x 384] . W_slice^T:
//     wgmma m64n96k16 x 24, A = the h tile, B = this warpgroup's 96 gate columns, fp32 accumulators in registers.
//     The B rows are ordered so that 8-column block 2p holds (i, f) and block 2p + 1 holds (g, o) of the same four units
//     (unit 4p + lane%4 in a thread's columns 2(lane%4) + {0,1}): one thread holds all four gates of its (chunk, unit)
//     cells -- 2 chunks x 6 units -- and updates (c, h) in registers with no exchange inside the CTA.
//   * both operands are K-major without swizzle, [16-byte k-chunk][row][16 B], so the 48 units one CTA produces are
//     six k-chunks = 6 KB contiguous in every peer's h tile.
//   * h all-gather: the CTA stages its 6 KB block in global memory (it stays in L2) and ONE elected thread issues a
//     multicast bulk copy (cp.async.bulk ... .multicast::cluster) that lands it in the h tile of all eight CTAs and
//     completes 6 KB on each CTA's mbarrier.  The h tile is single-buffered: a cluster barrier (arrive right after the
//     CTA's wgmma of the step has drained, wait just before the copy) keeps the copies of step t from overwriting an
//     h_{t-1} a peer is still reading; the cell update runs between the arrive and the wait.
//   * gx of the next step is loaded into registers while the tensor cores work on this one.
//
// Operands: whh [4H][H] rows permuted [unit/8][gate][unit%8] (the order the generic kernel uses; the kernel picks its rows);
//           gx  [tile][T][8][64][192]  columns of rank r = [unit - 48r][gate];   y [tile][T][64][H].
#include "tc_common.cuh"

namespace {

constexpr int H = 384, CS = 8, UPC = H / CS, COLS = 4 * UPC, NB = 64;
constexpr int WG_COLS = COLS / 2;                    // 96 columns (24 units) per warpgroup
constexpr int PAIRS = WG_COLS / 16;                  // 6 (i,f | g,o) block pairs per warpgroup
constexpr int THREADS = 256;
constexpr int KCH = H / 8;                           // 48 k-chunks
constexpr uint32_t W_BYTES = KCH * COLS * 16;        // 147456
constexpr uint32_t HT_BYTES = KCH * NB * 16;         // 49152
constexpr uint32_t BLK_BYTES = (UPC / 8) * NB * 16;  // 6144: this CTA's block of the h tile
constexpr uint32_t OFF_W = 0, OFF_H = OFF_W + W_BYTES, OFF_ST = OFF_H + HT_BYTES, OFF_BAR = OFF_ST + BLK_BYTES;
constexpr uint32_t SMEM_BYTES = OFF_BAR + 16;
static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget");

__device__ __forceinline__ void bulk_multicast(uint32_t dst, const void* gsrc, uint32_t bytes, uint32_t bar, uint16_t mask) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;\n" ::
            "r"(dst), "l"(gsrc), "r"(bytes), "r"(bar), "h"(mask)
        : "memory");
}
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;\n" ::: "memory"); }
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;\n" ::: "memory"); }

__global__ void __cluster_dims__(CS, 1, 1) __launch_bounds__(THREADS, 1)
lstm_rec_tile_kernel(const __half* __restrict__ gx, const __half* __restrict__ whh, __half* __restrict__ y,
                     unsigned char* __restrict__ hx, int T, int N, int reverse) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const uint32_t base = smem_u32(smem_raw);
    const uint32_t hbar = base + OFF_BAR;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wg = warp >> 2, wq = warp & 3, q = lane & 3;
    const uint32_t rank = cluster_ctarank();
    const int tile = blockIdx.x / CS;
    const int nb = min(NB, N - tile * NB);   // valid chunks of this tile
    gx += (size_t)tile * T * (CS * NB * COLS) + (size_t)rank * (NB * COLS);
    y += (size_t)tile * T * (NB * H);
    hx += (size_t)(tile * CS + (int)rank) * 2 * BLK_BYTES;   // this CTA's exchange staging: [parity][6 KB]

    if (tid == 0) {
        mbar_init(hbar, 1);
        mbar_fence_init();
    }
    // resident W_hh slice: smem row n = [warpgroup][pair p][(i,f) | (g,o)][unit 4p + n%8/2][gate n%2]
    {
        const __half* wsrc = whh;
        for (int i = tid; i < COLS * KCH; i += THREADS) {
            const int n = i % COLS, kc = i / COLS;
            const int g = n / WG_COLS, m = n % WG_COLS, p = m / 16, half = (m % 16) / 8, e = m % 8;
            const int unit = (int)rank * UPC + g * (UPC / 2) + 4 * p + (e >> 1), gate = 2 * half + (e & 1);
            const int src_row = (unit >> 3) * 32 + gate * 8 + (unit & 7);
            cp_async_16(smem_raw + OFF_W + (uint32_t)kc * (COLS * 16) + (uint32_t)n * 16, wsrc + (size_t)src_row * H + kc * 8, true);
        }
        cp_async_commit();
        cp_async_wait<0>();
        fence_proxy_async_smem();
    }
    __syncthreads();
    cluster_sync_all();   // every CTA's barrier is initialised before any peer's copy can land

    // this thread's cells: chunks ch[h] = 16 wq + lane/4 + 8h, units ul[p] = 24 wg + 4p + q (CTA-local)
    const int ch0 = wq * 16 + (lane >> 2);
    const int ul0 = wg * (UPC / 2) + q;
    float c_state[PAIRS][2];
#pragma unroll
    for (int p = 0; p < PAIRS; ++p) c_state[p][0] = c_state[p][1] = 0.f;
    auto load_gx = [&](int step, uint2 (&g)[PAIRS][2]) {
        const int t = reverse ? (T - 1 - step) : step;
        const __half* src = gx + (size_t)t * (CS * NB * COLS);
#pragma unroll
        for (int p = 0; p < PAIRS; ++p)
#pragma unroll
            for (int h = 0; h < 2; ++h)
                g[p][h] = __ldg(reinterpret_cast<const uint2*>(src + (size_t)(ch0 + 8 * h) * COLS + (ul0 + 4 * p) * 4));
    };
    uint2 gnext[PAIRS][2];
    load_gx(0, gnext);

    const uint64_t da0 = wg_desc_noswz(base + OFF_H, NB * 16, 128);
    const uint64_t db0 = wg_desc_noswz(base + OFF_W + (uint32_t)wg * (WG_COLS * 16), COLS * 16, 128);
    float acc[48];
    for (int step = 0; step < T; ++step) {
        const int t = reverse ? (T - 1 - step) : step;
        const int par = step & 1;
        uint2 g[PAIRS][2];
#pragma unroll
        for (int p = 0; p < PAIRS; ++p) g[p][0] = gnext[p][0], g[p][1] = gnext[p][1];
#pragma unroll
        for (int i = 0; i < 48; ++i) acc[i] = 0.f;
        if (step > 0) {   // h_{-1} = 0: nothing to multiply at step 0
            mbar_wait(hbar, (uint32_t)((step - 1) & 1));
            wg_fence_regs(acc);
            wg_fence();
#pragma unroll
            for (int ks = 0; ks < H / 16; ++ks)   // one k16 step = two k-chunks
                wgmma_m64n96k16_f16(acc, da0 + (uint64_t)(ks * 2 * NB * 16 / 16), db0 + (uint64_t)(ks * 2 * COLS * 16 / 16), 1);
            wg_commit();
            if (step + 1 < T) load_gx(step + 1, gnext);   // off the critical path: in flight during the MMAs
            wg_wait<0>();
            wg_fence_regs(acc);
        } else if (step + 1 < T) {
            load_gx(step + 1, gnext);
        }
        if (step + 1 < T) cluster_arrive();   // this CTA is done reading h_{t-1}

#pragma unroll
        for (int p = 0; p < PAIRS; ++p)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const __half2 g01 = *reinterpret_cast<const __half2*>(&g[p][h].x);
                const __half2 g23 = *reinterpret_cast<const __half2*>(&g[p][h].y);
                const float ai = acc[(2 * p) * 4 + h * 2] + __low2float(g01);
                const float af = acc[(2 * p) * 4 + h * 2 + 1] + __high2float(g01);
                const float ag = acc[(2 * p + 1) * 4 + h * 2] + __low2float(g23);
                const float ao = acc[(2 * p + 1) * 4 + h * 2 + 1] + __high2float(g23);
                float si, sf, tg, so;
                gate_activations(ai, af, ag, ao, si, sf, tg, so);
                const float c = fmaf(sf, c_state[p][h], si * tg);
                c_state[p][h] = c;
                const int ul = ul0 + 4 * p, chunk = ch0 + 8 * h;
                *reinterpret_cast<__half*>(smem_raw + OFF_ST + (uint32_t)(ul >> 3) * (NB * 16) + (uint32_t)chunk * 16 +
                                           (uint32_t)(ul & 7) * 2) = __float2half_rn(so * tanh_f(c));
            }
        __syncthreads();   // the block of h_t is staged
        unsigned char* stg = hx + (size_t)par * BLK_BYTES;
        for (int i = tid; i < (int)(BLK_BYTES / 16); i += THREADS) {
            const uint4 v = *reinterpret_cast<const uint4*>(smem_raw + OFF_ST + (uint32_t)i * 16);
            if (step + 1 < T) reinterpret_cast<uint4*>(stg)[i] = v;
            const int kc = i / NB, chunk = i % NB;
            if (chunk < nb) *reinterpret_cast<uint4*>(y + ((size_t)t * NB + chunk) * H + rank * UPC + kc * 8) = v;
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

}  // namespace

int lstm_rec_tile_chunks(int hidden) { return hidden == H ? NB : 0; }
int lstm_rec_tile_cluster(int hidden) { return hidden == H ? CS : 0; }
size_t lstm_rec_tile_workspace_bytes(int N) { return (size_t)((N + NB - 1) / NB) * CS * 2 * BLK_BYTES; }

// gx [tiles][T][8][64][192], y [tiles][T][64][H]; tiles = ceil(N / 64), the last one may be partial;
// workspace: lstm_rec_tile_workspace_bytes(N) bytes of exchange staging (contents irrelevant)
int launch_lstm_rec_tile(const __half* gx, const __half* whh, __half* y, void* workspace, int T, int N, int hidden,
                         int reverse, cudaStream_t stream) {
    B200_REQUIRE(hidden == H, "lstm_rec_tile: hidden size %d is not supported (384)", hidden);
    B200_REQUIRE(((uintptr_t)gx % 16) == 0 && ((uintptr_t)y % 16) == 0 && ((uintptr_t)whh % 16) == 0 &&
                     ((uintptr_t)workspace % 16) == 0,
                 "lstm_rec_tile: operands must be 16-byte aligned");
    static bool configured = false;
    if (!configured) {
        B200_CHECK_CUDA(cudaFuncSetAttribute(lstm_rec_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
        configured = true;
    }
    const int tiles = (N + NB - 1) / NB;
    lstm_rec_tile_kernel<<<tiles * CS, THREADS, SMEM_BYTES, stream>>>(gx, whh, y, (unsigned char*)workspace, T, N, reverse);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}
