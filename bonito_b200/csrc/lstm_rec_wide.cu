// Persistent recurrent part of one LSTM layer for the wide models (H = 768: dna_r9.4.1@v3.1, H = 1024: dna_r10.4.1@v4.3) on
// the Hopper tensor cores, grid-wide.  Reference semantics: bonito/nn.py:353-415 (torch.nn.LSTM, gate order i,f,g,o, zero
// initial state, optional time reversal), the span `Model.use_koi` hands to koi.lstm (bonito/crf/model.py:240-246).
//
// Why a grid: W_hh is 4H x H fp16, 4.5 MiB at H = 768 and 8 MiB at H = 1024.  The cluster kernels (lstm_rec.cu,
// lstm_rec_tile.cu) keep it in the shared memory of one cluster, and even a 16-CTA cluster has only ~3.6 MB.  Here the
// weights are spread over G = H / 8 CTAs (96 or 128, one per SM) and h_t is exchanged through L2 every step.
//
// Decomposition (what ships):
//   * CTA g owns hidden units [8g, 8g + 8) = 32 gate columns.  Its W_hh slice (32 x H fp16: 48 / 64 KB) stays in shared
//     memory for the whole launch, K-major without swizzle, [16-byte k-chunk][row][16 B].  The rows are ordered as in
//     lstm_rec_tile.cu: 8-column block 2p holds (i, f) and block 2p + 1 holds (g, o) of units 4p + lane%4, so one thread
//     holds all four gates of its (chunk, unit) cells -- 2 chunks x 2 units per 64-chunk tile -- and updates (c, h) in
//     registers with the shared `gate_activations` / `tanh_f` cell math (same rounding as the other LSTM kernels).
//   * one warpgroup (128 threads) per CTA.  Per step and per 64-chunk tile: gates[64 x 32] = h_{t-1}[64 x H] . W_slice^T,
//     wgmma m64n32k16 x H/16, fp32 accumulators.  The cell state of every tile lives in shared memory (float4 per thread
//     and tile); gx of the tile is loaded into registers before its MMAs are issued.
//   * h exchange: CTA g writes its 8 units of h_t as one 16-byte k-chunk per chunk row into a global exchange buffer laid
//     out [parity][tile][k-chunk][64][16 B] (the no-swizzle K-major operand layout, so a tile's k-slice is contiguous),
//     and writes y.  Grid-wide step barrier: one `red.release.gpu` add per CTA on a counter in the workspace; one thread
//     spins with `ld.acquire.gpu` until all G CTAs have arrived, then `fence.proxy.async.global` orders the acquired
//     generic stores ahead of the async-proxy reads.  h_{t-1} then streams into shared memory as 8 KB bulk copies (8
//     k-chunks x 64 rows) through a ring of 8 mbarrier stages, so that the copies overlap the MMAs.  The exchange buffer
//     is double-buffered by step parity: the barrier of step t+1 orders every read of h_t before any write of h_{t+2}.
//   * clusters / multicast are NOT used in this version: every CTA reads the whole h_{t-1} from L2 itself, G x N x H x 2
//     bytes per step (24 MB at N = 96, H = 1024).  Fetching 1/8 of each slice per CTA with `.multicast::cluster` inside
//     8-CTA clusters would divide that by 8, but needs the cooperative launch together with a cluster dimension; the
//     cluster-free cooperative launch keeps the co-residency guarantee simple and is the baseline that variant must beat.
//     Measured on one H100 80GB HBM3 at a 400 W power limit (scripts/bench_lstm_wide.py, v4.3 shape, T = 1666): 7.7 us
//     per time step at N = 96 and 30.3 us at N = 512, against MMA-only bounds of 0.8 / 4.3 us (989 TFLOP/s data-sheet
//     rate): the L2 exchange and the barrier, not the tensor cores, set the pace.
//
// Co-residency is a correctness condition (CTAs spin on each other): the launch is cooperative (cudaLaunchKernelEx +
// cudaLaunchAttributeCooperative), so the runtime refuses a grid that cannot be co-resident instead of running it, and
// lstm_rec_wide_resident() lets the engine check the fit when it builds a plan.  Every inter-CTA wait is bounded by a
// deadline on %globaltimer (2 s, far above any time slice another context can take); on expiry the CTA sets the status
// word of the workspace and returns, every other CTA sees the status and returns too.  The counter and the status word
// are reset on the stream before each launch.
//
// Operands: whh [4H][H] rows permuted [unit/8][gate][unit%8] (as for the generic kernel);
//           gx  [T][G][N][32]  columns of CTA g = [unit - 8g][gate];   y [T][N][H].
#include "tc_common.cuh"

namespace {

constexpr int UPC = 8, COLS = 4 * UPC, NB = 64, THREADS = 128;
constexpr int KS = 8;                                  // k-chunks per bulk-copy slice
constexpr uint32_t SLICE_BYTES = KS * NB * 16;         // 8192
constexpr int STAGES = 8;
constexpr int MAX_TILES = 40;                          // cell state capacity: N <= 2560 chunks per launch
constexpr uint32_t C_BYTES = MAX_TILES * THREADS * 16;
constexpr uint32_t CTRL_BYTES = 256;                   // counter at +0, status word at +128
constexpr uint32_t STATUS_OFFSET = 128;
constexpr uint64_t DEADLINE_NS = 2000000000ull;

template <int H>
struct Geo {
    static constexpr int G = H / UPC, KCH = H / 8, SLICES = KCH / KS;
    static constexpr uint32_t W_BYTES = KCH * COLS * 16;
    static constexpr uint32_t TILE_BYTES = KCH * NB * 16;   // one tile of h in the exchange buffer
    static constexpr uint32_t OFF_W = 0, OFF_RING = OFF_W + W_BYTES, OFF_C = OFF_RING + STAGES * SLICE_BYTES,
                              OFF_STG = OFF_C + C_BYTES, OFF_BAR = OFF_STG + NB * 16, OFF_FLAG = OFF_BAR + STAGES * 8;
    static constexpr uint32_t SMEM_BYTES = OFF_FLAG + 16;
    static_assert(KCH % KS == 0, "slices must tile H");
    static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget");
};

__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* gsrc, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(dst),
                 "l"(gsrc), "r"(bytes), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;\n" ::: "memory"); }
__device__ __forceinline__ uint64_t globaltimer() {
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;\n" : "=l"(t));
    return t;
}
__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];\n" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void red_release_gpu_add(unsigned* p, unsigned v) {
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;\n" ::"l"(p), "r"(v) : "memory");
}

// spin until `*counter >= target`; false (and the status word set) once the deadline passes or another CTA gave up
__device__ bool grid_wait(const unsigned* counter, unsigned* status, unsigned target) {
    const uint64_t t0 = globaltimer();
    while (ld_acquire_gpu(counter) < target) {
        if (*(volatile unsigned*)status != 0) return false;
        if (globaltimer() - t0 > DEADLINE_NS) {
            atomicExch(status, 1u);
            return false;
        }
    }
    return true;
}

template <int H>
__global__ void __launch_bounds__(THREADS, 1)
lstm_rec_wide_kernel(const __half* __restrict__ gx, const __half* __restrict__ whh, __half* __restrict__ y,
                     unsigned char* __restrict__ xbuf, unsigned* ctrl, int T, int N, int reverse) {
    using Q = Geo<H>;
    constexpr int G = Q::G, SLICES = Q::SLICES;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const uint32_t base = smem_u32(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, q = lane & 3;
    const int g = blockIdx.x;
    const int tiles = (N + NB - 1) / NB;
    const int total = tiles * SLICES;                  // slices of h_{t-1} per step
    const size_t par_bytes = (size_t)tiles * Q::TILE_BYTES;
    unsigned* counter = ctrl;
    unsigned* status = ctrl + STATUS_OFFSET / 4;
    volatile int* s_abort = reinterpret_cast<volatile int*>(smem_raw + Q::OFF_FLAG);
    auto bar = [&](uint32_t s) { return base + Q::OFF_BAR + s * 8; };

    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s) mbar_init(bar(s), 1);
        mbar_fence_init();
    }
    // resident W_hh slice: smem row n = [pair p][(i,f) | (g,o)][unit 4p + n%8/2][gate n%2]
    for (int i = tid; i < COLS * Q::KCH; i += THREADS) {
        const int n = i % COLS, kc = i / COLS;
        const int blk = n / 8, e = n % 8, p = blk / 2, half = blk % 2;
        const int ul = 4 * p + (e >> 1), gate = 2 * half + (e & 1);
        const int src_row = g * 32 + gate * 8 + ul;   // [unit/8 = g][gate][unit%8 = ul]
        cp_async_16(smem_raw + Q::OFF_W + (uint32_t)kc * (COLS * 16) + (uint32_t)n * 16, whh + (size_t)src_row * H + kc * 8,
                    true);
    }
    cp_async_commit();
    for (int tl = 0; tl < tiles; ++tl)
        *reinterpret_cast<float4*>(smem_raw + Q::OFF_C + (uint32_t)(tl * THREADS + tid) * 16) = make_float4(0.f, 0.f, 0.f, 0.f);
    cp_async_wait<0>();
    fence_proxy_async_smem();
    __syncthreads();

    // this thread's cells in every tile: rows r0 + 8h, CTA-local units 4p + q
    const int r0 = warp * 16 + (lane >> 2);
    const uint64_t db0 = wg_desc_noswz(base + Q::OFF_W, COLS * 16, 128);
    uint32_t seq = 0;   // slices consumed before this step (ring position / mbarrier phase)
    float acc[16];
    for (int step = 0; step < T; ++step) {
        const int t = reverse ? (T - 1 - step) : step;
        const unsigned char* hsrc = xbuf + (size_t)((step & 1) ^ 1) * par_bytes;   // h_{t-1}, written at step - 1
        unsigned char* hdst = xbuf + (size_t)(step & 1) * par_bytes;
        auto issue = [&](int i) {   // slice i of this step -> its ring stage
            const uint32_t s = (seq + (uint32_t)i) % STAGES;
            const int tl = i / SLICES, sl = i % SLICES;
            mbar_expect_tx(bar(s), SLICE_BYTES);
            bulk_g2s(base + Q::OFF_RING + s * SLICE_BYTES, hsrc + (size_t)tl * Q::TILE_BYTES + (size_t)sl * SLICE_BYTES,
                     SLICE_BYTES, bar(s));
        };
        if (step > 0) {
            if (tid == 0) {
                const bool ok = grid_wait(counter, status, (unsigned)(G * step));   // every CTA has published h_{t-1}
                if (ok) {
                    fence_proxy_async_global();
                    for (int i = 0; i < min(STAGES, total); ++i) issue(i);
                }
                *s_abort = !ok;
            }
            __syncthreads();
            if (*s_abort) return;   // nothing in flight: the copies of this step were not issued
        }
        const __half* gsrc = gx + ((size_t)t * G + g) * (size_t)N * COLS;
        for (int tl = 0; tl < tiles; ++tl) {
            uint2 gv[2][2];
#pragma unroll
            for (int p = 0; p < 2; ++p)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int chunk = tl * NB + r0 + 8 * h;
                    gv[p][h] = chunk < N ? __ldg(reinterpret_cast<const uint2*>(gsrc + (size_t)chunk * COLS + (4 * p + q) * 4))
                                         : make_uint2(0u, 0u);
                }
#pragma unroll
            for (int i = 0; i < 16; ++i) acc[i] = 0.f;
            if (step > 0) {   // h_{-1} = 0: nothing to multiply at step 0
                for (int sl = 0; sl < SLICES; ++sl) {
                    const int i = tl * SLICES + sl;
                    const uint32_t s = (seq + (uint32_t)i) % STAGES, phase = ((seq + (uint32_t)i) / STAGES) & 1u;
                    mbar_wait(bar(s), phase);
                    wg_fence_regs(acc);
                    wg_fence();
                    const uint64_t da = wg_desc_noswz(base + Q::OFF_RING + s * SLICE_BYTES, NB * 16, 128);
#pragma unroll
                    for (int kk = 0; kk < KS / 2; ++kk)   // one k16 step = two k-chunks
                        wgmma_m64n32k16_f16(acc, da + (uint64_t)(kk * 2 * NB * 16 / 16),
                                            db0 + (uint64_t)((sl * KS + 2 * kk) * COLS * 16 / 16), 1);
                    wg_commit();
                    wg_wait<1>();                         // the MMAs of slice i - 1 have drained ...
                    wg_fence_regs(acc);
                    if (i >= 1 && i - 1 + STAGES < total) {
                        __syncthreads();                  // ... in all four warps: its stage may be refilled
                        if (tid == 0) issue(i - 1 + STAGES);
                    }
                }
                wg_wait<0>();
                wg_fence_regs(acc);
            }
            float4 cs = *reinterpret_cast<const float4*>(smem_raw + Q::OFF_C + (uint32_t)(tl * THREADS + tid) * 16);
            float* c_state = reinterpret_cast<float*>(&cs);
#pragma unroll
            for (int p = 0; p < 2; ++p)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const __half2 g01 = *reinterpret_cast<const __half2*>(&gv[p][h].x);
                    const __half2 g23 = *reinterpret_cast<const __half2*>(&gv[p][h].y);
                    const float ai = acc[(2 * p) * 4 + h * 2] + __low2float(g01);
                    const float af = acc[(2 * p) * 4 + h * 2 + 1] + __high2float(g01);
                    const float ag = acc[(2 * p + 1) * 4 + h * 2] + __low2float(g23);
                    const float ao = acc[(2 * p + 1) * 4 + h * 2 + 1] + __high2float(g23);
                    float si, sf, tg, so;
                    gate_activations(ai, af, ag, ao, si, sf, tg, so);
                    const float c = fmaf(sf, c_state[2 * p + h], si * tg);
                    c_state[2 * p + h] = c;
                    *reinterpret_cast<__half*>(smem_raw + Q::OFF_STG + (uint32_t)(r0 + 8 * h) * 16 + (uint32_t)(4 * p + q) * 2) =
                        __float2half_rn(so * tanh_f(c));
                }
            *reinterpret_cast<float4*>(smem_raw + Q::OFF_C + (uint32_t)(tl * THREADS + tid) * 16) = cs;
            __syncthreads();   // the 64 x 8 block of h_t is staged
            if (tid < NB) {
                const uint4 v = *reinterpret_cast<const uint4*>(smem_raw + Q::OFF_STG + (uint32_t)tid * 16);
                if (step + 1 < T)
                    *reinterpret_cast<uint4*>(hdst + (size_t)tl * Q::TILE_BYTES + (size_t)g * (NB * 16) + (size_t)tid * 16) = v;
                const int chunk = tl * NB + tid;
                if (chunk < N) *reinterpret_cast<uint4*>(y + ((size_t)t * N + chunk) * H + g * UPC) = v;
            }
            __syncthreads();   // the staging block may be overwritten
        }
        if (step > 0) seq += (uint32_t)total;
        if (step + 1 < T && tid == 0) {   // publish h_t: the block's stores precede this CTA's arrival
            __threadfence();
            fence_proxy_async_global();
            red_release_gpu_add(counter, 1u);
        }
    }
}

template <int H>
int configure() {
    static bool configured = false;
    if (!configured) {
        B200_CHECK_CUDA(cudaFuncSetAttribute(lstm_rec_wide_kernel<H>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)Geo<H>::SMEM_BYTES));
        configured = true;
    }
    return 0;
}

template <int H>
int resident() {
    if (configure<H>() != 0) return -1;
    int dev = 0, sms = 0, per_sm = 0;
    B200_CHECK_CUDA(cudaGetDevice(&dev));
    B200_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    B200_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lstm_rec_wide_kernel<H>, THREADS,
                                                                  Geo<H>::SMEM_BYTES));
    return per_sm * sms;
}

template <int H>
int launch(const __half* gx, const __half* whh, __half* y, void* workspace, int T, int N, int reverse, cudaStream_t stream) {
    if (configure<H>() != 0) return -1;
    const int tiles = (N + NB - 1) / NB;
    unsigned char* xbuf = (unsigned char*)workspace;
    unsigned* ctrl = (unsigned*)(xbuf + 2 * (size_t)tiles * Geo<H>::TILE_BYTES);
    B200_CHECK_CUDA(cudaMemsetAsync(ctrl, 0, CTRL_BYTES, stream));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(Geo<H>::G);
    cfg.blockDim = dim3(THREADS);
    cfg.dynamicSmemBytes = Geo<H>::SMEM_BYTES;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative;
    attr[0].val.cooperative = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    B200_CHECK_CUDA(cudaLaunchKernelEx(&cfg, lstm_rec_wide_kernel<H>, gx, whh, y, xbuf, ctrl, T, N, reverse));
    return 0;
}

}  // namespace

int lstm_rec_wide_ctas(int hidden) { return (hidden == 768 || hidden == 1024) ? hidden / UPC : 0; }

size_t lstm_rec_wide_workspace_bytes(int N, int hidden) {
    if (lstm_rec_wide_ctas(hidden) == 0 || N <= 0) return 0;
    return 2 * (size_t)((N + NB - 1) / NB) * (size_t)(hidden / 8) * NB * 16 + CTRL_BYTES;
}

size_t lstm_rec_wide_status_offset(int N, int hidden) {
    const size_t ws = lstm_rec_wide_workspace_bytes(N, hidden);
    return ws == 0 ? 0 : ws - CTRL_BYTES + STATUS_OFFSET;
}

int lstm_rec_wide_max_chunks(int hidden) { return lstm_rec_wide_ctas(hidden) ? MAX_TILES * NB : 0; }

int lstm_rec_wide_resident(int hidden) {
    switch (hidden) {
        case 768: return resident<768>();
        case 1024: return resident<1024>();
        default:
            b200_set_error("lstm_rec_wide: hidden size %d is not supported (768, 1024)", hidden);
            return -2;
    }
}

// gx [T][G][N][32], y [T][N][H], workspace: lstm_rec_wide_workspace_bytes(N, hidden) bytes (exchange buffer, barrier counter,
// status word); launches on the same workspace must not overlap
int launch_lstm_rec_wide(const __half* gx, const __half* whh, __half* y, void* workspace, int T, int N, int hidden,
                         int reverse, cudaStream_t stream) {
    B200_REQUIRE(lstm_rec_wide_ctas(hidden) > 0, "lstm_rec_wide: hidden size %d is not supported (768, 1024)", hidden);
    B200_REQUIRE(N <= MAX_TILES * NB, "lstm_rec_wide: at most %d chunks per launch (got %d)", MAX_TILES * NB, N);
    B200_REQUIRE(((uintptr_t)gx % 16) == 0 && ((uintptr_t)y % 16) == 0 && ((uintptr_t)whh % 16) == 0 &&
                     ((uintptr_t)workspace % 16) == 0,
                 "lstm_rec_wide: operands must be 16-byte aligned");
    return hidden == 768 ? launch<768>(gx, whh, y, workspace, T, N, reverse, stream)
                         : launch<1024>(gx, whh, y, workspace, T, N, reverse, stream);
}
