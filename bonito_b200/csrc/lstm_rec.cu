// Persistent recurrent part of one LSTM layer (reference semantics: bonito/nn.py:353-415,
// torch.nn.LSTM single layer, gate order i,f,g,o, optional time reversal instead of flip()).
//
//   gates_t = Gx_t (= x_t W_ih^T + b, precomputed by the GEMM) + h_{t-1} W_hh^T
//   c_t = sigmoid(f) c_{t-1} + sigmoid(i) tanh(g) ;  h_t = sigmoid(o) tanh(c_t)
//
// Decomposition (weight-stationary, hidden-split): a thread-block cluster of CS CTAs owns one
// batch tile of NB=32 chunks for the whole sequence.  CTA `rank` keeps the W_hh rows of its
// UPC = H/CS hidden units (4*UPC x H fp16) resident in shared memory for all T steps; per step
// it computes the 4*UPC x NB gate tile on the tensor pipe, updates its slice of (c, h) in
// registers, writes the h slice into the layer output Y[t] (which doubles as the exchange
// buffer), and after a cluster barrier every CTA re-reads the full NB x H h_t tile from L2.
//
// Packed operand layouts (built by bonito_b200/engine.py):
//   whh : [CS][UPC/8][gate(4)][8 units][H]     -- rows of a 32-row block = (gate, unit%8), so
//          one thread's mma accumulators hold i,f,g,o of the same (unit, chunk)
//   gx  : [T][N][CS][UPC/8][8 units][gate(4)]  -- a thread reads its 4 gate pre-activations as 8 B
//   y   : [T][N][H]
#include "common.cuh"

namespace {

constexpr int NB = 32;  // chunks per cluster

template <int H, int CS>
struct RecCfg {
    static constexpr int UPC = H / CS;        // hidden units per CTA
    static constexpr int RB = UPC / 8;        // 32-row blocks (8 units x 4 gates)
    static constexpr int WARPS = RB * 2;      // (row block, 16-chunk half)
    static constexpr int THREADS = WARPS * 32;
    static constexpr int LDW = H + 8;         // padded smem row (halves)
    static constexpr int LDS = UPC + 8;       // padded stage row
    static constexpr size_t SMEM = (size_t)(4 * UPC + NB) * LDW * 2 + (size_t)NB * LDS * 2;
    static_assert(H % 16 == 0 && UPC % 8 == 0 && THREADS <= 1024, "unsupported LSTM shape");
};

__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;\n" ::: "memory");
}

template <int H, int CS>
__global__ void __launch_bounds__(RecCfg<H, CS>::THREADS, 1)
lstm_rec_kernel(const __half* __restrict__ gx, const __half* __restrict__ whh, __half* __restrict__ y, int T, int N,
                int reverse) {
    using Cfg = RecCfg<H, CS>;
    constexpr int UPC = Cfg::UPC, LDW = Cfg::LDW, LDS = Cfg::LDS, THREADS = Cfg::THREADS;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __half* Ws = reinterpret_cast<__half*>(smem_raw);   // [4*UPC][LDW]
    __half* hs = Ws + (size_t)4 * UPC * LDW;             // [NB][LDW]   h_{t-1} tile
    __half* stage = hs + (size_t)NB * LDW;               // [NB][LDS]   this CTA's h_t slice

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int rank = blockIdx.x % CS;      // == %cluster_ctarank for 1-D clusters
    const int group = blockIdx.x / CS;
    const int n0 = group * NB;
    const int rb = warp >> 1, nh = warp & 1;
    const int r = lane >> 2, q = lane & 3;

    // resident weights
    {
        const __half* wsrc = whh + (size_t)rank * 4 * UPC * H;
        constexpr int CH = H / 8;  // 16-B chunks per row
        for (int i = tid; i < 4 * UPC * CH; i += THREADS) {
            int row = i / CH, c = i % CH;
            cp_async_16(Ws + (size_t)row * LDW + c * 8, wsrc + (size_t)row * H + c * 8, true);
        }
        cp_async_commit();
        for (int i = tid; i < NB * LDW / 8; i += THREADS) reinterpret_cast<uint4*>(hs)[i] = make_uint4(0, 0, 0, 0);
    }

    float c_state[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
    const int unit_local = rb * 8 + r;
    // this thread's gate quadruple inside a gx row
    const size_t gx_col = (size_t)rank * 4 * UPC + (size_t)rb * 32 + r * 4;

    for (int step = 0; step < T; ++step) {
        const int t = reverse ? (T - 1 - step) : step;

        // prefetch this step's input pre-activations (independent of the recurrence)
        uint2 gxr[2][2];
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                int n = n0 + nh * 16 + j * 8 + 2 * q + e;
                gxr[j][e] = (n < N) ? __ldg(reinterpret_cast<const uint2*>(gx + ((size_t)t * N + n) * 4 * H + gx_col))
                                    : make_uint2(0, 0);
            }

        cp_async_wait<0>();
        __syncthreads();  // hs (and, first step, Ws) landed

        float acc[2][2][4];
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
            for (int j = 0; j < 2; ++j)
#pragma unroll
                for (int x = 0; x < 4; ++x) acc[m][j][x] = 0.f;

        if (step > 0) {
#pragma unroll 4
            for (int kk = 0; kk < H; kk += 16) {
                uint32_t a[2][4], b[2][2];
#pragma unroll
                for (int m = 0; m < 2; ++m) {
                    int row = rb * 32 + m * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
                    ldmatrix_x4(a[m][0], a[m][1], a[m][2], a[m][3], smem_u32(Ws + (size_t)row * LDW + kk + (lane >> 4) * 8));
                }
                {
                    int row = nh * 16 + (lane & 7) + (lane >> 4) * 8;
                    ldmatrix_x4(b[0][0], b[0][1], b[1][0], b[1][1],
                                smem_u32(hs + (size_t)row * LDW + kk + ((lane >> 3) & 1) * 8));
                }
#pragma unroll
                for (int m = 0; m < 2; ++m)
#pragma unroll
                    for (int j = 0; j < 2; ++j) mma_16816(acc[m][j], a[m], b[j][0], b[j][1]);
            }
        }

        // cell update for (unit, 4 chunks) held by this thread
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const __half2 g01 = *reinterpret_cast<const __half2*>(&gxr[j][e].x);
                const __half2 g23 = *reinterpret_cast<const __half2*>(&gxr[j][e].y);
                float ai = acc[0][j][e] + __low2float(g01);
                float af = acc[0][j][2 + e] + __high2float(g01);
                float ag = acc[1][j][e] + __low2float(g23);
                float ao = acc[1][j][2 + e] + __high2float(g23);
                float c, h;
                if constexpr (H == 384) {   // the cell math of the tile kernel: the two width-384 kernels agree bitwise
                    float si, sf, tg, so;
                    gate_activations(ai, af, ag, ao, si, sf, tg, so);
                    c = fmaf(sf, c_state[j][e], si * tg);
                    h = so * tanh_f(c);
                } else {
                    c = sigmoid_f(af) * c_state[j][e] + sigmoid_f(ai) * tanh_f(ag);
                    h = sigmoid_f(ao) * tanh_f(c);
                }
                c_state[j][e] = c;
                int b = nh * 16 + j * 8 + 2 * q + e;
                stage[b * LDS + unit_local] = __float2half_rn(h);
            }
        __syncthreads();  // stage complete; every warp is done reading hs

        // publish the h_t slice: Y[t][n0+b][rank*UPC .. +UPC)
        {
            constexpr int CH = UPC / 8;
            for (int i = tid; i < NB * CH; i += THREADS) {
                int b = i / CH, c = i % CH;
                int n = n0 + b;
                if (n < N)
                    *reinterpret_cast<uint4*>(y + ((size_t)t * N + n) * H + rank * UPC + c * 8) =
                        *reinterpret_cast<const uint4*>(stage + b * LDS + c * 8);
            }
        }
        if (step + 1 == T) break;
        __threadfence();
        if (CS > 1) cluster_sync_all(); else __syncthreads();

        // gather the full h_t tile for the next step (L2 -> smem, bypassing L1)
        {
            constexpr int CH = H / 8;
            for (int i = tid; i < NB * CH; i += THREADS) {
                int b = i / CH, c = i % CH;
                int n = n0 + b;
                bool valid = n < N;
                cp_async_16(hs + (size_t)b * LDW + c * 8, y + ((size_t)t * N + (valid ? n : 0)) * H + c * 8, valid);
            }
            cp_async_commit();
        }
    }
}

template <int H, int CS>
int launch_rec(const __half* gx, const __half* whh, __half* y, int T, int N, int reverse, cudaStream_t stream) {
    using Cfg = RecCfg<H, CS>;
    auto kern = lstm_rec_kernel<H, CS>;
    B200_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::SMEM));
    const int groups = (N + NB - 1) / NB;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(groups * CS);
    cfg.blockDim = dim3(Cfg::THREADS);
    cfg.dynamicSmemBytes = Cfg::SMEM;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = CS;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    B200_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kern, gx, whh, y, T, N, reverse));
    return 0;
}

}  // namespace

// Cluster size the packed layouts must be built for (0 = unsupported hidden size).
int lstm_rec_cluster_size(int H) {
    if (H == 384) return 8;
    if (H == 96 || H == 128) return 1;
    if (H == 256) return 4;
    return 0;
}

int launch_lstm_rec(const __half* gx, const __half* whh, __half* y, int T, int N, int H, int reverse,
                    cudaStream_t stream) {
    switch (H) {
        case 384: return launch_rec<384, 8>(gx, whh, y, T, N, reverse, stream);
        case 256: return launch_rec<256, 4>(gx, whh, y, T, N, reverse, stream);
        case 128: return launch_rec<128, 1>(gx, whh, y, T, N, reverse, stream);
        case 96: return launch_rec<96, 1>(gx, whh, y, T, N, reverse, stream);
        default:
            b200_set_error("lstm_rec: hidden size %d is not supported (96, 128, 256, 384)", H);
            return -2;
    }
}
