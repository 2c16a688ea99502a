// C[M,N] = epilogue(A[M,K] * B[N,K]^T) -- legacy tensor path (mma.sync m16n8k16).
//
// Cross-check implementation: the wgmma GEMM in gemm_wgmma.cu is validated against it on the
// device (tests/test_gpu_kernels.py) and it is selectable at run time with B200_GEMM_IMPL=mma.
// Not the product path.
//
// A rows may overlap (lda < K): conv3 of the LSTM-CRF encoder is run as a GEMM over the
// channels-last, zero-padded output of the conv stem, where row t is the 19x16 window that
// starts 6*16 elements after row t-1 (reference: bonito/nn.py:235-241, Conv1d k19 s6).
#include "common.cuh"

namespace {

constexpr int BM = 128, BN = 128, BK = 32, STAGES = 3, PADK = BK + 8;
constexpr int THREADS = 256;

struct Smem {
    __half a[STAGES][BM][PADK];
    __half b[STAGES][BN][PADK];
};

__global__ void __launch_bounds__(THREADS, 1)
gemm_mma_kernel(const __half* __restrict__ A, long long lda, const __half* __restrict__ B, __half* __restrict__ C,
                long long ldc, int M, int N, int K, GemmEpilogue ep) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    Smem& s = *reinterpret_cast<Smem*>(smem_raw);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp >> 2, wn = warp & 3;  // 2 x 4 warps, warp tile 64 x 32
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
    const int ktiles = (K + BK - 1) / BK;

    auto load_stage = [&](int stage, int kt) {
        const int k0 = kt * BK;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            int chunk = tid + i * THREADS;  // 512 chunks of 16 B per operand tile
            int row = chunk >> 2, col = (chunk & 3) * 8;
            bool kin = (k0 + col) < K;
            int gm = m0 + row;
            bool va = kin && gm < M;
            cp_async_16(&s.a[stage][row][col], A + (va ? (long long)gm * lda + k0 + col : 0), va);
            int gn = n0 + row;
            bool vb = kin && gn < N;
            cp_async_16(&s.b[stage][row][col], B + (vb ? (long long)gn * K + k0 + col : 0), vb);
        }
    };

    float acc[4][4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int r = 0; r < 4; ++r) acc[i][j][r] = 0.f;

#pragma unroll
    for (int st = 0; st < STAGES - 1; ++st) {
        if (st < ktiles) load_stage(st, st);
        cp_async_commit();
    }

    for (int kt = 0; kt < ktiles; ++kt) {
        cp_async_wait<STAGES - 2>();
        __syncthreads();
        {
            int nk = kt + STAGES - 1;
            if (nk < ktiles) load_stage(nk % STAGES, nk);
            cp_async_commit();
        }
        const int st = kt % STAGES;
#pragma unroll
        for (int kk = 0; kk < BK; kk += 16) {
            uint32_t af[4][4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                int row = wm * 64 + i * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
                int col = kk + (lane >> 4) * 8;
                ldmatrix_x4(af[i][0], af[i][1], af[i][2], af[i][3], smem_u32(&s.a[st][row][col]));
            }
            uint32_t bf[4][2];
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                int row = wn * 32 + j * 16 + (lane & 7) + (lane >> 4) * 8;
                int col = kk + ((lane >> 3) & 1) * 8;
                ldmatrix_x4(bf[2 * j][0], bf[2 * j][1], bf[2 * j + 1][0], bf[2 * j + 1][1],
                            smem_u32(&s.b[st][row][col]));
            }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) mma_16816(acc[i][j], af[i], bf[j][0], bf[j][1]);
        }
    }
    cp_async_wait<0>();

    // epilogue: bias -> fp16 round -> activation -> fp16, rows remapped
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            int gm = m0 + wm * 64 + i * 16 + (lane >> 2) + h * 8;
            if (gm >= M) continue;
            long long orow = map_row(ep.map, gm);
            if (orow < 0) continue;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                int gn = n0 + wn * 32 + j * 8 + (lane & 3) * 2;
                if (gn >= N) continue;
                float v0 = acc[i][j][h * 2 + 0], v1 = acc[i][j][h * 2 + 1];
                if (ep.bias) {
                    v0 += __half2float(ep.bias[gn]);
                    if (gn + 1 < N) v1 += __half2float(ep.bias[gn + 1]);
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
                __half* dst = C + drow * ldc + dcol;
                if (gn + 1 < N) {
                    *reinterpret_cast<__half2*>(dst) = __floats2half2_rn(v0, v1);
                } else {
                    *dst = __float2half_rn(v0);
                }
            }
        }
    }
}

}  // namespace

int launch_gemm_mma(const __half* A, long long lda, const __half* B, __half* C, long long ldc, int M, int N, int K,
                    const GemmEpilogue& ep, cudaStream_t stream) {
    B200_REQUIRE(K % 8 == 0 && lda % 8 == 0, "gemm_mma: K (%d) and lda (%lld) must be multiples of 8", K, lda);
    B200_REQUIRE(N % 2 == 0 && ldc % 2 == 0, "gemm_mma: N (%d) and ldc (%lld) must be even", N, ldc);
    static bool configured = false;
    if (!configured) {
        B200_CHECK_CUDA(cudaFuncSetAttribute(gemm_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)sizeof(Smem)));
        configured = true;
    }
    dim3 grid((N + BN - 1) / BN, (M + BM - 1) / BM);
    gemm_mma_kernel<<<grid, THREADS, sizeof(Smem), stream>>>(A, lda, B, C, ldc, M, N, K, ep);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}
