// CTC-CRF scoring and loss: the sequence distribution CTC_CRF of bonito/crf/model.py:30-143 (logZ, forward / backward
// scores, posteriors, Viterbi, and the target-constrained lattice behind ctc_loss / ctc_viterbi_alignments).
//
// Two lattices, each in the Log (logsumexp) and the Max semiring, all in fp32 in the natural-log domain with the accurate
// expf / logf / log1pf (gradients are compared against float64, so none of the ex2.approx shortcuts of crf_decode.cu):
//
//  * the sparse k-mer lattice: S = 4^k states, in-edge e of state s comes from idx[s, e] (e = 0: s itself, e = 1 + j:
//    j*S/4 + s/4); scores [T][N][S*5] fp32 with the edge (s, e) at column s*5 + e; alpha_0 = beta_T = 0 for every state.
//    Forward: alpha_{t+1}[s] = (+)_e M[t,s,e] + alpha_t[idx[s,e]]; logZ = (+)_s alpha_T[s].
//    Log gradient: dlogZ/dM[t,s,e] = g * exp(alpha_t[idx[s,e]] + M[t,s,e] + beta_{t+1}[s] - logZ).
//    Max gradient: g on the edges of the best path, ties to the lowest in-edge at every frame, then the lowest final state.
//  * the target lattice: stay [T][N][L], move [T][N][L-1], lengths [N]; alpha_0 = [0, -inf, ...],
//    alpha_{t+1}[j] = (+)(alpha_t[j] + stay[t,j], alpha_t[j-1] + move[t,j-1]), logZ = alpha_T[lengths-1].  Max ties go to the
//    stay.  A chunk with lengths < 1, lengths > L or lengths - 1 > T (more moves than frames) is infeasible: logZ = -inf and
//    a gradient of exactly 0 whatever g holds.
//
// One CTA per chunk, one thread per state (the target lattice: J states per thread, strided by the block size), a
// double-buffered alpha / beta row in shared memory and one barrier per frame.  Score rows (and, for the gradient, the
// forward's alpha rows) stream through a PF-deep cp.async ring.  Every row is re-centred on one of its entries (k-mer: state
// 0; target: the previous row's maximum, since most of its states are -inf early on) and the shifts are summed in fp64, so
// the fp32 error does not grow with |logZ|.  The training path keeps the re-centred alpha rows, their fp64 offsets and the
// fp64 logZ in a caller-allocated workspace; the gradient kernel is then one backward pass that produces beta and writes the
// gradient.  Every index into a [T][N][...] tensor is 64-bit.  No atomics: every output is bitwise deterministic.
#include <limits.h>

#include "common.cuh"

namespace {

constexpr int PF = 4;  // score rows in flight

inline size_t align256(size_t x) { return (x + 255) / 256 * 256; }

__device__ __forceinline__ float lse2(float a, float b) {
    const float m = fmaxf(a, b);
    if (m == -INFINITY) return m;
    return m + log1pf(expf(fminf(a, b) - m));
}

template <bool MAX>
__device__ __forceinline__ float sum5(const float (&x)[5]) {
    const float m = fmaxf(fmaxf(fmaxf(x[0], x[1]), fmaxf(x[2], x[3])), x[4]);
    if (MAX || m == -INFINITY) return m;
    float s = 0.f;
#pragma unroll
    for (int e = 0; e < 5; ++e) s += expf(x[e] - m);
    return m + logf(s);
}

__device__ __forceinline__ void cp_async_4(void* smem_dst, const void* gmem_src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(smem_u32(smem_dst)), "l"(gmem_src));
}

// `bytes` (a multiple of 16) from global to shared memory, 16 bytes per copy, spread over the whole CTA
__device__ __forceinline__ void copy_row(void* dst, const void* src, int bytes) {
    for (int i = threadIdx.x * 16; i < bytes; i += blockDim.x * 16)
        cp_async_16(static_cast<char*>(dst) + i, static_cast<const char*>(src) + i, true);
}

// Block-wide max with the lowest index among equal maxima (every thread gets the result).  `red` holds 2 * 32 words.
__device__ __forceinline__ void block_argmax(float& v, int& i, float* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int oi = __shfl_xor_sync(0xffffffffu, i, o);
        if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }
    }
    __syncthreads();
    if (lane == 0) { red[warp] = v; reinterpret_cast<int*>(red)[32 + warp] = i; }
    __syncthreads();
    v = red[0];
    i = reinterpret_cast<int*>(red)[32];
    for (int w = 1; w < nw; ++w) {
        const float ov = red[w];
        const int oi = reinterpret_cast<int*>(red)[32 + w];
        if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }
    }
}

// Block-wide sum in a fixed order (bitwise reproducible).
__device__ __forceinline__ float block_sum(float v, float* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float s = 0.f;
    for (int w = 0; w < nw; ++w) s += red[w];
    return s;
}

// =====================================================================================================================
// sparse k-mer lattice
// =====================================================================================================================
template <int S>
struct SparseSmem {
    static constexpr int NT = S < 32 ? 32 : S;                          // threads (states >= S idle)
    static constexpr size_t kBuf = 0;                                   // float [2][S]
    static constexpr size_t kRed = kBuf + 2 * S * sizeof(float);        // 64 words
    static constexpr size_t kRing = kRed + 64 * sizeof(float);          // float [PF][5S]: score rows
    static constexpr size_t kARing = kRing + PF * 5 * S * sizeof(float);  // float [PF][S]: alpha' rows (gradient)
    static constexpr size_t bytes(bool grad) { return kARing + (grad ? PF * S * sizeof(float) : 0); }
};

// Workspace of the sparse lattice, for N chunks of T frames.
//   Log: alpha' float [N][T+1][S], offsets double [N][T+1], logZ double [N]
//   Max: back-pointers u8 [N][T][S], best final state int [N], path int [N][T]
struct SparseWs {
    float* alpha = nullptr;
    double* off = nullptr;
    double* logz = nullptr;
    uint8_t* bp = nullptr;
    int* final_state = nullptr;
    int* path = nullptr;
    size_t bytes = 0;
    SparseWs(void* base, int N, int T, int S, bool max_semiring) {
        unsigned char* ws = static_cast<unsigned char*>(base);
        auto take = [&](size_t b) { unsigned char* p = ws ? ws + bytes : nullptr; bytes += align256(b); return p; };
        if (max_semiring) {
            bp = take((size_t)N * T * S);
            final_state = reinterpret_cast<int*>(take((size_t)N * sizeof(int)));
            path = reinterpret_cast<int*>(take((size_t)N * T * sizeof(int)));
        } else {
            alpha = reinterpret_cast<float*>(take((size_t)N * (T + 1) * S * sizeof(float)));
            off = reinterpret_cast<double*>(take((size_t)N * (T + 1) * sizeof(double)));
            logz = reinterpret_cast<double*>(take((size_t)N * sizeof(double)));
        }
    }
};

// Forward pass.  Optional outputs: alpha_out [T+1][N][S] (true alpha), the workspace (Log: alpha' rows + offsets + fp64
// logZ; Max: back-pointers + best final state).  Without either only the two alpha rows in shared memory are kept.
template <int S, bool MAX>
__global__ void __launch_bounds__(SparseSmem<S>::NT)
sparse_fwd_kernel(const float* __restrict__ scores, int T, int N, float* __restrict__ logz, float* __restrict__ alpha_out,
                  float* __restrict__ ws_alpha, double* __restrict__ ws_off, double* __restrict__ ws_logz,
                  uint8_t* __restrict__ ws_bp, int* __restrict__ ws_final) {
    using L = SparseSmem<S>;
    constexpr int Q = S / 4;
    extern __shared__ __align__(16) unsigned char sm[];
    float (*buf)[S] = reinterpret_cast<float (*)[S]>(sm + L::kBuf);
    float* red = reinterpret_cast<float*>(sm + L::kRed);
    float (*ring)[5 * S] = reinterpret_cast<float (*)[5 * S]>(sm + L::kRing);

    const int n = blockIdx.x, s = threadIdx.x;
    const bool act = s < S;
    const size_t frame = (size_t)N * 5 * S;                 // floats from one frame to the next
    const float* sc = scores + (size_t)n * 5 * S;
    if (act) {
        buf[0][s] = 0.f;
        if (alpha_out) alpha_out[(size_t)n * S + s] = 0.f;
        if (ws_alpha) ws_alpha[(size_t)n * (T + 1) * S + s] = 0.f;
    }
    if (ws_off && s == 0) ws_off[(size_t)n * (T + 1)] = 0.0;
    for (int r = 0; r < PF - 1; ++r) {
        if (r < T) copy_row(ring[r], sc + (size_t)r * frame, 5 * S * sizeof(float));
        cp_async_commit();
    }
    double off = 0.0;                                       // alpha_t = alpha'_t + off
    for (int t = 0; t < T; ++t) {
        cp_async_wait<PF - 2>();                            // this thread's pieces of row t
        __syncthreads();                                    // everyone's pieces; step t-1 done with its ring slot and row
        {
            const int r = t + PF - 1;
            if (r < T) copy_row(ring[r % PF], sc + (size_t)r * frame, 5 * S * sizeof(float));
            cp_async_commit();
        }
        const float* cur = buf[t & 1];
        const float b0 = cur[0];
        const float shift = (b0 > -INFINITY && b0 < INFINITY) ? b0 : 0.f;
        if (act) {
            const float* m = ring[t % PF] + 5 * s;
            float x[5];
            x[0] = m[0] + cur[s];
#pragma unroll
            for (int j = 0; j < 4; ++j) x[1 + j] = m[1 + j] + cur[j * Q + s / 4];
            float v;
            if constexpr (MAX) {
                int best = 0;
                v = x[0];
#pragma unroll
                for (int e = 1; e < 5; ++e)
                    if (x[e] > v) { v = x[e]; best = e; }
                if (ws_bp) ws_bp[((size_t)n * T + t) * S + s] = (uint8_t)best;
            } else {
                v = sum5<false>(x);
            }
            v -= shift;
            buf[(t & 1) ^ 1][s] = v;
            if (ws_alpha) ws_alpha[((size_t)n * (T + 1) + t + 1) * S + s] = v;
            if (alpha_out) alpha_out[((size_t)(t + 1) * N + n) * S + s] = (float)((double)v + (off + (double)shift));
        }
        off += (double)shift;
        if (ws_off && s == 0) ws_off[(size_t)n * (T + 1) + t + 1] = off;
    }
    cp_async_wait<0>();
    __syncthreads();
    const float* fin = buf[T & 1];
    float v = act ? fin[s] : -INFINITY;
    int arg = act ? s : INT_MAX;
    block_argmax(v, arg, red);
    if constexpr (MAX) {
        if (s == 0) {
            logz[n] = (float)(off + (double)v);
            if (ws_final) ws_final[n] = arg;
        }
    } else {
        const float m = v;
        float e = (act && m > -INFINITY) ? expf(fin[s] - m) : 0.f;
        const float sum = block_sum(e, red);
        if (s == 0) {
            const double lz = m > -INFINITY ? off + (double)m + (double)logf(sum) : -(double)INFINITY;
            logz[n] = (float)lz;
            if (ws_logz) ws_logz[n] = lz;
        }
    }
}

// Backward pass: beta_t[p] = (+) over the out-edges of p: the stay (p, 0) and the moves into 4(p%Q)+c, in-edge 1 + p/Q.
// beta_out [T+1][N][S] when given.  GRAD (Log only): also the gradient g[n] * exp(alpha_t[idx] + M + beta_{t+1} - logZ)
// from the forward's workspace, written as grad [T][N][S*5].
template <int S, bool MAX, bool GRAD>
__global__ void __launch_bounds__(SparseSmem<S>::NT)
sparse_bwd_kernel(const float* __restrict__ scores, int T, int N, float* __restrict__ beta_out,
                  const float* __restrict__ g, const float* __restrict__ ws_alpha, const double* __restrict__ ws_off,
                  const double* __restrict__ ws_logz, float* __restrict__ grad) {
    using L = SparseSmem<S>;
    constexpr int Q = S / 4;
    extern __shared__ __align__(16) unsigned char sm[];
    float (*buf)[S] = reinterpret_cast<float (*)[S]>(sm + L::kBuf);
    float (*ring)[5 * S] = reinterpret_cast<float (*)[5 * S]>(sm + L::kRing);
    float (*aring)[S] = reinterpret_cast<float (*)[S]>(sm + L::kARing);

    const int n = blockIdx.x, p = threadIdx.x;
    const bool act = p < S;
    const size_t frame = (size_t)N * 5 * S;
    const float* sc = scores + (size_t)n * 5 * S;
    const float* alpha_n = GRAD ? ws_alpha + (size_t)n * (T + 1) * S : nullptr;
    const double* off_n = GRAD ? ws_off + (size_t)n * (T + 1) : nullptr;
    float gn = 0.f;
    double lz = 0.0;
    if constexpr (GRAD) {
        gn = g[n];
        lz = ws_logz[n];
    }
    if (act) {
        buf[0][p] = 0.f;
        if (beta_out) beta_out[((size_t)T * N + n) * S + p] = 0.f;
    }
    auto fetch = [&](int i) {                               // iteration i handles frame T-1-i
        const int r = T - 1 - i;
        if (r >= 0) {
            copy_row(ring[i % PF], sc + (size_t)r * frame, 5 * S * sizeof(float));
            if constexpr (GRAD) copy_row(aring[i % PF], alpha_n + (size_t)r * S, S * sizeof(float));
        }
        cp_async_commit();
    };
    for (int i = 0; i < PF - 1; ++i) fetch(i);
    double off = 0.0;                                       // beta_{t+1} = beta'_{t+1} + off
    for (int i = 0; i < T; ++i) {
        const int t = T - 1 - i;
        cp_async_wait<PF - 2>();
        __syncthreads();
        fetch(i + PF - 1);
        const float* cur = buf[i & 1];
        const float* m = ring[i % PF];
        const float b0 = cur[0];
        const float shift = (b0 > -INFINITY && b0 < INFINITY) ? b0 : 0.f;
        if (act) {
            if constexpr (GRAD) {
                const float* a = aring[i % PF];
                const float k = (float)(off_n[t] + off - lz);
                const float bs = cur[p] + k;
                float* gr = grad + ((size_t)t * N + n) * 5 * S + 5 * p;
                gr[0] = gn * expf(a[p] + m[5 * p] + bs);
#pragma unroll
                for (int j = 0; j < 4; ++j) gr[1 + j] = gn * expf(a[j * Q + p / 4] + m[5 * p + 1 + j] + bs);
            }
            const int e = 1 + p / Q, base = 4 * (p % Q);
            float x[5];
            x[0] = m[5 * p] + cur[p];
#pragma unroll
            for (int c = 0; c < 4; ++c) x[1 + c] = m[5 * (base + c) + e] + cur[base + c];
            const float v = sum5<MAX>(x) - shift;
            buf[(i & 1) ^ 1][p] = v;
            if (beta_out) beta_out[((size_t)t * N + n) * S + p] = (float)((double)v + (off + (double)shift));
        }
        off += (double)shift;
    }
    cp_async_wait<0>();
}

// Max-semiring gradient: trace the best path back through the forward's back-pointers (thread 0), then write the
// one-hot rows grad [T][N][S*5] (g[n] on the path's edge, 0 elsewhere) with the whole CTA.
template <int S>
__global__ void __launch_bounds__(256)
sparse_max_grad_kernel(int T, int N, const float* __restrict__ g, const uint8_t* __restrict__ ws_bp,
                       const int* __restrict__ ws_final, int* __restrict__ ws_path, float* __restrict__ grad) {
    constexpr int Q = S / 4;
    const int n = blockIdx.x;
    int* path = ws_path + (size_t)n * T;
    if (threadIdx.x == 0) {
        int s = ws_final[n];
        for (int t = T - 1; t >= 0; --t) {
            const int e = ws_bp[((size_t)n * T + t) * S + s];
            path[t] = s * 5 + e;
            s = e == 0 ? s : (e - 1) * Q + s / 4;
        }
    }
    __syncthreads();
    const float gn = g[n];
    for (int t = 0; t < T; ++t) {
        const int hot = path[t];
        float* row = grad + ((size_t)t * N + n) * 5 * S;
        for (int c = threadIdx.x; c < 5 * S; c += blockDim.x) row[c] = c == hot ? gn : 0.f;
    }
}

template <int S>
int sparse_fwd(const float* scores, int T, int N, int semiring, float* logz, float* alpha, void* workspace,
               cudaStream_t stream) {
    const bool mx = semiring == B200_SEMIRING_MAX;
    SparseWs ws(workspace, N, T, S, mx);
    const size_t smem = SparseSmem<S>::bytes(false);
    if (mx) {
        auto k = sparse_fwd_kernel<S, true>;
        B200_CHECK_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k<<<N, SparseSmem<S>::NT, smem, stream>>>(scores, T, N, logz, alpha, nullptr, nullptr, nullptr, ws.bp,
                                                  ws.final_state);
    } else {
        auto k = sparse_fwd_kernel<S, false>;
        B200_CHECK_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k<<<N, SparseSmem<S>::NT, smem, stream>>>(scores, T, N, logz, alpha, ws.alpha, ws.off, ws.logz, nullptr, nullptr);
    }
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

template <int S>
int sparse_bwd(const float* scores, int T, int N, int semiring, float* beta, cudaStream_t stream) {
    const size_t smem = SparseSmem<S>::bytes(false);
    auto k = semiring == B200_SEMIRING_MAX ? sparse_bwd_kernel<S, true, false> : sparse_bwd_kernel<S, false, false>;
    B200_CHECK_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k<<<N, SparseSmem<S>::NT, smem, stream>>>(scores, T, N, beta, nullptr, nullptr, nullptr, nullptr, nullptr);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

template <int S>
int sparse_grad(const float* scores, int T, int N, int semiring, const float* g, void* workspace, float* grad,
                cudaStream_t stream) {
    const bool mx = semiring == B200_SEMIRING_MAX;
    SparseWs ws(workspace, N, T, S, mx);
    if (mx) {
        sparse_max_grad_kernel<S><<<N, 256, 0, stream>>>(T, N, g, ws.bp, ws.final_state, ws.path, grad);
    } else {
        const size_t smem = SparseSmem<S>::bytes(true);
        auto k = sparse_bwd_kernel<S, false, true>;
        B200_CHECK_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k<<<N, SparseSmem<S>::NT, smem, stream>>>(scores, T, N, nullptr, g, ws.alpha, ws.off, ws.logz, grad);
    }
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// =====================================================================================================================
// target-constrained lattice
// =====================================================================================================================
constexpr int TGT_MAX_THREADS = 1024;
constexpr int TGT_MAX_J = 4;  // states per thread: L <= 4096

// Workspace of the target lattice, for N chunks of T frames and L states.
//   Log: alpha' float [N][T+1][L], offsets double [N][T+1], logZ double [N]
//   Max: back-pointers u8 [N][T][L] (1 = arrived by the move), path int [N][T]
struct TargetWs {
    float* alpha = nullptr;
    double* off = nullptr;
    double* logz = nullptr;
    uint8_t* bp = nullptr;
    int* path = nullptr;
    size_t bytes = 0;
    TargetWs(void* base, int N, int T, int L, bool max_semiring) {
        unsigned char* ws = static_cast<unsigned char*>(base);
        auto take = [&](size_t b) { unsigned char* p = ws ? ws + bytes : nullptr; bytes += align256(b); return p; };
        if (max_semiring) {
            bp = take((size_t)N * T * L);
            path = reinterpret_cast<int*>(take((size_t)N * T * sizeof(int)));
        } else {
            alpha = reinterpret_cast<float*>(take((size_t)N * (T + 1) * L * sizeof(float)));
            off = reinterpret_cast<double*>(take((size_t)N * (T + 1) * sizeof(double)));
            logz = reinterpret_cast<double*>(take((size_t)N * sizeof(double)));
        }
    }
};

struct TargetSmem {
    // buf float [2][Lp], per-warp row maxima float [2][32], stay / move / alpha' rings float [PF][Lp] each
    static size_t bytes(int Lp, bool grad) { return (2 * Lp + 64 + (grad ? 3 : 2) * PF * Lp) * sizeof(float); }
};

__device__ __forceinline__ bool target_feasible(int len, int T, int L) { return len >= 1 && len <= L && len - 1 <= T; }

// Re-centring shift of a row from the per-warp maxima its step left in `wmax` (0 when the row holds no finite value).
__device__ __forceinline__ float row_shift(const float* wmax, int nw) {
    float m = -INFINITY;
    for (int w = 0; w < nw; ++w) m = fmaxf(m, wmax[w]);
    return m > -INFINITY ? m : 0.f;
}

__device__ __forceinline__ void warp_max_store(float v, float* wmax) {
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = v;
}

template <int J, bool MAX>
__global__ void __launch_bounds__(TGT_MAX_THREADS)
target_fwd_kernel(const float* __restrict__ stay, const float* __restrict__ move, const int* __restrict__ lengths, int T,
                  int N, int L, float* __restrict__ logz, float* __restrict__ ws_alpha, double* __restrict__ ws_off,
                  double* __restrict__ ws_logz, uint8_t* __restrict__ ws_bp) {
    const int n = blockIdx.x, tid = threadIdx.x, B = blockDim.x, nw = B >> 5, Lp = B * J;
    const int len = lengths[n];
    if (!target_feasible(len, T, L)) {
        if (tid == 0) {
            logz[n] = -INFINITY;
            if (ws_logz) ws_logz[n] = -(double)INFINITY;
        }
        return;
    }
    extern __shared__ __align__(16) float smf[];
    float* buf = smf;                      // [2][Lp]
    float* wmax = buf + 2 * Lp;            // [2][32]
    float* rs = wmax + 64;                 // [PF][Lp]
    float* rm = rs + PF * Lp;              // [PF][Lp]
    const float* st_n = stay + (size_t)n * L;
    const float* mv_n = move + (size_t)n * (L - 1);
    const size_t fs = (size_t)N * L, fm = (size_t)N * (L - 1);
    // each thread copies, and later reads, only its own states: its wait_group alone makes them visible to it
    auto fetch = [&](int r) {
        if (r < T) {
#pragma unroll
            for (int u = 0; u < J; ++u) {
                const int j = tid + u * B;
                if (j < L) cp_async_4(&rs[(r % PF) * Lp + j], st_n + (size_t)r * fs + j);
                if (j >= 1 && j < L) cp_async_4(&rm[(r % PF) * Lp + j], mv_n + (size_t)r * fm + j - 1);
            }
        }
        cp_async_commit();
    };
#pragma unroll
    for (int u = 0; u < J; ++u) {
        const int j = tid + u * B;
        buf[j] = j == 0 ? 0.f : -INFINITY;
        if (ws_alpha && j < L) ws_alpha[(size_t)n * (T + 1) * L + j] = buf[j];
    }
    if (tid < 32) wmax[tid] = 0.f;
    if (ws_off && tid == 0) ws_off[(size_t)n * (T + 1)] = 0.0;
    for (int r = 0; r < PF - 1; ++r) fetch(r);
    double off = 0.0;
    for (int t = 0; t < T; ++t) {
        cp_async_wait<PF - 2>();
        __syncthreads();
        fetch(t + PF - 1);
        const float* cur = buf + (t & 1) * Lp;
        float* nxt = buf + ((t & 1) ^ 1) * Lp;
        const float shift = row_shift(wmax + (t & 1) * 32, nw);
        float vmax = -INFINITY;
#pragma unroll
        for (int u = 0; u < J; ++u) {
            const int j = tid + u * B;
            float v = -INFINITY;
            if (j < L) {
                const float a = cur[j] + rs[(t % PF) * Lp + j];
                const float b = j >= 1 ? cur[j - 1] + rm[(t % PF) * Lp + j] : -INFINITY;
                if constexpr (MAX) {
                    v = b > a ? b : a;
                    if (ws_bp) ws_bp[((size_t)n * T + t) * L + j] = b > a;
                } else {
                    v = lse2(a, b);
                }
                v -= shift;
                if (ws_alpha) ws_alpha[((size_t)n * (T + 1) + t + 1) * L + j] = v;
            }
            nxt[j] = v;
            vmax = fmaxf(vmax, v);
        }
        warp_max_store(vmax, wmax + ((t & 1) ^ 1) * 32);
        off += (double)shift;
        if (ws_off && tid == 0) ws_off[(size_t)n * (T + 1) + t + 1] = off;
    }
    cp_async_wait<0>();
    __syncthreads();
    if (tid == 0) {
        const double lz = off + (double)buf[(T & 1) * Lp + len - 1];
        logz[n] = (float)lz;
        if (ws_logz) ws_logz[n] = lz;
    }
}

// Log-semiring gradient: beta_T = [.., 0 at lengths-1, ..] (-inf elsewhere), beta_t[j] = lse(stay[t,j] + beta_{t+1}[j],
// move[t,j] + beta_{t+1}[j+1]); dstay / dmove = g * exp(alpha_t + edge + beta_{t+1} - logZ).
template <int J>
__global__ void __launch_bounds__(TGT_MAX_THREADS)
target_grad_kernel(const float* __restrict__ stay, const float* __restrict__ move, const int* __restrict__ lengths, int T,
                   int N, int L, const float* __restrict__ g, const float* __restrict__ ws_alpha,
                   const double* __restrict__ ws_off, const double* __restrict__ ws_logz, float* __restrict__ dstay,
                   float* __restrict__ dmove) {
    const int n = blockIdx.x, tid = threadIdx.x, B = blockDim.x, nw = B >> 5, Lp = B * J;
    const int len = lengths[n];
    const size_t fs = (size_t)N * L, fm = (size_t)N * (L - 1);
    if (!target_feasible(len, T, L)) {                      // exactly zero, whatever g holds
        for (int t = 0; t < T; ++t) {
            for (int j = tid; j < L; j += B) dstay[(size_t)t * fs + (size_t)n * L + j] = 0.f;
            for (int j = tid; j < L - 1; j += B) dmove[(size_t)t * fm + (size_t)n * (L - 1) + j] = 0.f;
        }
        return;
    }
    extern __shared__ __align__(16) float smf[];
    float* buf = smf;
    float* wmax = buf + 2 * Lp;
    float* rs = wmax + 64;
    float* rm = rs + PF * Lp;
    float* ra = rm + PF * Lp;
    const float* st_n = stay + (size_t)n * L;
    const float* mv_n = move + (size_t)n * (L - 1);
    const float* alpha_n = ws_alpha + (size_t)n * (T + 1) * L;
    const double* off_n = ws_off + (size_t)n * (T + 1);
    const float gn = g[n];
    const double lz = ws_logz[n];
    auto fetch = [&](int i) {
        const int r = T - 1 - i;
        if (r >= 0) {
#pragma unroll
            for (int u = 0; u < J; ++u) {
                const int j = tid + u * B;
                if (j < L) {
                    cp_async_4(&rs[(i % PF) * Lp + j], st_n + (size_t)r * fs + j);
                    cp_async_4(&ra[(i % PF) * Lp + j], alpha_n + (size_t)r * L + j);
                }
                if (j < L - 1) cp_async_4(&rm[(i % PF) * Lp + j], mv_n + (size_t)r * fm + j);
            }
        }
        cp_async_commit();
    };
#pragma unroll
    for (int u = 0; u < J; ++u) {
        const int j = tid + u * B;
        buf[j] = j == len - 1 ? 0.f : -INFINITY;
    }
    if (tid < 32) wmax[tid] = 0.f;
    for (int i = 0; i < PF - 1; ++i) fetch(i);
    double off = 0.0;
    for (int i = 0; i < T; ++i) {
        const int t = T - 1 - i;
        cp_async_wait<PF - 2>();
        __syncthreads();
        fetch(i + PF - 1);
        const float* cur = buf + (i & 1) * Lp;
        float* nxt = buf + ((i & 1) ^ 1) * Lp;
        const float shift = row_shift(wmax + (i & 1) * 32, nw);
        const float k = (float)(off_n[t] + off - lz);
        float vmax = -INFINITY;
#pragma unroll
        for (int u = 0; u < J; ++u) {
            const int j = tid + u * B;
            float v = -INFINITY;
            if (j < L) {
                const float a = ra[(i % PF) * Lp + j] + k;
                const float s = rs[(i % PF) * Lp + j] + cur[j];
                dstay[(size_t)t * fs + (size_t)n * L + j] = gn * expf(a + s);
                float m = -INFINITY;
                if (j < L - 1) {
                    m = rm[(i % PF) * Lp + j] + cur[j + 1];
                    dmove[(size_t)t * fm + (size_t)n * (L - 1) + j] = gn * expf(a + m);
                }
                v = lse2(s, m) - shift;
            }
            nxt[j] = v;
            vmax = fmaxf(vmax, v);
        }
        warp_max_store(vmax, wmax + ((i & 1) ^ 1) * 32);
        off += (double)shift;
    }
    cp_async_wait<0>();
}

// Max-semiring gradient: the best path traced back from state lengths-1 (thread 0), then one-hot dstay / dmove rows.
__global__ void __launch_bounds__(256)
target_max_grad_kernel(const int* __restrict__ lengths, int T, int N, int L, const float* __restrict__ g,
                       const uint8_t* __restrict__ ws_bp, int* __restrict__ ws_path, float* __restrict__ dstay,
                       float* __restrict__ dmove) {
    const int n = blockIdx.x;
    const int len = lengths[n];
    const bool ok = target_feasible(len, T, L);
    int* path = ws_path + (size_t)n * T;                    // 2 * (state at frame t) + 1 if the frame moves
    if (threadIdx.x == 0 && ok) {
        int j = len - 1;
        for (int t = T - 1; t >= 0; --t) {
            const int b = ws_bp[((size_t)n * T + t) * L + j];
            j -= b;
            path[t] = 2 * j + b;
        }
    }
    __syncthreads();
    const float gn = ok ? g[n] : 0.f;
    const size_t fs = (size_t)N * L, fm = (size_t)N * (L - 1);
    for (int t = 0; t < T; ++t) {
        const int hot = ok ? path[t] : -1;
        for (int j = threadIdx.x; j < L; j += blockDim.x) dstay[(size_t)t * fs + (size_t)n * L + j] = hot == 2 * j ? gn : 0.f;
        for (int j = threadIdx.x; j < L - 1; j += blockDim.x)
            dmove[(size_t)t * fm + (size_t)n * (L - 1) + j] = hot == 2 * j + 1 ? gn : 0.f;
    }
}

// threads and states per thread for L target states
void target_shape(int L, int& threads, int& J) {
    J = (L + TGT_MAX_THREADS - 1) / TGT_MAX_THREADS;
    if (J == 3) J = 4;
    const int per = (L + J - 1) / J;
    threads = (per + 31) / 32 * 32;
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------------
// host entry points (abi.cu)
// ---------------------------------------------------------------------------------------------------------------------
static int states_of(int state_len) {
    int S = 1;
    for (int i = 0; i < state_len; ++i) S *= 4;
    return S;
}

size_t ctc_crf_sparse_workspace_bytes(int N, int T, int state_len, int semiring) {
    return SparseWs(nullptr, N, T, states_of(state_len), semiring == B200_SEMIRING_MAX).bytes;
}

size_t ctc_crf_target_workspace_bytes(int N, int T, int L, int semiring) {
    return TargetWs(nullptr, N, T, L, semiring == B200_SEMIRING_MAX).bytes;
}

#define SPARSE_DISPATCH(call)                                      \
    switch (state_len) {                                           \
        case 1: { constexpr int S = 4; return call; }              \
        case 2: { constexpr int S = 16; return call; }             \
        case 3: { constexpr int S = 64; return call; }             \
        case 4: { constexpr int S = 256; return call; }            \
        case 5: { constexpr int S = 1024; return call; }           \
        default:                                                   \
            b200_set_error("ctc_crf: state_len %d is not supported (1..5)", state_len); \
            return -2;                                             \
    }

int launch_ctc_crf_sparse_fwd(const float* scores, int T, int N, int state_len, int semiring, float* logz, float* alpha,
                              void* workspace, cudaStream_t stream) {
    SPARSE_DISPATCH((sparse_fwd<S>(scores, T, N, semiring, logz, alpha, workspace, stream)))
}

int launch_ctc_crf_sparse_bwd(const float* scores, int T, int N, int state_len, int semiring, float* beta,
                              cudaStream_t stream) {
    SPARSE_DISPATCH((sparse_bwd<S>(scores, T, N, semiring, beta, stream)))
}

int launch_ctc_crf_sparse_grad(const float* scores, int T, int N, int state_len, int semiring, const float* g,
                               void* workspace, float* grad, cudaStream_t stream) {
    SPARSE_DISPATCH((sparse_grad<S>(scores, T, N, semiring, g, workspace, grad, stream)))
}

int ctc_crf_target_max_states() { return TGT_MAX_THREADS * TGT_MAX_J; }

int launch_ctc_crf_target_fwd(const float* stay, const float* move, const int* lengths, int T, int N, int L, int semiring,
                              float* logz, void* workspace, cudaStream_t stream) {
    const bool mx = semiring == B200_SEMIRING_MAX;
    TargetWs ws(workspace, N, T, L, mx);
    int threads, J;
    target_shape(L, threads, J);
    const size_t smem = TargetSmem::bytes(threads * J, false);
    void (*k)(const float*, const float*, const int*, int, int, int, float*, float*, double*, double*, uint8_t*);
    switch (J * 2 + mx) {
        case 2: k = target_fwd_kernel<1, false>; break;
        case 3: k = target_fwd_kernel<1, true>; break;
        case 4: k = target_fwd_kernel<2, false>; break;
        case 5: k = target_fwd_kernel<2, true>; break;
        case 8: k = target_fwd_kernel<4, false>; break;
        default: k = target_fwd_kernel<4, true>; break;
    }
    B200_CHECK_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k<<<N, threads, smem, stream>>>(stay, move, lengths, T, N, L, logz, ws.alpha, ws.off, ws.logz, ws.bp);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int launch_ctc_crf_target_grad(const float* stay, const float* move, const int* lengths, int T, int N, int L, int semiring,
                               const float* g, void* workspace, float* dstay, float* dmove, cudaStream_t stream) {
    const bool mx = semiring == B200_SEMIRING_MAX;
    TargetWs ws(workspace, N, T, L, mx);
    if (mx) {
        target_max_grad_kernel<<<N, 256, 0, stream>>>(lengths, T, N, L, g, ws.bp, ws.path, dstay, dmove);
    } else {
        int threads, J;
        target_shape(L, threads, J);
        const size_t smem = TargetSmem::bytes(threads * J, true);
        auto k = J == 1 ? target_grad_kernel<1> : J == 2 ? target_grad_kernel<2> : target_grad_kernel<4>;
        B200_CHECK_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k<<<N, threads, smem, stream>>>(stay, move, lengths, T, N, L, g, ws.alpha, ws.off, ws.logz, dstay, dmove);
    }
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}
