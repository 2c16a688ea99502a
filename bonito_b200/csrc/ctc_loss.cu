// CTC loss: torch.nn.functional.ctc_loss as the QuartzNet models' `Model.loss` uses it (bonito/ctc/model.py:48-57),
// forward (per-sample negative log-likelihood) and gradient, in fp32 in the natural-log domain.
//
// Sample n has the extended label sequence blank, l_1, blank, l_2, ..., blank of S = 2 L + 1 states (L = its target
// length); state s has the class c(s) = blank for even s and l_{(s+1)/2} for odd s.  With lp = log_probs[t][n][:]:
//   alpha_0 = lp_0[c(0)] at s = 0, lp_0[c(1)] at s = 1, -inf elsewhere;
//   alpha_t[s] = lp_t[c(s)] + lse(alpha_{t-1}[s], alpha_{t-1}[s-1], alpha_{t-1}[s-2] when s is odd and l(s) != l(s-2));
//   nll = -lse(alpha_{T_n-1}[S-1], alpha_{T_n-1}[S-2]), T_n = input_lengths[n];
//   beta (torch's, which includes lp_t like alpha) mirrors alpha from beta_{T_n-1} = lp at S-1 and S-2;
//   grad[t][n][c] = (exp(lp_t[c]) - sum over the states s of class c of exp(alpha_t[s] + beta_t[s] + nll - lp_t[c])) * g[n]
//     for t < T_n, and exactly 0 for t >= T_n.
// The sum is torch's exp(lcab + nll - lp) written as a sum of per-state posteriors, which stay in [0, 1] in fp32.  Where
// torch's CPU expression is not finite this one is not either, in the same places: a sample with nll = inf gets NaN on
// every frame t < T_n (0 with zero_infinity), and a class with lp = -inf gets NaN, also when no state has that class.
//
// One CTA per sample, one thread per state (strided by the block size for S > 1024), a double-buffered alpha / beta row
// in shared memory and one barrier per frame.  Every row is re-centred on the previous row's maximum and the shifts are
// summed in fp64, so the fp32 error does not grow with |nll|.  The forward keeps the re-centred alpha rows ([N][T][S_max],
// what torch keeps too), their fp64 offsets and the fp64 nll in the caller's workspace; the gradient kernel is one
// backward pass that streams those rows and the log-prob rows through a PF-deep cp.async ring (PF = 4, or 2 when the
// longest targets would not fit in shared memory), produces beta and writes each frame's posteriors to shared memory.
// The per-class sums of a frame are done one frame later, by warp c % warps for class c: each lane adds its states in
// order and the warp combines the lanes by a fixed butterfly, so every output is bitwise reproducible (no atomics).
// log_probs may have any strides on T and N (the class axis is contiguous); targets are read through per-sample offsets,
// so the padded [N, S] and the concatenated 1-D forms are the same to the kernels.  A sample whose lengths, target offset
// or labels are out of range gets a NaN loss and gradient and is never read out of bounds.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int MAX_THREADS = 1024;

struct Args {
    const float* lp;
    long long st, sn;             // strides of log_probs on T and N, in elements
    int T, N, C;
    const int* in_len;
    const int* targets;
    long long n_targets;          // elements of `targets`
    const long long* tgt_off;     // start of each sample's labels in `targets`
    const int* tgt_len;
    int max_target, blank;
};

inline size_t align256(size_t x) { return (x + 255) / 256 * 256; }
__host__ __device__ inline int states_max(int max_target) { return 2 * max_target + 1; }
__host__ __device__ inline int pad4(int x) { return (x + 3) & ~3; }

// Workspace for N samples of T frames: alpha' float [N][T][S_max], offsets double [N][T], nll double [N].
struct Ws {
    float* alpha = nullptr;
    double* off = nullptr;
    double* nll = nullptr;
    size_t bytes = 0;
    Ws(void* base, int N, int T, int max_target) {
        unsigned char* ws = static_cast<unsigned char*>(base);
        auto take = [&](size_t b) { unsigned char* p = ws ? ws + bytes : nullptr; bytes += align256(b); return p; };
        alpha = reinterpret_cast<float*>(take((size_t)N * T * states_max(max_target) * sizeof(float)));
        off = reinterpret_cast<double*>(take((size_t)N * T * sizeof(double)));
        nll = reinterpret_cast<double*>(take((size_t)N * sizeof(double)));
    }
};

__device__ __forceinline__ void cp_async_4(void* smem_dst, const void* gmem_src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(smem_u32(smem_dst)), "l"(gmem_src));
}

__device__ __forceinline__ float lse3(float a, float b, float c) {
    const float m = fmaxf(fmaxf(a, b), c);
    if (m == -INFINITY) return m;
    return m + logf(expf(a - m) + expf(b - m) + expf(c - m));
}

__device__ __forceinline__ float row_shift(const float* wmax, int nw) {
    float m = -INFINITY;
    for (int w = 0; w < nw; ++w) m = fmaxf(m, wmax[w]);
    return m > -INFINITY ? m : 0.f;
}

__device__ __forceinline__ void warp_max_store(float v, float* wmax) {
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = v;
}

// Sample n's labels into tg (bytes: C <= 256), its input length into il.  Returns its target length, or -1 when a length,
// the target offset or a label is out of range.  Every thread of the CTA must call it.
__device__ int load_sample(const Args& a, int n, unsigned char* tg, int& il) {
    il = a.in_len[n];
    const int tl = a.tgt_len[n];
    const long long off = a.tgt_off[n];
    const bool ok = il >= 1 && il <= a.T && tl >= 0 && tl <= a.max_target && off >= 0 && off + tl <= a.n_targets;
    int bad = !ok;
    if (ok) {
        for (int j = threadIdx.x; j < tl; j += blockDim.x) {
            const int c = a.targets[off + j];
            bad |= c < 0 || c >= a.C;
            tg[j] = (unsigned char)c;
        }
    }
    return __syncthreads_or(bad) ? -1 : tl;
}

__device__ __forceinline__ int state_class(int s, const unsigned char* tg, int blank) {
    return s & 1 ? tg[s >> 1] : blank;
}

// Forward.  nll [N]; with WS also the alpha' rows, their offsets and the fp64 nll for the gradient kernel.
template <bool WS>
__global__ void __launch_bounds__(MAX_THREADS)
ctc_loss_fwd_kernel(Args a, float* __restrict__ nll, float* __restrict__ ws_alpha, double* __restrict__ ws_off,
                    double* __restrict__ ws_nll) {
    constexpr int PF = 4;
    const int Sm = states_max(a.max_target), Sp = pad4(Sm), Cp = pad4(a.C);
    extern __shared__ __align__(16) float smf[];
    float* buf = smf;                    // [2][Sp]
    float* ring = buf + 2 * Sp;          // [PF][Cp] log-prob rows
    float* wmax = ring + PF * Cp;        // [2][32]
    unsigned char* tg = reinterpret_cast<unsigned char*>(wmax + 64);
    const int n = blockIdx.x, tid = threadIdx.x, B = blockDim.x, nw = B >> 5;
    int il;
    const int tl = load_sample(a, n, tg, il);
    if (tl < 0) {
        if (tid == 0) {
            nll[n] = NAN;
            if (WS) ws_nll[n] = NAN;
        }
        return;
    }
    const int S = 2 * tl + 1;
    const float* lp_n = a.lp + (long long)n * a.sn;
    auto fetch = [&](int t) {
        if (t < il)
            for (int c = tid; c < a.C; c += B) cp_async_4(&ring[(t % PF) * Cp + c], lp_n + (long long)t * a.st + c);
        cp_async_commit();
    };
    // the row before frame 0 is [0, -inf, ...]: the recursion then gives alpha_0
    for (int s = tid; s < Sp; s += B) buf[s] = s == 0 ? 0.f : -INFINITY;
    for (int i = tid; i < 64; i += B) wmax[i] = 0.f;
    for (int r = 0; r < PF - 1; ++r) fetch(r);
    double off = 0.0;                    // alpha_t = alpha'_t + off
    for (int t = 0; t < il; ++t) {
        cp_async_wait<PF - 2>();
        __syncthreads();
        fetch(t + PF - 1);
        const float* cur = buf + (t & 1) * Sp;
        float* nxt = buf + ((t & 1) ^ 1) * Sp;
        const float* row = ring + (t % PF) * Cp;
        const float shift = row_shift(wmax + (t & 1) * 32, nw);
        float vmax = -INFINITY;
        for (int s = tid; s < S; s += B) {
            const float x1 = s >= 1 ? cur[s - 1] : -INFINITY;
            const float x2 = (s & 1) && s >= 3 && tg[s >> 1] != tg[(s >> 1) - 1] ? cur[s - 2] : -INFINITY;
            const float v = row[state_class(s, tg, a.blank)] + lse3(cur[s], x1, x2) - shift;
            nxt[s] = v;
            if (WS) ws_alpha[((size_t)n * a.T + t) * Sm + s] = v;
            vmax = fmaxf(vmax, v);
        }
        warp_max_store(vmax, wmax + ((t & 1) ^ 1) * 32);
        off += (double)shift;
        if (WS && tid == 0) ws_off[(size_t)n * a.T + t] = off;
    }
    cp_async_wait<0>();
    __syncthreads();
    if (tid == 0) {
        const float* fin = buf + (il & 1) * Sp;
        const float m = lse3(fin[S - 1], tl > 0 ? fin[S - 2] : -INFINITY, -INFINITY);
        const double v = m == -INFINITY ? (double)INFINITY : -(off + (double)m);
        nll[n] = (float)v;
        if (WS) ws_nll[n] = v;
    }
}

// Gradient from the forward's workspace: grad [T][N][C] contiguous.
template <int PF>
__global__ void __launch_bounds__(MAX_THREADS)
ctc_loss_grad_kernel(Args a, const float* __restrict__ g, int zero_infinity, const float* __restrict__ ws_alpha,
                     const double* __restrict__ ws_off, const double* __restrict__ ws_nll, float* __restrict__ grad) {
    const int Sm = states_max(a.max_target), Sp = pad4(Sm), Cp = pad4(a.C);
    extern __shared__ __align__(16) float smf[];
    float* bbuf = smf;                   // [2][Sp] beta' rows
    float* post = bbuf + 2 * Sp;         // [2][Sp] per-state posteriors of a frame
    float* aring = post + 2 * Sp;        // [PF][Sp] alpha' rows
    float* lring = aring + PF * Sp;      // [PF][Cp] log-prob rows
    float* lprev = lring + PF * Cp;      // [2][Cp] the log-prob row of the frame whose posteriors are in post
    float* wmax = lprev + 2 * Cp;        // [2][32]
    unsigned char* tg = reinterpret_cast<unsigned char*>(wmax + 64);
    const int n = blockIdx.x, tid = threadIdx.x, B = blockDim.x, nw = B >> 5, lane = tid & 31, warp = tid >> 5;
    const int C = a.C;
    auto fill = [&](int t0, int t1, float v) {
        for (int t = t0; t < t1; ++t)
            for (int c = tid; c < C; c += B) grad[((size_t)t * a.N + n) * C + c] = v;
    };
    int il;
    const int tl = load_sample(a, n, tg, il);
    if (tl < 0) {
        fill(0, a.T, NAN);
        return;
    }
    fill(il, a.T, 0.f);
    const double nll = ws_nll[n];
    if (!(nll < (double)INFINITY)) {     // infeasible (inf) or NaN: torch's exp(-inf + inf) is NaN on every frame
        fill(0, il, zero_infinity && nll == (double)INFINITY ? 0.f : NAN);
        return;
    }
    const int S = 2 * tl + 1;
    const float gn = g[n];
    const float* lp_n = a.lp + (long long)n * a.sn;
    const float* alpha_n = ws_alpha + (size_t)n * a.T * Sm;
    const double* off_n = ws_off + (size_t)n * a.T;
    // each thread copies, and later reads, only its own states of the alpha' rows; the log-prob rows are read by all
    auto fetch = [&](int i) {                                // iteration i handles frame il - 1 - i
        const int r = il - 1 - i;
        if (r >= 0) {
            for (int c = tid; c < C; c += B) cp_async_4(&lring[(i % PF) * Cp + c], lp_n + (long long)r * a.st + c);
            for (int s = tid; s < S; s += B) cp_async_4(&aring[(i % PF) * Sp + s], alpha_n + (size_t)r * Sm + s);
        }
        cp_async_commit();
    };
    // the row after frame il - 1 is 0 at S - 1 and -inf elsewhere: the recursion then gives beta_{il-1}
    for (int s = tid; s < Sp; s += B) bbuf[s] = s == S - 1 ? 0.f : -INFINITY;
    for (int i = tid; i < 64; i += B) wmax[i] = 0.f;
    for (int r = 0; r < PF - 1; ++r) fetch(r);
    double off = 0.0;                                       // beta_t = beta'_t + off
    for (int i = 0; i <= il; ++i) {
        cp_async_wait<PF - 2>();
        __syncthreads();
        if (i > 0) {                                        // the class sums of frame il - i, computed last iteration
            const float* p = post + ((i - 1) & 1) * Sp;
            const float* lrow = lprev + ((i - 1) & 1) * Cp;
            const int t = il - i;
            for (int c = warp; c < C; c += nw) {
                float sum = 0.f;
                int any = 0;
                if (c == a.blank) {
                    any = 1;
                    for (int s = 2 * lane; s < S; s += 64) sum += p[s];
                }
                for (int j = lane; j < tl; j += 32)
                    if (tg[j] == c) { sum += p[2 * j + 1]; any = 1; }
                for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
                any = __any_sync(0xffffffffu, any);
                if (lane == 0) {
                    const float l = lrow[c];
                    const float term = any ? sum : (l == -INFINITY ? NAN : 0.f);
                    grad[((size_t)t * a.N + n) * C + c] = (expf(l) - term) * gn;
                }
            }
        }
        if (i == il) break;
        const int t = il - 1 - i;
        fetch(i + PF - 1);
        const float* cur = bbuf + (i & 1) * Sp;
        float* nxt = bbuf + ((i & 1) ^ 1) * Sp;
        const float* lrow = lring + (i % PF) * Cp;
        const float* arow = aring + (i % PF) * Sp;
        float* p = post + (i & 1) * Sp;
        const float shift = row_shift(wmax + (i & 1) * 32, nw);
        off += (double)shift;
        const float k = (float)(off_n[t] + off + nll);
        for (int c = tid; c < C; c += B) lprev[(i & 1) * Cp + c] = lrow[c];
        float vmax = -INFINITY;
        for (int s = tid; s < S; s += B) {
            const float x1 = s + 1 < S ? cur[s + 1] : -INFINITY;
            const float x2 = (s & 1) && s + 2 < S && tg[s >> 1] != tg[(s >> 1) + 1] ? cur[s + 2] : -INFINITY;
            const float l = lrow[state_class(s, tg, a.blank)];
            const float v = l + lse3(cur[s], x1, x2) - shift;
            nxt[s] = v;
            vmax = fmaxf(vmax, v);
            p[s] = expf(arow[s] + v + k - l);
        }
        warp_max_store(vmax, wmax + ((i & 1) ^ 1) * 32);
    }
    cp_async_wait<0>();
}

int block_threads(int max_target) {
    const int Sm = states_max(max_target);
    return Sm >= MAX_THREADS ? MAX_THREADS : (Sm + 31) / 32 * 32;
}

size_t fwd_smem(int max_target, int C) {
    return (2 * pad4(states_max(max_target)) + 4 * pad4(C) + 64) * sizeof(float) + (size_t)max_target;
}

size_t grad_smem(int max_target, int C, int pf) {
    return ((4 + pf) * pad4(states_max(max_target)) + (pf + 2) * pad4(C) + 64) * sizeof(float) + (size_t)max_target;
}

}  // namespace

#define CTC_LOSS_CHECK(what)                                                                                           \
    B200_REQUIRE(n >= 0 && t >= 1 && c >= 1 && c <= B200_CTC_LOSS_MAX_CLASSES,                                         \
                 what ": bad sizes n=%d t=%d c=%d (1 <= c <= %d)", n, t, c, B200_CTC_LOSS_MAX_CLASSES);                \
    B200_REQUIRE(max_target >= 0 && max_target <= B200_CTC_LOSS_MAX_TARGET,                                            \
                 what ": max_target %d is outside 0..%d", max_target, B200_CTC_LOSS_MAX_TARGET);                       \
    B200_REQUIRE(blank >= 0 && blank < c, what ": blank %d is outside [0, %d)", blank, c);                             \
    B200_REQUIRE(stride_t >= 0 && stride_n >= 0 && n_targets >= 0, what ": negative stride or target count");          \
    B200_REQUIRE(log_probs && input_lengths && target_off && target_lengths && (targets || n_targets == 0),            \
                 what ": null pointer argument")

#define CTC_LOSS_ARGS                                                                                                  \
    Args{(const float*)log_probs, stride_t, stride_n, t, n, c, (const int*)input_lengths, (const int*)targets,         \
         n_targets, (const long long*)target_off, (const int*)target_lengths, max_target, blank}

extern "C" {

int b200_ctc_loss_max_target(void) { return B200_CTC_LOSS_MAX_TARGET; }

size_t b200_ctc_loss_workspace_bytes(int n, int t, int max_target) {
    if (n < 0 || t < 0 || max_target < 0 || max_target > B200_CTC_LOSS_MAX_TARGET) return 0;
    return Ws(nullptr, n, t, max_target).bytes;
}

int b200_ctc_loss_fwd(const void* log_probs, long long stride_t, long long stride_n, int t, int n, int c,
                      const void* input_lengths, const void* targets, long long n_targets, const void* target_off,
                      const void* target_lengths, int max_target, int blank, void* nll, void* workspace, void* stream) {
    CTC_LOSS_CHECK("ctc_loss_fwd");
    B200_REQUIRE(nll, "ctc_loss_fwd: null nll");
    if (n == 0) return 0;
    const Args a = CTC_LOSS_ARGS;
    const Ws ws(workspace, n, t, max_target);
    const size_t smem = fwd_smem(max_target, c);
    auto k = workspace ? ctc_loss_fwd_kernel<true> : ctc_loss_fwd_kernel<false>;
    B200_CHECK_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k<<<n, block_threads(max_target), smem, (cudaStream_t)stream>>>(a, (float*)nll, ws.alpha, ws.off, ws.nll);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int b200_ctc_loss_grad(const void* log_probs, long long stride_t, long long stride_n, int t, int n, int c,
                       const void* input_lengths, const void* targets, long long n_targets, const void* target_off,
                       const void* target_lengths, int max_target, int blank, const void* g, int zero_infinity,
                       void* workspace, void* grad, void* stream) {
    CTC_LOSS_CHECK("ctc_loss_grad");
    B200_REQUIRE(g && workspace && grad, "ctc_loss_grad: null pointer argument");
    if (n == 0) return 0;
    const Args a = CTC_LOSS_ARGS;
    const Ws ws(workspace, n, t, max_target);
    int dev, optin;
    B200_CHECK_CUDA(cudaGetDevice(&dev));
    B200_CHECK_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    const bool deep = grad_smem(max_target, c, 4) <= (size_t)optin;
    const size_t smem = grad_smem(max_target, c, deep ? 4 : 2);
    B200_REQUIRE(smem <= (size_t)optin, "ctc_loss_grad: %zu bytes of shared memory needed, the device has %d", smem, optin);
    auto k = deep ? ctc_loss_grad_kernel<4> : ctc_loss_grad_kernel<2>;
    B200_CHECK_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k<<<n, block_threads(max_target), smem, (cudaStream_t)stream>>>(a, (const float*)g, zero_infinity, ws.alpha, ws.off,
                                                                     ws.nll, (float*)grad);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // extern "C"
