// CRF decode: forward-backward posteriors followed by a Viterbi pass over the log-posteriors,
// i.e. the in-repo decode definition of the reference
//     SeqdistModel.decode_batch  (bonito/crf/model.py:196-199)
//       posteriors(x.float()) + 1e-8 -> log -> CTC_CRF.viterbi (bonito/crf/model.py:98-103)
// on the sparse 5-edge state graph of CTC_CRF (bonito/crf/model.py:37-42):
//     in-edge e=0 of state s comes from s itself (stay, fixed blank score),
//     in-edge e=1+j comes from state j*S/4 + s/4 (move, emits base s%4).
// Scores arrive without the blank column, [N][T][S*4] fp16 (the layout the reference hands to
// koi.decode.beam_search, bonito/crf/basecall.py:36-40); outputs follow that call's contract:
// three [N][T] byte arrays (moves 0/1, base char or 0, quality char or 0).
//
// One CTA per chunk, one thread per state.  All recurrences run in fp32 on values re-centred on
// state 0 every step; the accumulated shifts are carried in fp64 so the per-step posterior
// normaliser is exact to fp32 rounding no matter how long the chunk is.
//   pass 1 (t = T-1..0): beta'      -> workspace (fp32 [T+1][S]) + shift sums (fp64 [T+1]) + logZ
//   pass 2 (t = 0..T-1): alpha', posteriors, per-base move mass, Viterbi scores + back-pointers
//   pass 3: trace-back through the back-pointers (staged through shared memory in blocks)
// Tie-breaks (the reference's are whatever argmax over koi's Max-semiring gradient gives):
// lowest in-edge index, lowest final state.
//
// Learned blank scores (LB = true, b200_crf_decode_lb): heads without a fixed blank_score emit the stay score of every state at
// every frame, [N][T][S*5] in the CTC_CRF layout [state][stay, move 0..3].  Rows of 10*S bytes do not split into one aligned
// 8-byte piece per thread, so each score row is copied whole into the shared-memory ring with cooperative 16-byte cp.async
// copies (5S/8 threads, one piece each) and every thread reads its five values from there.  A thread now reads what other
// threads copied, so a row must be complete and published by a barrier before its step: the rings run one step further
// ahead (each step waits for the row after next) and the per-step barrier that is already there publishes it.  Every other
// line of the three passes is the fixed-blank code, which these rows also keep bit-identical when the stay column is the
// fixed score.
#include <stdlib.h>

#include "common.cuh"

namespace {

constexpr float LOG2E = 1.4426950408889634f;

__device__ __forceinline__ float lg2_approx(float x) {
    float y;
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
// log2(sum_i 2^x_i) of five values: one max tree, five bare ex2 and one bare lg2 (the largest term contributes 2^0 = 1, so
// the sum is in [1, 5] and flushing sub-normal terms to zero changes nothing)
__device__ __forceinline__ float lse2_5(float a, float b, float c, float d, float e) {
    const float m = fmaxf(fmaxf(fmaxf(a, b), fmaxf(c, d)), e);
    const float s = ex2_approx(a - m) + ex2_approx(b - m) + ex2_approx(c - m) + ex2_approx(d - m) + ex2_approx(e - m);
    return m + lg2_approx(s);
}

template <int S, bool LB>
struct DecodeSmem {
    static constexpr int NW = (S + 31) / 32;
    static constexpr int TB = 16384 / S;                 // back-pointer rows per trace-back block
    static constexpr size_t kAv = 0;                                   // float2 [2][S]: (alpha', Viterbi score) | float [2][S] in pass 1
    static constexpr size_t kUnion = kAv + 2 * S * sizeof(float2);     // float [2][4*S]  |  u8 [TB][S]
    static constexpr size_t kUnionBytes = (2 * 4 * S * sizeof(float) > (size_t)TB * S) ? 2 * 4 * S * sizeof(float) : (size_t)TB * S;
    static constexpr size_t kPart = kUnion + kUnionBytes;              // float [2][NW][4]
    static constexpr size_t kKt = kPart + 2 * NW * 4 * sizeof(float);  // float [2]: per-step posterior normaliser
    static constexpr int PF = 4;                                       // prefetch depth (steps) of the cp.async rings
    static constexpr size_t kScRow = LB ? 5 * S * sizeof(__half) : S * sizeof(uint2);   // bytes per score row
    static constexpr size_t kScRing = kKt + 16;                        // [PF] score rows in flight: uint2 [S] | half [S][5]
    static constexpr size_t kBetaRing = kScRing + PF * kScRow;         // float [PF][S]: beta' rows in flight (pass 2)
    static constexpr size_t kRed = kBetaRing + PF * S * sizeof(float);
    static constexpr size_t kRedI = kRed + NW * sizeof(float);
    static constexpr size_t kOut = kRedI + NW * sizeof(int) + 16;      // u8 [3][T]
    static size_t bytes(int T) { return kOut + 3 * (size_t)T + 16; }
};

template <int V>
struct IntC { static constexpr int value = V; };

// 8- / 4-byte asynchronous copies global -> shared (LDGSTS): the per-step score and beta' rows are fetched PF steps ahead
// into shared-memory rings; every thread reads back only the element it copied itself, so its own wait_group is enough.
// (With a one-step register prefetch the global-load latency was the top stall of this kernel next to the per-step barrier.)
__device__ __forceinline__ void cp_async_8(void* smem_dst, const void* gmem_src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"(smem_u32(smem_dst)), "l"(gmem_src));
}
__device__ __forceinline__ void cp_async_4(void* smem_dst, const void* gmem_src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(smem_u32(smem_dst)), "l"(gmem_src));
}

// All recurrences run in the log2 domain (scores are multiplied by log2(e) once when they are loaded): every
// exponential / logarithm is then a single bare MUFU instruction.  (The first version of this kernel used __expf / __logf
// in the natural-log domain: 195 + 86 SASS instructions per forward / backward state-step, a third of them the FMUL /
// FSETP range handling around each MUFU; this one needs ~105 + ~55.)  The step loops are unrolled by two so that every
// buffer that flips with the step parity is a compile-time address.
template <int S, bool LB>
__global__ void __launch_bounds__(S)
crf_decode_kernel(const __half* __restrict__ scores, int T, float blank, float qscale, float qbias,
                  float* __restrict__ ws_beta, double* __restrict__ ws_bsum, uint8_t* __restrict__ ws_bp,
                  float* __restrict__ ws_pm, uint8_t* __restrict__ moves, uint8_t* __restrict__ seq,
                  uint8_t* __restrict__ qual) {
    using L = DecodeSmem<S, LB>;
    constexpr int Q = S / 4, NW = L::NW, TB = L::TB;
    extern __shared__ __align__(16) unsigned char sm[];
    float (*buf)[S] = reinterpret_cast<float (*)[S]>(sm + L::kAv);            // pass 1: beta'
    float2 (*av)[S] = reinterpret_cast<float2 (*)[S]>(sm + L::kAv);           // pass 2: (alpha', Viterbi)
    float (*msh)[4 * S] = reinterpret_cast<float (*)[4 * S]>(sm + L::kUnion);
    uint8_t (*bp_blk)[S] = reinterpret_cast<uint8_t (*)[S]>(sm + L::kUnion);
    float (*part)[NW][4] = reinterpret_cast<float (*)[NW][4]>(sm + L::kPart);
    float* kt_sh = reinterpret_cast<float*>(sm + L::kKt);
    constexpr int PF = L::PF;
    uint2 (*sc_ring)[S] = reinterpret_cast<uint2 (*)[S]>(sm + L::kScRing);
    unsigned char* sc_ring_lb = sm + L::kScRing;                             // LB: half [PF][S][5]
    float (*beta_ring)[S] = reinterpret_cast<float (*)[S]>(sm + L::kBetaRing);
    float* red = reinterpret_cast<float*>(sm + L::kRed);
    int* red_i = reinterpret_cast<int*>(sm + L::kRedI);
    uint8_t* out_sh = sm + L::kOut;
    __shared__ float logz_sh;

    const int n = blockIdx.x;
    const int s = threadIdx.x;
    const int lane = s & 31, warp = s >> 5;
    const uint2* sc = reinterpret_cast<const uint2*>(scores + (size_t)n * T * S * 4) + s;  // row stride S
    const unsigned char* sc_lb = reinterpret_cast<const unsigned char*>(scores + (size_t)n * T * S * 5);  // LB: rows of kScRow B
    // score row r -> ring slot r % PF: fixed blank, this thread's 8 bytes; learned blank, the whole row in 16-byte pieces
    auto fetch_row = [&](int r) {
        if constexpr (LB) {
            if (s < (int)(L::kScRow / 16))
                cp_async_16(sc_ring_lb + (r & (PF - 1)) * L::kScRow + s * 16, sc_lb + (size_t)r * L::kScRow + s * 16, true);
        } else {
            cp_async_8(&sc_ring[r & (PF - 1)][s], sc + (size_t)r * S);
        }
    };
    // LB: the five scores of state s in ring slot `slot`
    auto lb_row = [&](int slot) { return reinterpret_cast<const __half*>(sc_ring_lb + slot * L::kScRow) + 5 * s; };
    float* beta = ws_beta + (size_t)n * (T + 1) * S;
    double* bsum = ws_bsum + (size_t)n * (T + 1);
    uint8_t* bp = ws_bp + (size_t)n * T * S;
    float* pm = ws_pm + (size_t)n * T * 4;
    const float blank2 = blank * LOG2E;

    // ---------------- pass 1: backward ----------------
    // beta'_t[p] = log2-sum over the out-edges of p (stay, and the moves into the four successors 4(p%Q)+c), re-centred on
    // state 0 of the previous step; the accumulated shifts are kept in fp64 by thread 0 (bsum).
    {
        buf[0][s] = 0.f;
        beta[(size_t)T * S + s] = 0.f;
        if (s == 0) bsum[T] = 0.0;
        // scatter the 4 in-edge move scores of state s to their consumers: in-edge j of s leaves predecessor
        // p = j*Q + s/4 as its b = s%4 -th out-edge -> msh[4p+b] = msh[j*S+s]
        auto scatter = [&](float* dst, uint2 raw) {
            const float2 m01 = __half22float2(*reinterpret_cast<const __half2*>(&raw.x));
            const float2 m23 = __half22float2(*reinterpret_cast<const __half2*>(&raw.y));
            dst[0 * S + s] = m01.x * LOG2E; dst[1 * S + s] = m01.y * LOG2E;
            dst[2 * S + s] = m23.x * LOG2E; dst[3 * S + s] = m23.y * LOG2E;
        };
        // LB: the moves of state s from its five scores [stay, m0..m3]; returns the stay score (log2 units)
        auto scatter_lb = [&](float* dst, const __half* e) {
            dst[0 * S + s] = __half2float(e[1]) * LOG2E; dst[1 * S + s] = __half2float(e[2]) * LOG2E;
            dst[2 * S + s] = __half2float(e[3]) * LOG2E; dst[3 * S + s] = __half2float(e[4]) * LOG2E;
            return __half2float(e[0]) * LOG2E;
        };
        float stay_cur = blank2;                                   // LB: stay score of state s at the current step
        if constexpr (LB) {
            stay_cur = scatter_lb(msh[0], reinterpret_cast<const __half*>(sc_lb + (size_t)(T - 1) * L::kScRow) + 5 * s);
        } else {
            scatter(msh[0], sc[(size_t)(T - 1) * S]);
        }
        // score rows T-2, T-3, ... travel through the ring: row r lives in slot r % PF; PF-1 groups are kept in flight
        for (int r = T - 2; r > T - 2 - (PF - 1); --r) {
            if (r >= 0) fetch_row(r);
            cp_async_commit();
        }
        if constexpr (LB) cp_async_wait<PF - 2>();                 // row T-2, published by the barrier below
        float* beta_p = beta + (size_t)(T - 1) * S + s;
        double* bsum_p = bsum + (T - 1);
        double acc_shift = 0.0;
        __syncthreads();
        auto bwd = [&](int t, auto cur_c) {
            constexpr int CUR = decltype(cur_c)::value;
            {   // next row into the ring (row t-PF; its slot held row t, scattered in the previous step), then wait for row t-1
                // (LB: for row t-2, which the barrier at the end of this step publishes for the next one)
                const int r = t - PF;
                if (r >= 0) fetch_row(r);
                cp_async_commit();
                if constexpr (LB) cp_async_wait<PF - 2>();
                else cp_async_wait<PF - 1>();
            }
            [[maybe_unused]] float stay_next = 0.f;
            if constexpr (LB) {
                if (t > 0) stay_next = scatter_lb(msh[CUR ^ 1], lb_row((t - 1) & (PF - 1)));
            } else {
                if (t > 0) scatter(msh[CUR ^ 1], sc_ring[(t - 1) & (PF - 1)][s]);
            }
            const float b0 = buf[CUR][0];
            const float4 mv = *reinterpret_cast<const float4*>(&msh[CUR][4 * s]);
            const float4 bs = *reinterpret_cast<const float4*>(&buf[CUR][4 * (s % Q)]);
            const float v = lse2_5(stay_cur + buf[CUR][s], mv.x + bs.x, mv.y + bs.y, mv.z + bs.z, mv.w + bs.w) - b0;
            if constexpr (LB) stay_cur = stay_next;
            buf[CUR ^ 1][s] = v;
            *beta_p = v;
            beta_p -= S;
            if (warp == 0) {
                if (lane == 0) {
                    acc_shift += (double)b0;
                    *bsum_p = acc_shift;
                }
            }
            --bsum_p;
            __syncthreads();
        };
        int t = T - 1;
        for (; t >= 1; t -= 2) { bwd(t, IntC<0>()); bwd(t - 1, IntC<1>()); }
        if (t == 0) bwd(0, IntC<0>());
        // log2 Z = bsum[0] + log2-sum_s beta'_0[s]
        const float v = buf[T & 1][s];
        float mx = v;
        for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        if (lane == 0) red[warp] = mx;
        __syncthreads();
        mx = red[0];
        for (int w = 1; w < NW; ++w) mx = fmaxf(mx, red[w]);
        __syncthreads();
        float ex = ex2_approx(v - mx);
        for (int o = 16; o > 0; o >>= 1) ex += __shfl_xor_sync(0xffffffffu, ex, o);
        if (lane == 0) red[warp] = ex;
        __syncthreads();
        if (s == 0) {
            float tot = 0.f;
            for (int w = 0; w < NW; ++w) tot += red[w];
            logz_sh = mx + lg2_approx(tot);
        }
        __syncthreads();
    }

    // ---------------- pass 2: forward + posteriors + Viterbi ----------------
    // Rows are stored re-centred: alpha'_{t+1}[s] = log2-sum_e(alpha'_t[pred] + M_t[s,e]) - alpha'_t[0], so the true
    // alpha_t = alpha'_t + asum_t with asum_{t+1} = asum_t + alpha'_t[0]; likewise beta_t = beta'_t + bsum[t].  The
    // posterior of edge (s, e) at step t is 2^(alpha'_t[pred] + M_t[s,e] + beta'_{t+1}[s] + k_t) with the per-step normaliser
    //   k_t = asum_t + bsum[t+1] - log2 Z,
    // computed in fp64 by thread 0 one step ahead (exact to fp32 rounding however long the chunk is) and broadcast
    // through shared memory.
    {
        const double logz = bsum[0] + (double)logz_sh;
        const int pq = s / 4;  // predecessor along in-edge 1+j is j*Q + pq
        av[0][s] = make_float2(0.f, 0.f);
        double asum = 0.0;     // thread 0: sum of the alpha' re-centring shifts before step t
        if (s == 0) kt_sh[0] = (float)(bsum[1] - logz);       // step 0: alpha'_0 = 0, asum = 0
        __syncthreads();
        cp_async_wait<0>();
        // score row t and beta' row t+1 of step t live in slot t % PF of the rings; PF-1 steps are kept in flight
        for (int r = 0; r < PF - 1; ++r) {
            if (r < T) {
                fetch_row(r);
                cp_async_4(&beta_ring[r][s], beta + (size_t)(r + 1) * S + s);
            }
            cp_async_commit();
        }
        if constexpr (LB) {                                   // row 0, complete and published before step 0
            cp_async_wait<PF - 2>();
            __syncthreads();
        }
        double bs_next2 = (T > 1 && s == 0) ? bsum[2] : 0.0;   // thread 0: bsum[t+2], for the normaliser of step t+1
        const double* bsum_p = bsum + 3;
        uint8_t* bp_p = bp + s;
        float* pm_p = pm + s;                                 // used by threads 0..3
        auto fwd = [&](int t, auto cur_c) {
            constexpr int CUR = decltype(cur_c)::value;
            double bs_n = 0.0;
            {
                const int r = t + PF - 1;
                if (r < T) {
                    fetch_row(r);
                    cp_async_4(&beta_ring[r & (PF - 1)][s], beta + (size_t)(r + 1) * S + s);
                }
                cp_async_commit();
                if (s == 0 && t + 3 <= T) bs_n = *bsum_p;
                // LB: row t+1 as well, published for the next step by the barrier of this one
                if constexpr (LB) cp_async_wait<PF - 2>();
                else cp_async_wait<PF - 1>();
            }
            ++bsum_p;
            const float bnext = beta_ring[t & (PF - 1)][s];
            float2 m01, m23;
            float stay2 = blank2;
            if constexpr (LB) {
                const __half* e = lb_row(t & (PF - 1));
                stay2 = __half2float(e[0]) * LOG2E;
                m01 = make_float2(__half2float(e[1]), __half2float(e[2]));
                m23 = make_float2(__half2float(e[3]), __half2float(e[4]));
            } else {
                const uint2 mraw = sc_ring[t & (PF - 1)][s];
                m01 = __half22float2(*reinterpret_cast<const __half2*>(&mraw.x));
                m23 = __half22float2(*reinterpret_cast<const __half2*>(&mraw.y));
            }
            const float2 a0v0 = av[CUR][0];
            const float kt = kt_sh[CUR];
            float2 p[5];
            p[0] = av[CUR][s];
#pragma unroll
            for (int j = 0; j < 4; ++j) p[1 + j] = av[CUR][j * Q + pq];
            float x[5];
            x[0] = p[0].x + stay2;
            x[1] = fmaf(m01.x, LOG2E, p[1].x);
            x[2] = fmaf(m01.y, LOG2E, p[2].x);
            x[3] = fmaf(m23.x, LOG2E, p[3].x);
            x[4] = fmaf(m23.y, LOG2E, p[4].x);
            // log2-sum of the five in-edges; its exponentials 2^(x_e - m) are shared with the posteriors:
            //   post_e = 2^(x_e + beta'_{t+1}[s] + k_t) = 2^(x_e - m) * 2^(m + beta'_{t+1}[s] + k_t)      (12 MUFU per state-step, not 16)
            const float m = fmaxf(fmaxf(fmaxf(x[0], x[1]), fmaxf(x[2], x[3])), x[4]);
            const float g = ex2_approx(m + bnext + kt);
            float best = -INFINITY, mass = 0.f, esum = 0.f;
            int arg = 0;
#pragma unroll
            for (int e = 0; e < 5; ++e) {
                const float ee = ex2_approx(x[e] - m);
                esum += ee;
                const float post = ee * g;
                if (e > 0) mass += post;
                const float cand = lg2_approx(post + 1e-8f) + p[e].y;
                if (cand > best) { best = cand; arg = e; }
            }
            const float anew = m + lg2_approx(esum) - a0v0.x;
            av[CUR ^ 1][s] = make_float2(anew, best - a0v0.y);
            *bp_p = (uint8_t)arg;
            bp_p += S;
            if (warp == 0) {   // (warp-uniform branch: the fp64 arithmetic below is issued by one warp only)
                if (lane == 0) {   // normaliser of step t+1: k_{t+1} = asum_{t+1} + bsum[t+2] - log2 Z, asum_{t+1} = asum_t + alpha'_t[0]
                    asum += (double)a0v0.x;
                    kt_sh[CUR ^ 1] = (float)(asum + bs_next2 - logz);
                    bs_next2 = bs_n;
                }
            }
            // move mass per emitted base (s % 4): reduce lanes of equal lane%4
            mass += __shfl_xor_sync(0xffffffffu, mass, 4);
            mass += __shfl_xor_sync(0xffffffffu, mass, 8);
            mass += __shfl_xor_sync(0xffffffffu, mass, 16);
            if (lane < 4) part[CUR][warp][lane] = mass;
            __syncthreads();
            if (s < 4) {
                float tot = 0.f;
#pragma unroll
                for (int w = 0; w < NW; ++w) tot += part[CUR][w][s];
                *pm_p = tot;
            }
            pm_p += 4;
        };
        int t = 0;
        for (; t + 1 < T; t += 2) { fwd(t, IntC<0>()); fwd(t + 1, IntC<1>()); }
        if (t < T) fwd(t, IntC<0>());
        // best final state: max Viterbi score, lowest state on ties
        float v = av[T & 1][s].y;
        int idx = s;
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, v, o);
            const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
            if (ov > v || (ov == v && oi < idx)) { v = ov; idx = oi; }
        }
        if (lane == 0) { red[warp] = v; red_i[warp] = idx; }
        __syncthreads();
    }

    // ---------------- pass 3: trace-back ----------------
    {
        uint8_t* o_mov = out_sh;
        uint8_t* o_seq = out_sh + T;
        uint8_t* o_q = out_sh + 2 * T;
        int state = 0;
        if (s == 0) {
            float v = red[0];
            state = red_i[0];
            for (int w = 1; w < NW; ++w)
                if (red[w] > v) { v = red[w]; state = red_i[w]; }
        }
        for (int hi = T; hi > 0; hi -= TB) {
            const int lo = max(hi - TB, 0), rows = hi - lo;
            __syncthreads();
            for (int i = s; i < rows * (S / 16); i += S) {
                const int row = i / (S / 16), c = i % (S / 16);
                *reinterpret_cast<uint4*>(&bp_blk[row][c * 16]) =
                    *reinterpret_cast<const uint4*>(bp + (size_t)(lo + row) * S + c * 16);
            }
            __syncthreads();
            if (s == 0) {
                for (int t = hi - 1; t >= lo; --t) {
                    const int e = bp_blk[t - lo][state];
                    const int base = state & 3;
                    if (e != 0) {
                        const float p = pm[(size_t)t * 4 + base];
                        const float err = fmaxf(1.0f - p, 1e-4f);
                        const float qv = -10.0f * log10f(err) * qscale + qbias;
                        int qi = (int)rintf(qv) + 33;
                        qi = min(max(qi, 33), 126);
                        o_mov[t] = 1;
                        o_seq[t] = (uint8_t)("ACGT"[base]);
                        o_q[t] = (uint8_t)qi;
                        state = (e - 1) * Q + (state >> 2);
                    } else {
                        o_mov[t] = 0; o_seq[t] = 0; o_q[t] = 0;
                    }
                }
            }
        }
        __syncthreads();
        for (int t = s; t < T; t += S) {
            moves[(size_t)n * T + t] = o_mov[t];
            seq[(size_t)n * T + t] = o_seq[t];
            qual[(size_t)n * T + t] = o_q[t];
        }
    }
}

inline size_t align256(size_t x) { return (x + 255) / 256 * 256; }

template <int S, bool LB = false>
int launch_decode(const __half* scores, int N, int T, float blank, float qscale, float qbias, void* workspace,
                  uint8_t* moves, uint8_t* seq, uint8_t* qual, cudaStream_t stream) {
    unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
    size_t off = 0;
    float* beta = reinterpret_cast<float*>(ws + off); off += align256((size_t)N * (T + 1) * S * sizeof(float));
    double* bsum = reinterpret_cast<double*>(ws + off); off += align256((size_t)N * (T + 1) * sizeof(double));
    float* pm = reinterpret_cast<float*>(ws + off); off += align256((size_t)N * T * 4 * sizeof(float));
    uint8_t* bp = ws + off;
    size_t dyn = DecodeSmem<S, LB>::bytes(T);
    // B200_DECODE_SMEM_KB pads the request to bound the CTAs per SM (room for a co-resident recurrent CTA)
    if (const char* pad = getenv("B200_DECODE_SMEM_KB")) {
        const size_t want = (size_t)atoi(pad) * 1024;
        if (want > dyn && want <= 200 * 1024) dyn = want;
    }
    auto kern = crf_decode_kernel<S, LB>;
    B200_REQUIRE(dyn <= 200 * 1024, "crf_decode: chunk of %d frames needs %zu B of shared memory", T, dyn);
    B200_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn));
    kern<<<N, S, dyn, stream>>>(scores, T, blank, qscale, qbias, beta, bsum, bp, pm, moves, seq, qual);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}


// ---------------------------------------------------------------------------------------------------------------------
// Beam search behind the koi.decode.beam_search call contract (bonito/crf/basecall.py:36-40).  koi's decoder is a closed
// binary with no pinned outputs, so this is THIS repository's beam search (restated for the tests by
// oracle/crf_oracle.py::beam_search_native), offered next to the exact posterior-Viterbi decoder above:
// a backward-guided prefix search over (sequence, k-mer state) entries, one WARP per chunk, one LANE per beam entry
// (beam_width <= 32).  Per frame a lane spawns a "stay" and four "move" candidates; a stay candidate and the move candidate
// that spells the same sequence are merged by log-add; the 160 candidates are ranked by forward score + beta'_{t+1}[state]
// (the backward scores the forward-backward kernel left in the workspace), cut at `beam_cut` below the best, and the best
// `beam_width` survive (ties: lower parent entry, stay before moves, lower base).  All scores in log2 units.
// Runs after crf_decode_kernel on the same workspace: it reads beta' and the posterior move mass (qualities) and reuses
// the back-pointer area (32 bytes per frame).
__device__ __forceinline__ float lse2_2(float a, float b) {
    const float hi = fmaxf(a, b), lo = fminf(a, b);
    return hi + lg2_approx(1.0f + ex2_approx(lo - hi));
}

template <int S>
__global__ void __launch_bounds__(128)
crf_beam_kernel(const __half* __restrict__ scores, int N, int T, float blank, int width, float cut, float qscale,
                float qbias, const float* __restrict__ ws_beta, uint8_t* __restrict__ ws_bp,
                const float* __restrict__ ws_pm, uint8_t* __restrict__ moves, uint8_t* __restrict__ seq,
                uint8_t* __restrict__ qual) {
    constexpr int Q = S / 4;
    constexpr unsigned long long MULT = 0x9E3779B97F4A7C15ull;
    const int lane = threadIdx.x & 31;
    const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (n >= N) return;
    const __half* sc = scores + (size_t)n * T * S * 4;
    const float* beta = ws_beta + (size_t)n * (T + 1) * S;
    uint8_t* bp = ws_bp + (size_t)n * T * S;                 // [T][32] used
    const float* pm = ws_pm + (size_t)n * T * 4;
    const float blank2 = blank * LOG2E, cut2 = cut * LOG2E;
    const unsigned FULL = 0xffffffffu;

    // ---- start beam: the `width` best start states by beta'_0 (ties: lower state) ----
    unsigned long long h = 0;
    int st = 0;
    float a = 0.f;
    bool valid = false;
    {
        constexpr int PER = S / 32;                           // states per lane: lane l owns states l*PER .. l*PER+PER-1
        float v[PER];
#pragma unroll
        for (int i = 0; i < PER; ++i) v[i] = beta[lane * PER + i];
        for (int r = 0; r < width; ++r) {
            float best = -INFINITY;
            int bi = 0;
#pragma unroll
            for (int i = 0; i < PER; ++i)
                if (v[i] > best) { best = v[i]; bi = i; }
            int bidx = lane * PER + bi;
            for (int o = 16; o > 0; o >>= 1) {
                const float ov = __shfl_xor_sync(FULL, best, o);
                const int oi = __shfl_xor_sync(FULL, bidx, o);
                if (ov > best || (ov == best && oi < bidx)) { best = ov; bidx = oi; }
            }
            if (bidx / PER == lane) {
#pragma unroll
                for (int i = 0; i < PER; ++i)
                    if (i == bidx % PER) v[i] = -INFINITY;
            }
            if (lane == r && best > -INFINITY) { h = (unsigned long long)bidx + 1ull; st = bidx; a = 0.f; valid = true; }
        }
    }

    // ---- frames ----
    for (int t = 0; t < T; ++t) {
        const __half* m = sc + (size_t)t * S * 4;
        const float* bn = beta + (size_t)(t + 1) * S;
        float csc[5], key[5];
        int cst[5], ccode[5], cpar[5];
        unsigned long long ch[5];
        const int sq = st % Q, j = st / Q;
        const float4 b4 = *reinterpret_cast<const float4*>(bn + sq * 4);
        const float bmove[4] = {b4.x, b4.y, b4.z, b4.w};
        ch[0] = h; cst[0] = st; csc[0] = a + blank2; ccode[0] = 0; cpar[0] = lane;
        key[0] = valid ? csc[0] + bn[st] : -INFINITY;
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            const int s2 = sq * 4 + b;
            ch[1 + b] = h * MULT + (unsigned long long)(b + 1);
            cst[1 + b] = s2;
            csc[1 + b] = fmaf(__half2float(m[s2 * 4 + j]), LOG2E, a);
            ccode[1 + b] = 1 + b; cpar[1 + b] = lane;
            key[1 + b] = valid ? csc[1 + b] + bmove[b] : -INFINITY;
        }
        // merge: the stay candidate of entry jj with the move candidate (of some entry) that spells the same sequence
        for (int jj = 0; jj < 32; ++jj) {
            const unsigned long long hj = __shfl_sync(FULL, h, jj);
            const bool vj = __shfl_sync(FULL, (int)valid, jj) != 0;
            if (!vj) continue;                                         // warp-uniform
            int mb = -1;
#pragma unroll
            for (int b = 0; b < 4; ++b)
                if (valid && key[1 + b] > -INFINITY && ch[1 + b] == hj && mb < 0) mb = b;
            const unsigned hit = __ballot_sync(FULL, mb >= 0);
            if (hit == 0) continue;                                    // warp-uniform
            const int src = __ffs(hit) - 1;
            float msc = 0.f;
#pragma unroll
            for (int b = 0; b < 4; ++b)
                if (b == mb) msc = csc[1 + b];
            msc = __shfl_sync(FULL, msc, src);
            const int mbase = __shfl_sync(FULL, mb, src);
            if (lane == src) {
#pragma unroll
                for (int b = 0; b < 4; ++b)
                    if (b == mb) key[1 + b] = -INFINITY;
            }
            if (lane == jj) {
                const float stay = csc[0];
                csc[0] = lse2_2(stay, msc);
                if (msc > stay) { ccode[0] = 1 + mbase; cpar[0] = src; }
                key[0] = csc[0] + bn[st];
            }
        }
        // cut
        float kbest = fmaxf(fmaxf(fmaxf(key[0], key[1]), fmaxf(key[2], key[3])), key[4]);
        for (int o = 16; o > 0; o >>= 1) kbest = fmaxf(kbest, __shfl_xor_sync(FULL, kbest, o));
#pragma unroll
        for (int c = 0; c < 5; ++c)
            if (key[c] < kbest - cut2) key[c] = -INFINITY;
        // selection: `width` rounds of (lane-local best, warp arg-max by (key desc, candidate index asc))
        unsigned long long nh = 0;
        int nst = 0, nbp = 0;
        float na = 0.f;
        bool nvalid = false;
        for (int r = 0; r < width; ++r) {
            float lk = key[0];
            int lc = 0;
#pragma unroll
            for (int c = 1; c < 5; ++c)
                if (key[c] > lk) { lk = key[c]; lc = c; }
            float wk = lk;
            int wi = lane * 5 + lc;
            for (int o = 16; o > 0; o >>= 1) {
                const float ok = __shfl_xor_sync(FULL, wk, o);
                const int oi = __shfl_xor_sync(FULL, wi, o);
                if (ok > wk || (ok == wk && oi < wi)) { wk = ok; wi = oi; }
            }
            if (!(wk > -INFINITY)) break;                              // warp-uniform: no candidate left
            const int wl = wi / 5, wc = wi % 5;
            unsigned long long xh = 0;
            int xs = 0, xb = 0;
            float xa = 0.f;
#pragma unroll
            for (int c = 0; c < 5; ++c)
                if (c == wc) { xh = ch[c]; xs = cst[c]; xa = csc[c]; xb = cpar[c] | (ccode[c] << 5); }
            xh = __shfl_sync(FULL, xh, wl);
            xs = __shfl_sync(FULL, xs, wl);
            xa = __shfl_sync(FULL, xa, wl);
            xb = __shfl_sync(FULL, xb, wl);
            if (lane == wl) {
#pragma unroll
                for (int c = 0; c < 5; ++c)
                    if (c == wc) key[c] = -INFINITY;
            }
            if (lane == r) { nh = xh; nst = xs; na = xa; nbp = xb; nvalid = true; }
        }
        // renormalise on the best surviving score
        float amax = nvalid ? na : -INFINITY;
        for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(FULL, amax, o));
        h = nh; st = nst; a = na - amax; valid = nvalid;
        bp[(size_t)t * 32 + lane] = (uint8_t)nbp;
    }

    // ---- best final entry (ties: lower lane), trace-back ----
    float fa = valid ? a : -INFINITY;
    int fi = lane;
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(FULL, fa, o);
        const int oi = __shfl_xor_sync(FULL, fi, o);
        if (ov > fa || (ov == fa && oi < fi)) { fa = ov; fi = oi; }
    }
    __syncwarp();
    if (lane == 0) {
        int r = fi;
        for (int t = T - 1; t >= 0; --t) {
            const int e = bp[(size_t)t * 32 + r];
            const int code = e >> 5;
            uint8_t mv = 0, sq_ = 0, ql = 0;
            if (code) {
                const int base = code - 1;
                const float p = pm[(size_t)t * 4 + base];
                const float err = fmaxf(1.0f - p, 1e-4f);
                int qi = (int)rintf(-10.0f * log10f(err) * qscale + qbias) + 33;
                qi = min(max(qi, 33), 126);
                mv = 1; sq_ = (uint8_t)("ACGT"[base]); ql = (uint8_t)qi;
            }
            moves[(size_t)n * T + t] = mv;
            seq[(size_t)n * T + t] = sq_;
            qual[(size_t)n * T + t] = ql;
            r = e & 31;
        }
    }
}

template <int S>
int launch_beam(const __half* scores, int N, int T, float blank, int width, float cut, float qscale, float qbias,
                void* workspace, uint8_t* moves, uint8_t* seq, uint8_t* qual, cudaStream_t stream) {
    unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
    size_t off = 0;
    float* beta = reinterpret_cast<float*>(ws + off); off += align256((size_t)N * (T + 1) * S * sizeof(float));
    off += align256((size_t)N * (T + 1) * sizeof(double));
    float* pm = reinterpret_cast<float*>(ws + off); off += align256((size_t)N * T * 4 * sizeof(float));
    uint8_t* bp = ws + off;
    crf_beam_kernel<S><<<(N + 3) / 4, 128, 0, stream>>>(scores, N, T, blank, width, cut, qscale, qbias, beta, bp, pm, moves, seq, qual);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace

size_t crf_decode_workspace_bytes(int N, int T, int state_len) {
    size_t S = 1;
    for (int i = 0; i < state_len; ++i) S *= 4;
    return align256((size_t)N * (T + 1) * S * sizeof(float)) + align256((size_t)N * (T + 1) * sizeof(double)) +
           align256((size_t)N * T * 4 * sizeof(float)) + align256((size_t)N * T * S);
}

int launch_crf_decode(const __half* scores, int N, int T, int state_len, float blank, float qscale, float qbias,
                      void* workspace, uint8_t* moves, uint8_t* seq, uint8_t* qual, cudaStream_t stream) {
    if (N == 0 || T == 0) return 0;
    switch (state_len) {
        case 3: return launch_decode<64>(scores, N, T, blank, qscale, qbias, workspace, moves, seq, qual, stream);
        case 4: return launch_decode<256>(scores, N, T, blank, qscale, qbias, workspace, moves, seq, qual, stream);
        case 5: return launch_decode<1024>(scores, N, T, blank, qscale, qbias, workspace, moves, seq, qual, stream);
        default:
            b200_set_error("crf_decode: state_len %d is not supported (3, 4, 5)", state_len);
            return -2;
    }
}

int launch_crf_decode_lb(const __half* scores, int N, int T, int state_len, float qscale, float qbias, void* workspace,
                         uint8_t* moves, uint8_t* seq, uint8_t* qual, cudaStream_t stream) {
    if (N == 0 || T == 0) return 0;
    switch (state_len) {
        case 3: return launch_decode<64, true>(scores, N, T, 0.f, qscale, qbias, workspace, moves, seq, qual, stream);
        case 4: return launch_decode<256, true>(scores, N, T, 0.f, qscale, qbias, workspace, moves, seq, qual, stream);
        case 5: return launch_decode<1024, true>(scores, N, T, 0.f, qscale, qbias, workspace, moves, seq, qual, stream);
        default:
            b200_set_error("crf_decode_lb: state_len %d is not supported (3, 4, 5)", state_len);
            return -2;
    }
}

// exact forward-backward first (it fills beta' and the move mass), then the beam search over the same workspace
int launch_crf_beam_search(const __half* scores, int N, int T, int state_len, float blank, int width, float cut, float qscale,
                           float qbias, void* workspace, uint8_t* moves, uint8_t* seq, uint8_t* qual, cudaStream_t stream) {
    if (N == 0 || T == 0) return 0;
    B200_REQUIRE(width >= 1 && width <= 32, "beam_search: beam_width %d is not supported (1..32: one lane per beam entry)", width);
    int rc = launch_crf_decode(scores, N, T, state_len, blank, qscale, qbias, workspace, moves, seq, qual, stream);
    if (rc) return rc;
    switch (state_len) {
        case 3: return launch_beam<64>(scores, N, T, blank, width, cut, qscale, qbias, workspace, moves, seq, qual, stream);
        case 4: return launch_beam<256>(scores, N, T, blank, width, cut, qscale, qbias, workspace, moves, seq, qual, stream);
        case 5: return launch_beam<1024>(scores, N, T, blank, width, cut, qscale, qbias, workspace, moves, seq, qual, stream);
        default: return -2;
    }
}
