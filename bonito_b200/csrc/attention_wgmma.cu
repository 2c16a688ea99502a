// Windowed softmax attention of the transformer (sup) models on the Hopper tensor cores (wgmma, sm_90a).
// qkv [N][T][3][NH][64] fp16 (rotary already applied to q and k in place, rotary_kernel) -> out [N][T][NH*64]; key j is
// visible to query i iff i - wl <= j <= i + wr; softmax scale 1/sqrt(64).  Reference: flash_attn_qkvpacked_func with
// window_size = (wl, wr) as called by bonito/transformer/model.py:71-78.
//
//   * one CTA = 128 queries of one (chunk, head): two warpgroups of 64 query rows each; the keys the two windows need are
//     streamed as 64-key blocks of K and V through a double-buffered cp.async ring that both warpgroups share, so each
//     key block is fetched once per 128 queries;
//   * S = Q K^T is wgmma m64n64k16 x 4 with both operands in shared memory (K-major, no swizzle: [8-dim chunk][row][16 B]);
//   * the online softmax runs on the S fragment in registers (thread = rows lane/4, lane/4 + 8 of its warp's 16 rows),
//     P is packed to fp16 in place as the register A operand of O += P V (wgmma m64n64k16 x 4, A from registers);
//     V keeps the same shared-memory layout as K and is read as an MN-major (transposed) B operand: a core matrix is
//     8 keys x 8 dims = 128 contiguous bytes of that layout, so no transpose is ever materialised;
//   * a warpgroup skips the key blocks that lie wholly outside its own 64 queries' windows.
// Arithmetic as in the mma.sync kernel of transformer.cu (kept as the cross-check): fp32 scores and output accumulation,
// exponentials on ex2 with the scale folded in, P rounded to fp16 before the PV product.
#include "tc_common.cuh"

namespace {

constexpr int HD = 64, BQ = 128, BK = 64, THREADS = 256;
constexpr uint32_t Q_BYTES = BQ * HD * 2;            // 16 KB: [8 dim chunks][128 queries][16 B]
constexpr uint32_t KV_BYTES = BK * HD * 2;           // 8 KB:  [8 dim chunks][64 keys][16 B]
constexpr uint32_t OFF_Q = 0, OFF_K = Q_BYTES, OFF_V = OFF_K + 2 * KV_BYTES;
constexpr uint32_t SMEM_BYTES = OFF_V + 2 * KV_BYTES;   // 48 KB

// rows [t0, t0 + rows) of q / k / v (which = 0 / 1 / 2) of one (chunk, head) -> [dim chunk][row][16 B]; rows outside
// [0, T) are zero-filled
template <int ROWS>
__device__ __forceinline__ void load_rows(unsigned char* dst, const __half* __restrict__ qkv, int n, int T, int NH, int head,
                                          int which, int t0, int tid) {
    // a warp fills 8 consecutive rows x 4 dim chunks: 4 x 128 contiguous bytes of shared memory (no bank conflicts) from
    // 8 x 64 contiguous bytes of global memory
#pragma unroll
    for (int i = 0; i < ROWS * 8 / THREADS; ++i) {
        const int c = tid + i * THREADS, rest = c >> 5;
        const int row = (c & 7) + 8 * (rest >> 1), dc = ((c >> 3) & 3) + 4 * (rest & 1), t = t0 + row;
        const bool ok = t >= 0 && t < T;
        const __half* src = ok ? qkv + ((((size_t)n * T + t) * 3 + which) * NH + head) * HD + dc * 8 : qkv;
        cp_async_16(dst + (uint32_t)dc * (ROWS * 16) + (uint32_t)row * 16, src, ok);
    }
}

__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}

__global__ void __launch_bounds__(THREADS, 1)
attention_wgmma_kernel(const __half* __restrict__ qkv, __half* __restrict__ out, int T, int NH, int wl, int wr,
                       float scale_log2e) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const uint32_t base = smem_u32(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wg = warp >> 2, wq = warp & 3;
    const int g = lane >> 2, qd = lane & 3;
    const int q0 = blockIdx.x * BQ, head = blockIdx.y, n = blockIdx.z;
    const int qw0 = q0 + wg * 64;                                  // first query of this warpgroup
    const int qrow[2] = {qw0 + wq * 16 + g, qw0 + wq * 16 + g + 8};

    int k_lo = q0 - wl; if (k_lo < 0) k_lo = 0;
    int k_hi = q0 + BQ - 1 + wr + 1; if (k_hi > T) k_hi = T;
    const int kb0 = (k_lo / BK) * BK;
    // key range of this warpgroup's windows
    const int w_lo = qw0 - wl, w_hi = qw0 + 63 + wr;

    load_rows<BQ>(smem_raw + OFF_Q, qkv, n, T, NH, head, 0, q0, tid);
    if (kb0 < k_hi) {
        load_rows<BK>(smem_raw + OFF_K, qkv, n, T, NH, head, 1, kb0, tid);
        load_rows<BK>(smem_raw + OFF_V, qkv, n, T, NH, head, 2, kb0, tid);
    }
    cp_async_commit();

    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    const uint32_t qa = base + OFF_Q + (uint32_t)wg * (64 * 16);
    int buf = 0;
    for (int kb = kb0; kb < k_hi; kb += BK, buf ^= 1) {
        if (kb + BK < k_hi) {   // the other buffer was released by the barrier that ended the previous iteration
            load_rows<BK>(smem_raw + OFF_K + (buf ^ 1) * KV_BYTES, qkv, n, T, NH, head, 1, kb + BK, tid);
            load_rows<BK>(smem_raw + OFF_V + (buf ^ 1) * KV_BYTES, qkv, n, T, NH, head, 2, kb + BK, tid);
        }
        cp_async_commit();
        cp_async_wait<1>();          // everything but the group just committed: Q and this block's K / V have landed
        fence_proxy_async_smem();    // cp.async writes -> visible to wgmma
        __syncthreads();
        if (kb + BK - 1 >= w_lo && kb <= w_hi) {   // warpgroup-uniform: the block meets this warpgroup's windows
            const uint32_t ka = base + OFF_K + (uint32_t)buf * KV_BYTES, va = base + OFF_V + (uint32_t)buf * KV_BYTES;
            // S = Q K^T: A = Q [64 x 64 dims], B = K [64 keys x 64 dims], both K-major; one k16 step = two dim chunks
            float s[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) s[i] = 0.f;
            wg_fence_regs(s);
            wg_fence();
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
                wgmma_m64n64k16_f16(s, wg_desc_noswz(qa + (uint32_t)kk * 2 * (BQ * 16), BQ * 16, 128),
                                    wg_desc_noswz(ka + (uint32_t)kk * 2 * (BK * 16), BK * 16, 128), 1);
            wg_commit();
            wg_wait<0>();
            wg_fence_regs(s);
            // mask + online softmax (rows g and g+8; a row is shared by the 4 lanes of a quad)
            float m_new[2] = {m_run[0], m_run[1]};
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int r = e >> 1, key = kb + j * 8 + 2 * qd + (e & 1), q = qrow[r];
                    const bool ok = key < T && q < T && key >= q - wl && key <= q + wr;
                    s[j * 4 + e] = ok ? s[j * 4 + e] : -INFINITY;
                    m_new[r] = fmaxf(m_new[r], s[j * 4 + e]);
                }
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                m_new[r] = fmaxf(m_new[r], __shfl_xor_sync(0xffffffffu, m_new[r], 1));
                m_new[r] = fmaxf(m_new[r], __shfl_xor_sync(0xffffffffu, m_new[r], 2));
            }
            float corr[2], msafe[2];
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                msafe[r] = (m_new[r] == -INFINITY) ? 0.f : m_new[r];
                corr[r] = ex2_approx((m_run[r] - msafe[r]) * scale_log2e);   // ex2(-inf) = 0 for the first block
                m_run[r] = m_new[r];
                l_run[r] *= corr[r];
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                o[j * 4 + 0] *= corr[0]; o[j * 4 + 1] *= corr[0]; o[j * 4 + 2] *= corr[1]; o[j * 4 + 3] *= corr[1];
            }
            uint32_t pf[4][4];   // P as A fragments: k-step kk covers keys 16kk .. 16kk+15 = score blocks 2kk, 2kk+1
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float p[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    p[e] = ex2_approx((s[j * 4 + e] - msafe[e >> 1]) * scale_log2e);
                    l_run[e >> 1] += p[e];
                }
                pf[j >> 1][(j & 1) * 2 + 0] = pack_h2(p[0], p[1]);
                pf[j >> 1][(j & 1) * 2 + 1] = pack_h2(p[2], p[3]);
            }
            // O += P V: B = V [64 keys (K) x 64 dims (N)], MN-major: 8-key groups 128 B apart, 8-dim chunks BK*16 apart
            wg_fence_regs(o);
            wg_fence();
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
                wgmma_m64n64k16_f16_rs_tb(o, pf[kk], wg_desc_noswz(va + (uint32_t)kk * 16 * 16, 128, BK * 16));
            wg_commit();
            wg_wait<0>();
            wg_fence_regs(o);
        }
        __syncthreads();   // this buffer is refilled by the loads issued at the top of the next iteration
    }
    cp_async_wait<0>();
    // normalise and store
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
        l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int q = qrow[r];
        if (q >= T) continue;
        const float inv = 1.0f / l_run[r];
        __half* dst = out + ((size_t)n * T + q) * NH * HD + head * HD;
#pragma unroll
        for (int j = 0; j < 8; ++j)
            *reinterpret_cast<__half2*>(dst + j * 8 + 2 * qd) = __floats2half2_rn(o[j * 4 + 2 * r] * inv, o[j * 4 + 2 * r + 1] * inv);
    }
}

}  // namespace

// qkv [N][T][3][NH][64] (rotary already applied to q, k) -> out [N][T][NH*64]; wl / wr < 0: unlimited
int launch_attention_wgmma(const __half* qkv, __half* out, int N, int T, int NH, int wl, int wr, cudaStream_t stream) {
    static bool configured = false;
    if (!configured) {
        B200_CHECK_CUDA(cudaFuncSetAttribute(attention_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
        configured = true;
    }
    if (wl < 0) wl = T;
    if (wr < 0) wr = T;
    dim3 grid((T + BQ - 1) / BQ, NH, N);
    const float scale_log2e = 1.4426950408889634f / sqrtf((float)HD);
    attention_wgmma_kernel<<<grid, THREADS, SMEM_BYTES, stream>>>(qkv, out, T, NH, wl, wr, scale_log2e);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}
