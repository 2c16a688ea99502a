// Batched Smith-Waterman local alignment with affine gaps (Gotoh), for `python -m bonito_b200 evaluate`.
//
// Definition (the CPU oracle, tests/_oracle_align.py, implements the same rules with full matrices and a traceback):
//   query q (the basecall, m bases, rows i) against reference r (n bases, columns j), ASCII A/C/G/T;
//   s(a, b) = +5 if a == b else -4 (parasail's dnafull on ACGT); gap open 8, extend 4 (a gap of k costs 8 + 4 (k - 1));
//   E[i][j] = max(H[i][j-1] - 8, E[i][j-1] - 4)      op D, consumes a reference base
//   F[i][j] = max(H[i-1][j] - 8, F[i-1][j] - 4)      op I, consumes a query base
//   H[i][j] = max(0, H[i-1][j-1] + s(q_i, r_j), E[i][j], F[i][j])
//   with H = 0 and E = F = -2^29 on row and column 0.
// Ties: in E / F the open wins over the extend; in H a 0 wins every tie (the cell starts a new alignment), then the
// diagonal, then E, then F.  The end cell is the maximum H, ties to the smallest end_query, then the smallest end_ref (the
// first occurrence in query-major order); both ends are 0-based and inclusive.  A best score of 0 (an empty side, no
// common letter) reports score 0, ends -1 and zero counts.
//
// parasail's own tie rules are not pinned by anything here, so these rules are this library's definition.  Among
// co-optimal alignments the counts almost never differ: a gap shifted within a homopolymer keeps every count.
//
// Counts without a traceback: each cell's predecessor depends only on values at that cell, so the op counts of the traced
// path are carried forward along the chosen predecessor, per state (H, E, F), as two words: (=, X) and (I, D) in 16-bit
// halves.  Lengths are capped at 65535, so no half can overflow.  Under these rules a path never starts with a gap (a
// state E / F cell is only chosen by H when it is positive, and its opening H cell is then > 8).
//
// Shape: one warp per pair (pairs grid-strided over the warps).  Each lane owns AL_R consecutive query rows of a
// 32 * AL_R-row strip, and reference columns stream through in a wavefront: at step s lane l computes column s - l.  H, F
// and their counts of a lane's bottom row cross to the next lane by __shfl_up_sync; E, the left H and their counts stay
// in registers per row.  Lane 31 stores the strip's bottom row into a per-warp workspace row, which lane 0 of the next
// strip reads column by column (in place: lane 0 reads column s while lane 31 writes column s - 31).  The max / select
// steps use the sm_90 DPX instructions (__vibmax_s32 gives the max and the open-wins-tie predicate in one; H is one
// __vimax3_s32_relu).  The end cell is a 64-bit key (score, 65535 - i, 65535 - j) reduced by max over the warp, so the
// result is deterministic and does not depend on the other pairs of the launch.
#include "common.cuh"

namespace {

constexpr int AL_R = 8;                    // query rows per lane
constexpr int AL_STRIP = 32 * AL_R;        // query rows per strip
constexpr int AL_THREADS = 256;            // 8 warps per CTA
constexpr int AL_MAX_WARPS = 2048;         // workspace rows (the grid never has more warps)
constexpr int AL_NEG = -(1 << 29);
constexpr int AL_MAX_LEN = 65535;
constexpr unsigned FULL = 0xffffffffu;

struct AlignMeta {                          // the per-pair arrays, copied into the head of the workspace
    const long long* qoff;
    const long long* roff;
    const int* qlen;
    const int* rlen;
};

size_t meta_bytes(int n_pairs) { return (((size_t)n_pairs * 24) + 255) & ~(size_t)255; }

__global__ void __launch_bounds__(AL_THREADS)
sw_align_kernel(const uint8_t* __restrict__ query, const uint8_t* __restrict__ ref, AlignMeta meta, int n_pairs,
                int pitch, int4* __restrict__ ws, int* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int warp = (int)((blockIdx.x * (unsigned)AL_THREADS + threadIdx.x) >> 5);
    const int nwarps = (int)(gridDim.x * (AL_THREADS / 32));
    int4* row = ws + (size_t)warp * pitch * 2;        // per column: {H, F, H(=,X), H(I,D)}, {F(=,X), F(I,D), -, -}
    for (int p = warp; p < n_pairs; p += nwarps) {
        const int m = meta.qlen[p], n = meta.rlen[p];
        const uint8_t* qp = query + meta.qoff[p];
        const uint8_t* rp = ref + meta.roff[p];
        unsigned long long best = 0;
        uint32_t best1 = 0, best2 = 0;
        for (int base = 0; base < m; base += AL_STRIP) {
            const int i0 = base + lane * AL_R;        // 0-based query index of this lane's first row
            const bool first = base == 0, more = base + AL_STRIP < m;
            uint32_t qc[AL_R];
            int hl[AL_R], el[AL_R];                   // H[i][j-1], E[i][j-1]
            uint32_t h1[AL_R], h2[AL_R], e1[AL_R], e2[AL_R];
#pragma unroll
            for (int k = 0; k < AL_R; ++k) {
                qc[k] = i0 + k < m ? qp[i0 + k] : 0xffu;      // rows past the query never match and are never reported
                hl[k] = 0;
                el[k] = AL_NEG;
                h1[k] = h2[k] = e1[k] = e2[k] = 0u;
            }
            int dh = 0;                               // H[i0-1][j-1] and its counts: the top row's diagonal
            uint32_t d1 = 0u, d2 = 0u;
            int oh = 0, of = AL_NEG;                  // the bottom row's H / F at the last column computed
            uint32_t oh1 = 0u, oh2 = 0u, of1 = 0u, of2 = 0u;
            for (int s = 0; s < n + 31; ++s) {
                int uh = __shfl_up_sync(FULL, oh, 1), uf = __shfl_up_sync(FULL, of, 1);
                uint32_t uh1 = __shfl_up_sync(FULL, oh1, 1), uh2 = __shfl_up_sync(FULL, oh2, 1);
                uint32_t uf1 = __shfl_up_sync(FULL, of1, 1), uf2 = __shfl_up_sync(FULL, of2, 1);
                const int j = s - lane;
                if (j < 0 || j >= n) continue;
                if (lane == 0) {
                    if (first) {
                        uh = 0, uf = AL_NEG, uh1 = uh2 = uf1 = uf2 = 0u;
                    } else {
                        const int4 a = row[2 * j], b = row[2 * j + 1];
                        uh = a.x, uf = a.y, uh1 = (uint32_t)a.z, uh2 = (uint32_t)a.w, uf1 = (uint32_t)b.x, uf2 = (uint32_t)b.y;
                    }
                }
                const uint32_t rc = rp[j];
                int di = dh;
                uint32_t di1 = d1, di2 = d2;
                dh = uh, d1 = uh1, d2 = uh2;
#pragma unroll
                for (int k = 0; k < AL_R; ++k) {
                    bool open;
                    const int e = __vibmax_s32(hl[k] - 8, el[k] - 4, &open);
                    const uint32_t ne1 = open ? h1[k] : e1[k];
                    const uint32_t ne2 = (open ? h2[k] : e2[k]) + 0x10000u;        // + D
                    const int f = __vibmax_s32(uh - 8, uf - 4, &open);
                    const uint32_t nf1 = open ? uh1 : uf1;
                    const uint32_t nf2 = (open ? uh2 : uf2) + 1u;                  // + I
                    const bool match = qc[k] == rc;
                    const int d = di + (match ? 5 : -4);
                    const int h = __vimax3_s32_relu(d, e, f);
                    uint32_t nh1, nh2;
                    if (h == 0) {
                        nh1 = nh2 = 0u;
                    } else if (h == d) {
                        nh1 = di1 + (match ? 1u : 0x10000u);
                        nh2 = di2;
                    } else if (h == e) {
                        nh1 = ne1, nh2 = ne2;
                    } else {
                        nh1 = nf1, nh2 = nf2;
                    }
                    di = hl[k], di1 = h1[k], di2 = h2[k];     // the next row's diagonal is this row's left cell
                    hl[k] = h, h1[k] = nh1, h2[k] = nh2;
                    el[k] = e, e1[k] = ne1, e2[k] = ne2;
                    uh = h, uh1 = nh1, uh2 = nh2;
                    uf = f, uf1 = nf1, uf2 = nf2;
                    if (h > 0 && i0 + k < m) {
                        const unsigned long long key = ((unsigned long long)(uint32_t)h << 32) |
                                                       ((unsigned long long)(AL_MAX_LEN - (i0 + k)) << 16) |
                                                       (unsigned long long)(AL_MAX_LEN - j);
                        if (key > best) best = key, best1 = nh1, best2 = nh2;
                    }
                }
                oh = uh, of = uf, oh1 = uh1, oh2 = uh2, of1 = uf1, of2 = uf2;
                if (lane == 31 && more) {
                    row[2 * j] = make_int4(oh, of, (int)oh1, (int)oh2);
                    row[2 * j + 1] = make_int4((int)of1, (int)of2, 0, 0);
                }
            }
            __syncwarp();                             // lane 31's row is complete before lane 0 of the next strip reads it
        }
        unsigned long long top = best;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const unsigned long long o = __shfl_xor_sync(FULL, top, off);
            top = o > top ? o : top;
        }
        const unsigned owner = __ballot_sync(FULL, best == top);
        const int src = __ffs(owner) - 1;             // keys are unique per cell: one owner (all lanes when top == 0)
        const uint32_t c1 = __shfl_sync(FULL, best1, src), c2 = __shfl_sync(FULL, best2, src);
        if (lane == 0) {
            int* o = out + (size_t)p * 7;
            if (top == 0) {
                o[0] = 0, o[1] = -1, o[2] = -1, o[3] = o[4] = o[5] = o[6] = 0;
            } else {
                o[0] = (int)(top >> 32);
                o[1] = AL_MAX_LEN - (int)((top >> 16) & 0xffffu);
                o[2] = AL_MAX_LEN - (int)(top & 0xffffu);
                o[3] = (int)(c1 & 0xffffu), o[4] = (int)(c1 >> 16), o[5] = (int)(c2 & 0xffffu), o[6] = (int)(c2 >> 16);
            }
        }
    }
}

int align_warps(int n_pairs) { return n_pairs < AL_MAX_WARPS ? n_pairs : AL_MAX_WARPS; }

}  // namespace

size_t sw_align_workspace_bytes(int n_pairs, int max_ref_len) {
    if (n_pairs <= 0) return 0;
    const size_t pitch = max_ref_len > 0 ? (size_t)max_ref_len : 1;
    return meta_bytes(n_pairs) + (size_t)align_warps(n_pairs) * pitch * 2 * sizeof(int4);
}

int launch_sw_align(const uint8_t* query, const long long* query_off, const int* query_len, const uint8_t* ref,
                    const long long* ref_off, const int* ref_len, int n_pairs, void* workspace, int* out,
                    cudaStream_t stream) {
    B200_REQUIRE(n_pairs >= 0, "sw_align: bad pair count %d", n_pairs);
    if (n_pairs == 0) return 0;
    B200_REQUIRE(query && query_off && query_len && ref && ref_off && ref_len && workspace && out,
                 "sw_align: null pointer argument");
    int max_ref = 1;
    for (int p = 0; p < n_pairs; ++p) {
        B200_REQUIRE(query_len[p] >= 0 && query_len[p] <= AL_MAX_LEN && ref_len[p] >= 0 && ref_len[p] <= AL_MAX_LEN,
                     "sw_align: pair %d has lengths %d / %d; each side must be in [0, %d]", p, query_len[p], ref_len[p],
                     AL_MAX_LEN);
        B200_REQUIRE(query_off[p] >= 0 && ref_off[p] >= 0, "sw_align: pair %d has a negative offset", p);
        max_ref = ref_len[p] > max_ref ? ref_len[p] : max_ref;
    }
    // the per-pair arrays go into the head of the workspace: [qoff | roff] int64, [qlen | rlen] int32
    char* head = static_cast<char*>(workspace);
    long long* qoff = reinterpret_cast<long long*>(head);
    long long* roff = qoff + n_pairs;
    int* qlen = reinterpret_cast<int*>(roff + n_pairs);
    int* rlen = qlen + n_pairs;
    B200_CHECK_CUDA(cudaMemcpyAsync(qoff, query_off, sizeof(long long) * n_pairs, cudaMemcpyHostToDevice, stream));
    B200_CHECK_CUDA(cudaMemcpyAsync(roff, ref_off, sizeof(long long) * n_pairs, cudaMemcpyHostToDevice, stream));
    B200_CHECK_CUDA(cudaMemcpyAsync(qlen, query_len, sizeof(int) * n_pairs, cudaMemcpyHostToDevice, stream));
    B200_CHECK_CUDA(cudaMemcpyAsync(rlen, ref_len, sizeof(int) * n_pairs, cudaMemcpyHostToDevice, stream));
    int4* rows = reinterpret_cast<int4*>(head + meta_bytes(n_pairs));
    const int warps = align_warps(n_pairs);
    const unsigned grid = (unsigned)((warps + AL_THREADS / 32 - 1) / (AL_THREADS / 32));
    sw_align_kernel<<<grid, AL_THREADS, 0, stream>>>(query, ref, AlignMeta{qoff, roff, qlen, rlen}, n_pairs, max_ref, rows,
                                                      out);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}
