// Batched pairwise alignment with a stored traceback, for `python -m bonito_b200 duplex`.
//
// Query q (m bases, rows i, 1-based) against target r (n bases, columns j, 1-based), any bytes (equal bytes match).  The op
// string has one byte per op in forward order: '=' / 'X' consume one base of each, 'I' consumes a query base and 'D' a
// target base (SAM).  Two modes, this library's definitions (the CPU oracle, tests/_oracle_duplex.py, implements the same
// rules with full matrices):
//
// GLOBAL_EDIT (unit-cost global alignment):
//   D[i][j] = min(D[i-1][j-1] + [q_i != r_j], D[i-1][j] + 1 (I), D[i][j-1] + 1 (D)),  D[i][0] = i, D[0][j] = j,
//   traced back from (m, n); ties go to the diagonal, then I, then D.
//   Banded: only the diagonals j - i in [lo, hi] = [min(0, n-m) - k, max(0, n-m) + k] are computed, every other cell is
//   +inf.  The band always holds the diagonals 0 and n - m, so D[m][n] is finite.  A path that leaves the band crosses at
//   least k + 1 diagonals away from [min(0, n-m), max(0, n-m)] and back, so it costs more than k: when the banded D[m][n]
//   is <= k it is the unbanded distance, every cell on an optimal path holds its true value, and every predecessor the tie
//   rule can pick lies in the band with its true value -- the banded traceback is the unbanded one.  The caller checks the
//   bound and re-runs a failing pair with a wider band (bonito_b200/align.py doubles k); k >= max(m, n) covers the matrix.
//   Traceback: 2 bits per band cell (the op itself: 0 '=', 1 'X', 2 'I', 3 'D'), rows of ceil(W / 16) words, W = hi-lo+1,
//   cell (i, j) at band offset j - i - lo of row i.
//
// SEMIGLOBAL_AFFINE (free end gaps; match +5, mismatch -4, a gap of g costs 10 + 2 (g - 1)):
//   E[i][j] = max(H[i][j-1] - 10, E[i][j-1] - 2)      op D
//   F[i][j] = max(H[i-1][j] - 10, F[i-1][j] - 2)      op I
//   H[i][j] = max(H[i-1][j-1] + s(q_i, r_j), E[i][j], F[i][j]),   H = 0 and E = F = -inf on row and column 0.
//   In E / F the open wins a tie over the extend; in H the diagonal wins, then E, then F.  The end cell is the maximum H
//   over row m and column n (H[m][0] and H[0][n] included), ties to the largest i, then the largest j.  The op string
//   covers both sequences: the free trailing gap after the end cell and the free leading gap before the path reaches row
//   or column 0 are emitted as runs of D (target left over) or I (query left over).  Full matrix, no band.
//   Traceback: 4 bits per cell (bits 0-1 the H source: 0 '=', 1 'X', 2 F, 3 E; bit 2 E opened; bit 3 F opened), rows of
//   ceil(n / 8) words.
//
// Forward shape (the skeleton of align.cu): one warp per pair (pairs grid-strided over one-warp CTAs, so a small batch
// still spreads over the SMs).  Each lane owns PA_R consecutive rows of a 32 * PA_R-row strip; columns stream through as a
// wavefront (at step s lane l computes column first + s - l), the bottom row of a lane crosses to the next by
// __shfl_up_sync, the strip's bottom row goes through a per-warp workspace row to the next strip.  Each lane packs the
// traceback codes of a row into a register word and stores it once it is full (one 4-byte store per 16 / 8 cells).
//
// The traceback walk is sequential per pair, so it must not pay a global-memory latency per cell.  The warp copies a tile
// of the traceback (32 rows x 8 words: 128 band cells / 64 columns per row, positioned so the walk can only leave it
// through the top row or the left edge) into shared memory with 256 independent loads, then lane 0 walks inside the tile
// at shared-memory latency; a tile covers up to 32 rows of the path, so a pair of m rows costs about m / 32 tile loads,
// each one round trip.  Ops are written backwards from the end of the pair's slot (stores do not stall the walk); the
// gap runs at the matrix border are written by all lanes.
//
// Results depend only on the pair: no value crosses pairs, and the workspace rows are rewritten before they are read.
#include <limits.h>

#include <vector>

#include "common.cuh"

namespace {

constexpr int PA_R = 8;                     // rows per lane
constexpr int PA_STRIP = 32 * PA_R;         // rows per strip
constexpr int PA_MAX_WARPS = 1024;          // workspace rows (the grid never has more warps)
constexpr int PA_MAX_LEN = 1 << 28;         // keeps m + n and every band offset far inside int32
constexpr int PA_INF = 0x3fffffff;
constexpr int PA_NEG = -(1 << 30);
constexpr int PA_TILE_ROWS = 32;
constexpr int PA_TILE_WORDS = 8;
constexpr unsigned FULL = 0xffffffffu;
constexpr uint32_t OP_CHARS = 0x4449583Du;  // bytes '=', 'X', 'I', 'D' by code 0..3

struct PairMeta {                            // the per-pair arrays, copied into the head of the workspace
    const long long* qoff;
    const long long* roff;
    const long long* ooff;                  // op slot of the pair (m + n bytes)
    const long long* toff;                  // traceback bytes of the pair, from the start of the traceback region
    const int* qlen;
    const int* rlen;
    const int* band;
};

size_t meta_bytes(int n_pairs) { return (((size_t)n_pairs * (4 * 8 + 3 * 4)) + 255) & ~(size_t)255; }

__device__ __forceinline__ uint8_t op_char(uint32_t code) { return (uint8_t)(OP_CHARS >> (8 * code)); }

// D[r][c] of the row above a strip: the border, the previous strip's bottom row, or +inf outside the band
__device__ __forceinline__ int edit_top(const int2* row, int r, int c, int lo, int hi) {
    const int d = c - r;
    if (d < lo || d > hi) return PA_INF;
    if (r == 0) return c;
    if (c == 0) return r;
    return row[c].x;
}

// all lanes write `count` copies of `op` just below op_end[-cnt]
__device__ __forceinline__ void gap_run(uint8_t* op_end, int cnt, int count, uint8_t op, int lane) {
    for (int t = lane; t < count; t += 32) op_end[-1 - cnt - t] = op;
}

template <bool TB>
__global__ void __launch_bounds__(32)
edit_kernel(const uint8_t* __restrict__ query, const uint8_t* __restrict__ ref, PairMeta meta, int n_pairs, int pitch,
            int2* __restrict__ ws, char* __restrict__ trace, uint8_t* __restrict__ ops, int* __restrict__ out) {
    __shared__ uint32_t tile[PA_TILE_ROWS * PA_TILE_WORDS];
    const int lane = threadIdx.x;
    int2* row = ws + (size_t)blockIdx.x * pitch;
    for (int p = blockIdx.x; p < n_pairs; p += gridDim.x) {
        const int m = meta.qlen[p], n = meta.rlen[p], k = meta.band[p];
        const uint8_t* qp = query + meta.qoff[p];
        const uint8_t* rp = ref + meta.roff[p];
        const int lo = min(0, n - m) - k, hi = max(0, n - m) + k;
        const int wpr = (hi - lo + 1 + 15) >> 4;
        uint32_t* tb = reinterpret_cast<uint32_t*>(trace + (TB ? meta.toff[p] : 0));
        if (m == 0 || n == 0) {
            if (lane == 0) out[2 * p] = m + n;
        } else {
            for (int base = 0; base < m; base += PA_STRIP) {
                const int i0 = base + lane * PA_R + 1;     // this lane's first row
                const bool more = base + PA_STRIP < m;
                const int cb = max(1, base + 1 + lo), ce = min(n, base + PA_STRIP + hi);   // the strip's columns
                uint32_t qc[PA_R], acc[PA_R];
                int left[PA_R];                            // D[i][c-1]
#pragma unroll
                for (int kk = 0; kk < PA_R; ++kk) {
                    const int i = i0 + kk;
                    qc[kk] = i <= m ? qp[i - 1] : 0x100u;  // rows past the query are never stored
                    left[kk] = (cb == 1 && i <= -lo) ? i : PA_INF;   // column cb - 1 is the border or outside the band
                    acc[kk] = 0u;
                }
                // D[i0-1][cb-1], the top row's diagonal at the first column
                int dh = lane == 0 ? edit_top(row, base, cb - 1, lo, hi) : ((cb == 1 && i0 - 1 <= -lo) ? i0 - 1 : PA_INF);
                int oh = PA_INF;
                for (int s = 0; s < ce - cb + 32; ++s) {
                    int uh = __shfl_up_sync(FULL, oh, 1);
                    const int c = cb + s - lane;
                    if (c < cb || c > ce) continue;
                    if (lane == 0) uh = edit_top(row, base, c, lo, hi);
                    const uint32_t rc = rp[c - 1];
                    int di = dh;
                    dh = uh;
#pragma unroll
                    for (int kk = 0; kk < PA_R; ++kk) {
                        const int i = i0 + kk, b = c - i - lo;
                        const bool inb = i <= m && b >= 0 && c - i <= hi;
                        const bool x = qc[kk] != rc;
                        int v = di + (int)x;
                        uint32_t op = x ? 1u : 0u;
                        if (uh + 1 < v) v = uh + 1, op = 2u;
                        if (left[kk] + 1 < v) v = left[kk] + 1, op = 3u;
                        if (!inb) v = PA_INF;
                        di = left[kk];
                        left[kk] = v;
                        uh = v;
                        if (TB && inb) {
                            acc[kk] |= op << (2 * (b & 15));
                            if ((b & 15) == 15 || c == min(n, i + hi)) {
                                tb[(size_t)(i - 1) * wpr + (b >> 4)] = acc[kk];
                                acc[kk] = 0u;
                            }
                        }
                        if (i == m && c == n) out[2 * p] = v;
                    }
                    oh = uh;
                    if (lane == 31 && more) row[c].x = oh;
                }
                __syncwarp();                              // the strip's rows (and bits) are complete before they are read
            }
        }
        if (!TB) continue;
        // ---- traceback walk from (m, n)
        uint8_t* op_end = ops + meta.ooff[p] + m + n;
        int i = m, j = n, cnt = 0;
        while (i > 0 && j > 0) {
            const int b = j - i - lo;
            const int w0 = max(0, min((b >> 4) - 5, wpr - PA_TILE_WORDS));    // room for 80 D moves and 32 I moves
            const int r0 = i - (PA_TILE_ROWS - 1);
            for (int t = lane; t < PA_TILE_ROWS * PA_TILE_WORDS; t += 32) {
                const int rr = r0 + t / PA_TILE_WORDS, ww = w0 + t % PA_TILE_WORDS;
                tile[t] = (rr >= 1 && ww < wpr) ? tb[(size_t)(rr - 1) * wpr + ww] : 0u;
            }
            __syncwarp();
            if (lane == 0) {
                while (i > 0 && j > 0 && i >= r0) {
                    const int bb = j - i - lo - 16 * w0;
                    if (bb < 0 || bb >= 16 * PA_TILE_WORDS) break;
                    const uint32_t op = (tile[(i - r0) * PA_TILE_WORDS + (bb >> 4)] >> (2 * (bb & 15))) & 3u;
                    op_end[-1 - cnt] = op_char(op);
                    ++cnt;
                    i -= op != 3u;
                    j -= op != 2u;
                }
            }
            i = __shfl_sync(FULL, i, 0), j = __shfl_sync(FULL, j, 0), cnt = __shfl_sync(FULL, cnt, 0);
            __syncwarp();                                  // the walk has read the tile before it is reloaded
        }
        if (i > 0) gap_run(op_end, cnt, i, 'I', lane), cnt += i;
        if (j > 0) gap_run(op_end, cnt, j, 'D', lane), cnt += j;
        if (lane == 0) out[2 * p + 1] = cnt;
    }
}

__global__ void __launch_bounds__(32)
affine_kernel(const uint8_t* __restrict__ query, const uint8_t* __restrict__ ref, PairMeta meta, int n_pairs, int pitch,
              int2* __restrict__ ws, char* __restrict__ trace, uint8_t* __restrict__ ops, int* __restrict__ out) {
    __shared__ uint32_t tile[PA_TILE_ROWS * PA_TILE_WORDS];
    const int lane = threadIdx.x;
    int2* row = ws + (size_t)blockIdx.x * pitch;
    for (int p = blockIdx.x; p < n_pairs; p += gridDim.x) {
        const int m = meta.qlen[p], n = meta.rlen[p];
        const uint8_t* qp = query + meta.qoff[p];
        const uint8_t* rp = ref + meta.roff[p];
        const int wpr = (n + 7) >> 3;
        uint32_t* tb = reinterpret_cast<uint32_t*>(trace + meta.toff[p]);
        uint8_t* op_end = ops + meta.ooff[p] + m + n;
        if (m == 0 || n == 0) {                            // nothing to align: one free gap
            gap_run(op_end, 0, m, 'I', lane);
            gap_run(op_end, m, n, 'D', lane);
            if (lane == 0) out[2 * p] = 0, out[2 * p + 1] = m + n;
            continue;
        }
        // end-cell key: (H as an order-preserving uint32, rank), rank = m + j on row m, i on column n (i < m); H[m][0] = 0
        // is the starting candidate (it beats H[0][n] = 0 on the larger i)
        unsigned long long best = (0x80000000ull << 32) | (unsigned)m;
        for (int base = 0; base < m; base += PA_STRIP) {
            const int i0 = base + lane * PA_R + 1;
            const bool first = base == 0, more = base + PA_STRIP < m;
            uint32_t qc[PA_R], acc[PA_R];
            int hl[PA_R], el[PA_R];                        // H[i][c-1], E[i][c-1]
#pragma unroll
            for (int kk = 0; kk < PA_R; ++kk) {
                qc[kk] = i0 + kk <= m ? qp[i0 + kk - 1] : 0x100u;
                hl[kk] = 0;
                el[kk] = PA_NEG;
                acc[kk] = 0u;
            }
            int dh = 0;                                    // H[i0-1][0]
            int oh = 0, of = PA_NEG;
            for (int s = 0; s < n + 31; ++s) {
                int uh = __shfl_up_sync(FULL, oh, 1), uf = __shfl_up_sync(FULL, of, 1);
                const int c = s - lane + 1;
                if (c < 1 || c > n) continue;
                if (lane == 0) {
                    if (first) {
                        uh = 0, uf = PA_NEG;
                    } else {
                        const int2 a = row[c];
                        uh = a.x, uf = a.y;
                    }
                }
                const uint32_t rc = rp[c - 1];
                int di = dh;
                dh = uh;
#pragma unroll
                for (int kk = 0; kk < PA_R; ++kk) {
                    const int i = i0 + kk;
                    bool eo, fo;
                    const int e = __vibmax_s32(hl[kk] - 10, el[kk] - 2, &eo);
                    const int f = __vibmax_s32(uh - 10, uf - 2, &fo);
                    const bool match = qc[kk] == rc;
                    const int d = di + (match ? 5 : -4);
                    const int h = __vimax3_s32(d, e, f);
                    const uint32_t src = h == d ? (match ? 0u : 1u) : (h == e ? 3u : 2u);
                    di = hl[kk];
                    hl[kk] = h;
                    el[kk] = e;
                    uh = h;
                    uf = f;
                    if (i <= m) {
                        acc[kk] |= (src | (eo ? 4u : 0u) | (fo ? 8u : 0u)) << (4 * ((c - 1) & 7));
                        if (((c - 1) & 7) == 7 || c == n) {
                            tb[(size_t)(i - 1) * wpr + ((c - 1) >> 3)] = acc[kk];
                            acc[kk] = 0u;
                        }
                        if (i == m || c == n) {
                            const unsigned rank = i == m ? (unsigned)(m + c) : (unsigned)i;
                            const unsigned long long key = ((unsigned long long)((unsigned)h ^ 0x80000000u) << 32) | rank;
                            best = key > best ? key : best;
                        }
                    }
                }
                oh = uh, of = uf;
                if (lane == 31 && more) row[c] = make_int2(oh, of);
            }
            __syncwarp();
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const unsigned long long o = __shfl_xor_sync(FULL, best, off);
            best = o > best ? o : best;
        }
        const unsigned rank = (unsigned)(best & 0xffffffffu);
        const int ei = rank >= (unsigned)m ? m : (int)rank, ej = rank >= (unsigned)m ? (int)(rank - m) : n;
        // ---- traceback: the free trailing gap, the walk from (ei, ej), the free leading gap
        int cnt = 0;
        if (ei == m) gap_run(op_end, 0, n - ej, 'D', lane), cnt = n - ej;
        else gap_run(op_end, 0, m - ei, 'I', lane), cnt = m - ei;
        int i = ei, j = ej, state = 0;                     // 0: H, 1: E (D), 2: F (I)
        while (i > 0 && j > 0) {
            const int w0 = max(0, ((j - 1) >> 3) - (PA_TILE_WORDS - 1));
            const int r0 = i - (PA_TILE_ROWS - 1);
            for (int t = lane; t < PA_TILE_ROWS * PA_TILE_WORDS; t += 32) {
                const int rr = r0 + t / PA_TILE_WORDS, ww = w0 + t % PA_TILE_WORDS;
                tile[t] = (rr >= 1 && ww < wpr) ? tb[(size_t)(rr - 1) * wpr + ww] : 0u;
            }
            __syncwarp();
            if (lane == 0) {
                while (i > 0 && j > 0 && i >= r0 && ((j - 1) >> 3) >= w0) {
                    const uint32_t nib =
                        (tile[(i - r0) * PA_TILE_WORDS + ((j - 1) >> 3) - w0] >> (4 * ((j - 1) & 7))) & 15u;
                    if (state == 0) {
                        const uint32_t src = nib & 3u;
                        if (src < 2u) {
                            op_end[-1 - cnt] = op_char(src);
                            ++cnt, --i, --j;
                        } else {
                            state = src == 3u ? 1 : 2;
                        }
                    } else if (state == 1) {
                        op_end[-1 - cnt] = 'D';
                        ++cnt, --j;
                        if (nib & 4u) state = 0;
                    } else {
                        op_end[-1 - cnt] = 'I';
                        ++cnt, --i;
                        if (nib & 8u) state = 0;
                    }
                }
            }
            i = __shfl_sync(FULL, i, 0), j = __shfl_sync(FULL, j, 0), cnt = __shfl_sync(FULL, cnt, 0);
            state = __shfl_sync(FULL, state, 0);
            __syncwarp();
        }
        if (i > 0) gap_run(op_end, cnt, i, 'I', lane), cnt += i;
        if (j > 0) gap_run(op_end, cnt, j, 'D', lane), cnt += j;
        if (lane == 0) out[2 * p] = (int)((unsigned)(best >> 32) ^ 0x80000000u), out[2 * p + 1] = cnt;
    }
}

int pair_warps(int n_pairs) { return n_pairs < PA_MAX_WARPS ? n_pairs : PA_MAX_WARPS; }

int clamp_band(int k, int m, int n) {
    const int full = m > n ? m : n;
    return k < 0 ? 0 : (k > full ? full : k);
}

}  // namespace

size_t pair_align_trace_bytes(int mode, int m, int n, int band) {
    if (m <= 0 || n <= 0) return 0;
    size_t words;
    if (mode == B200_PAIR_GLOBAL_EDIT) {
        const long long k = clamp_band(band, m, n);
        const long long w = (long long)(n > m ? n - m : m - n) + 2 * k + 1;
        words = (size_t)m * (size_t)((w + 15) / 16);
    } else {
        words = (size_t)m * (size_t)((n + 7) / 8);
    }
    return (words * 4 + 15) & ~(size_t)15;
}

size_t pair_align_workspace_bytes(int mode, int n_pairs, const int* query_len, const int* ref_len, const int* band,
                                  int traceback) {
    if (n_pairs <= 0 || !query_len || !ref_len) return 0;
    size_t trace = 0;
    int max_ref = 1;
    for (int p = 0; p < n_pairs; ++p) {
        if (traceback) trace += pair_align_trace_bytes(mode, query_len[p], ref_len[p], band ? band[p] : 0);
        max_ref = ref_len[p] > max_ref ? ref_len[p] : max_ref;
    }
    return meta_bytes(n_pairs) + (size_t)pair_warps(n_pairs) * (size_t)(max_ref + 1) * sizeof(int2) + trace;
}

int launch_pair_align(int mode, const uint8_t* query, const long long* query_off, const int* query_len, const uint8_t* ref,
                      const long long* ref_off, const int* ref_len, const int* band, int n_pairs, int traceback,
                      void* workspace, uint8_t* ops, const long long* ops_off, int* out, cudaStream_t stream) {
    B200_REQUIRE(mode == B200_PAIR_GLOBAL_EDIT || mode == B200_PAIR_SEMIGLOBAL_AFFINE, "pair_align: unknown mode %d", mode);
    B200_REQUIRE(n_pairs >= 0, "pair_align: bad pair count %d", n_pairs);
    if (n_pairs == 0) return 0;
    B200_REQUIRE(query && query_off && query_len && ref && ref_off && ref_len && workspace && out,
                 "pair_align: null pointer argument");
    B200_REQUIRE(traceback || mode == B200_PAIR_GLOBAL_EDIT, "pair_align: SEMIGLOBAL_AFFINE always traces back");
    B200_REQUIRE(!traceback || (ops && ops_off), "pair_align: a traceback needs ops and ops_off");
    B200_REQUIRE(band || mode != B200_PAIR_GLOBAL_EDIT, "pair_align: GLOBAL_EDIT needs a band per pair");
    std::vector<long long> off64((size_t)n_pairs * 4, 0);
    std::vector<int> len32((size_t)n_pairs * 3, 0);
    size_t trace = 0;
    int max_ref = 1;
    for (int p = 0; p < n_pairs; ++p) {
        const int m = query_len[p], n = ref_len[p];
        B200_REQUIRE(m >= 0 && m <= PA_MAX_LEN && n >= 0 && n <= PA_MAX_LEN,
                     "pair_align: pair %d has lengths %d / %d; each side must be in [0, %d]", p, m, n, PA_MAX_LEN);
        B200_REQUIRE(query_off[p] >= 0 && ref_off[p] >= 0 && (!traceback || ops_off[p] >= 0),
                     "pair_align: pair %d has a negative offset", p);
        if (mode == B200_PAIR_GLOBAL_EDIT) B200_REQUIRE(band[p] >= 0, "pair_align: pair %d has band %d < 0", p, band[p]);
        off64[p] = query_off[p];
        off64[n_pairs + p] = ref_off[p];
        off64[2 * (size_t)n_pairs + p] = traceback ? ops_off[p] : 0;
        off64[3 * (size_t)n_pairs + p] = (long long)trace;
        len32[p] = m;
        len32[n_pairs + p] = n;
        len32[2 * (size_t)n_pairs + p] = mode == B200_PAIR_GLOBAL_EDIT ? clamp_band(band[p], m, n) : 0;
        if (traceback) trace += pair_align_trace_bytes(mode, m, n, len32[2 * (size_t)n_pairs + p]);
        max_ref = n > max_ref ? n : max_ref;
    }
    // the per-pair arrays go into the head of the workspace: [qoff | roff | ooff | toff] int64, [qlen | rlen | band] int32
    // (copied from pageable memory: cudaMemcpyAsync has staged them when it returns)
    char* head = static_cast<char*>(workspace);
    B200_CHECK_CUDA(cudaMemcpyAsync(head, off64.data(), off64.size() * sizeof(long long), cudaMemcpyHostToDevice, stream));
    B200_CHECK_CUDA(cudaMemcpyAsync(head + off64.size() * sizeof(long long), len32.data(), len32.size() * sizeof(int),
                                    cudaMemcpyHostToDevice, stream));
    const long long* d64 = reinterpret_cast<const long long*>(head);
    const int* d32 = reinterpret_cast<const int*>(head + off64.size() * sizeof(long long));
    const PairMeta meta{d64, d64 + n_pairs, d64 + 2 * (size_t)n_pairs, d64 + 3 * (size_t)n_pairs, d32, d32 + n_pairs,
                        d32 + 2 * (size_t)n_pairs};
    const int warps = pair_warps(n_pairs), pitch = max_ref + 1;
    int2* rows = reinterpret_cast<int2*>(head + meta_bytes(n_pairs));
    char* trace_base = reinterpret_cast<char*>(rows + (size_t)warps * pitch);
    if (mode == B200_PAIR_SEMIGLOBAL_AFFINE)
        affine_kernel<<<warps, 32, 0, stream>>>(query, ref, meta, n_pairs, pitch, rows, trace_base, ops, out);
    else if (traceback)
        edit_kernel<true><<<warps, 32, 0, stream>>>(query, ref, meta, n_pairs, pitch, rows, trace_base, ops, out);
    else
        edit_kernel<false><<<warps, 32, 0, stream>>>(query, ref, meta, n_pairs, pitch, rows, trace_base, ops, out);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}
