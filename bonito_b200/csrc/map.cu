// Read-to-reference mapping for `basecaller --reference`: minimizers, anchors, chaining and a banded local alignment
// along the chain.  minimap2 (what the reference maps with, through mappy) pins none of its heuristics, so the rules are
// this library's; the CPU oracle tests/_oracle_map.py restates every one of them and the tests hold the two byte-equal.
//
// Bases: A C G T (upper case) are 2-bit codes 0..3; every other byte is N.
//
// MINIMIZERS (b200_map_minimizers; sequences packed back to back, none crosses into the next):
//   the k-mer at position p (its first base) of a sequence is valid when its k bases are ACGT.  fwd = its 2-bit code
//   (first base most significant), rev = the code of its reverse complement; k is odd, so fwd != rev.  key = hash64(min(fwd,
//   rev)) << 1 | strand, strand = fwd > rev, hash64 = minimap2's invertible integer hash masked to 2k bits.
//   Window s = the k-mers s .. s+w-1 (all inside the sequence); its minimizer is the valid k-mer of the smallest hash, ties to
//   the leftmost; a window without a valid k-mer has none.  mm[p] = key if p is the minimizer of at least one window, else
//   -1.  A sequence shorter than k + w - 1 has no window and so no minimizer.
// INDEX (host side, bonito_b200/aligner.py): the reference minimizers sorted by (hash, position), a table of the unique
//   hashes, and for each entry val = global position << 1 | strand.  A hash with more than max_occ entries is never a seed.
// ANCHORS (b200_map_anchors, count then fill, so no atomic decides an order): for each read minimizer at read position x
//   and each index entry of its hash: relative strand s = read strand ^ entry strand; q = x on s = 0, L - x - k on s = 1
//   (the k-mer's start on the reverse complement of the read, L = read length); r = the entry's global position.
//   akey = read << 33 | s << 32 | r, written in (read minimizer, entry) order; the caller sorts stably by akey, so anchors
//   are in (read, strand, r) order and ties keep read-minimizer order.
// CHAINING (b200_map_chain; integers only), over the anchors of one read in that order:
//   f(i) = k + max(0, max_j f(j) + min(dq, dr, k) - gamma(|dr - dq|)), dr = r_i - r_j, dq = q_i - q_j,
//   j over the 50 anchors before i with the same strand and contig and 0 < dr <= 10000, 0 < dq <= 10000;
//   gamma(0) = 0, gamma(d) = floor(k d / 100) + floor(floor(log2 d) / 2).  pred(i) = the j of the maximum (ties to the
//   nearest, i.e. the largest j) when that maximum is > 0, else -1.
// EXTRACTION (b200_map_extract): anchors visited in decreasing f (ties to the lower index); an anchor not yet taken ends a
//   chain, which backtracks through pred, taking anchors, until an anchor already taken (or none).  Chain score = f(end) -
//   f(the taken anchor it stopped at) (or - 0).  The first chain is the primary (its score f1 is the largest).  f2 = the
//   largest score of the other chains whose query span overlaps the primary's by at least half of the shorter of the two
//   spans (spans in forward read coordinates, [first q, last q + k)).
// ALIGNMENT (b200_map_align), query = the read (reverse-complemented on strand 1, rows i = 1..m) against a target window
//   of the contig (columns j = 1..n), chain anchors (q, r) with r relative to the window:
//   band centre c(i) of row i (query base x = i - 1): r_a + floor((x - q_a)(r_b - r_a) / (q_b - q_a)) between consecutive
//   anchors a, b with q_a <= x < q_b, and slope 1 from the first anchor before it and from the last anchor after it.
//   Row i holds the columns j = c(i) + 1 - W + b, b = 0 .. 2W (W = band half-width), that lie in [1, n]; every other cell
//   is out of the band.  Local affine scores: s(a, b) = +2 if equal ACGT, -1 if either is N, -4 otherwise; a gap of g
//   bases costs 4 + 2 g:
//     E[i][j] = max(H[i][j-1] - 6, E[i][j-1] - 2)   op D          (open wins a tie over extend)
//     F[i][j] = max(H[i-1][j] - 6, F[i-1][j] - 2)   op I
//     H[i][j] = max(H[i-1][j-1] + s, E, F) when that is > 0 (ties: diagonal, then E, then F), else 0 (a start).
//   H = 0, E = F = NEG on row 0 and column 0; H = E = F = NEG out of the band.  The end cell is the largest H, ties to the
//   largest i, then the largest j; the walk back from it stops at a start cell (not aligned) or at row / column 0.  Ops
//   '=' (equal ACGT), 'X', 'I' (query base), 'D' (target base); a score of 0 means no alignment.
#include "common.cuh"

namespace {

constexpr int MAP_NEG = -(1 << 30);
constexpr int MAP_NEGA = -(1 << 29);      // the "no cell" of the E scan
constexpr int MAX_PRED = 50;
constexpr int MAX_GAP = 10000;
constexpr unsigned FULL = 0xffffffffu;
constexpr int THREADS = 256;

__device__ __forceinline__ int base_code(uint8_t c) {
    return c == 'A' ? 0 : c == 'C' ? 1 : c == 'G' ? 2 : c == 'T' ? 3 : -1;
}

// minimap2's hash64 (Thomas Wang's integer hash), invertible on the masked bits
__device__ __forceinline__ uint64_t hash64(uint64_t key, uint64_t mask) {
    key = (~key + (key << 21)) & mask;
    key = key ^ key >> 24;
    key = ((key + (key << 3)) + (key << 8)) & mask;
    key = key ^ key >> 14;
    key = ((key + (key << 2)) + (key << 4)) & mask;
    key = key ^ key >> 28;
    key = (key + (key << 31)) & mask;
    return key;
}

// the largest s with off[s] <= p (off: n + 1 ascending offsets)
__device__ __forceinline__ int seq_of(const long long* off, int n, long long p) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (off[mid] <= p) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

__global__ void kmer_kernel(const uint8_t* __restrict__ seq, long long n_bases, const long long* __restrict__ off, int n_seqs,
                            int k, long long* __restrict__ kmer) {
    const uint64_t mask = (1ull << (2 * k)) - 1;
    for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < n_bases; p += (long long)gridDim.x * blockDim.x) {
        const int s = seq_of(off, n_seqs, p);
        long long key = -1;
        if (p + k <= off[s + 1]) {
            uint64_t fwd = 0, rev = 0;
            bool ok = true;
            for (int t = 0; t < k; ++t) {
                const int c = base_code(seq[p + t]);
                if (c < 0) { ok = false; break; }
                fwd = (fwd << 2) | (uint64_t)c;
                rev |= (uint64_t)(3 - c) << (2 * t);
            }
            if (ok) key = (long long)((hash64(fwd < rev ? fwd : rev, mask) << 1) | (fwd > rev ? 1ull : 0ull));
        }
        kmer[p] = key;
    }
}

// one thread per window start; every winner writes its own key, so concurrent writers of one position agree
__global__ void window_kernel(long long n_bases, const long long* __restrict__ off, int n_seqs, int k, int w,
                              const long long* __restrict__ kmer, long long* __restrict__ mm) {
    for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < n_bases; p += (long long)gridDim.x * blockDim.x) {
        const int s = seq_of(off, n_seqs, p);
        if (p + w + k - 1 > off[s + 1]) continue;
        long long best = -1, at = -1;
        for (int t = 0; t < w; ++t) {
            const long long key = kmer[p + t];
            if (key >= 0 && (best < 0 || (key >> 1) < (best >> 1))) best = key, at = p + t;
        }
        if (at >= 0) mm[at] = best;
    }
}

// index of hash h in the sorted unique table, or -1
__device__ __forceinline__ long long find_hash(const long long* uniq, long long n_unique, long long h) {
    long long lo = 0, hi = n_unique;
    while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if (uniq[mid] < h) lo = mid + 1;
        else hi = mid;
    }
    return lo < n_unique && uniq[lo] == h ? lo : -1;
}

__global__ void anchor_kernel(const long long* __restrict__ mm, long long n_bases, const long long* __restrict__ off, int n_seqs,
                              int k, const long long* __restrict__ uniq, long long n_unique,
                              const long long* __restrict__ start, const long long* __restrict__ val, int max_occ,
                              int* __restrict__ count, const long long* __restrict__ aoff, long long* __restrict__ akey,
                              int* __restrict__ aq) {
    for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < n_bases; p += (long long)gridDim.x * blockDim.x) {
        const long long key = mm[p];
        const long long u = key < 0 ? -1 : find_hash(uniq, n_unique, key >> 1);
        const long long cnt = u < 0 ? 0 : start[u + 1] - start[u];
        const int use = cnt <= max_occ ? (int)cnt : 0;
        if (count) {
            count[p] = use;
            continue;
        }
        if (!use) continue;
        const int s = seq_of(off, n_seqs, p);
        const long long x = p - off[s], len = off[s + 1] - off[s];
        long long o = aoff[p];
        for (long long e = start[u]; e < start[u] + use; ++e, ++o) {
            const long long v = val[e];
            const long long rel = (key ^ v) & 1;
            akey[o] = ((long long)s << 33) | (rel << 32) | (v >> 1);
            aq[o] = (int)(rel ? len - x - k : x);
        }
    }
}

__device__ __forceinline__ int gap_cost(int d, int k) { return d == 0 ? 0 : (k * d) / 100 + (31 - __clz(d)) / 2; }

// one warp per read; lanes over the 50 predecessors, f of the last 64 anchors in a shared ring
constexpr int CHAIN_WARPS = 4;
__global__ void __launch_bounds__(32 * CHAIN_WARPS)
chain_kernel(const long long* __restrict__ akey, const int* __restrict__ aq, const long long* __restrict__ roff, int n_reads,
             const long long* __restrict__ ctg_off, int n_ctg, int k, int* __restrict__ f, int* __restrict__ pred) {
    __shared__ int ring[CHAIN_WARPS][64];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (int rd = blockIdx.x * CHAIN_WARPS + wid; rd < n_reads; rd += gridDim.x * CHAIN_WARPS) {
        const long long a0 = roff[rd], a1 = roff[rd + 1];
        for (long long i = a0; i < a1; ++i) {
            const long long ki = akey[i];
            const long long ri = ki & 0xffffffffll, si = (ki >> 32) & 1;
            const int qi = aq[i];
            const long long cstart = ctg_off[seq_of(ctg_off, n_ctg, ri)];
            unsigned long long best = 0;
            for (int t = lane; t < MAX_PRED; t += 32) {
                const long long j = i - 1 - t;
                if (j < a0) break;
                const long long kj = akey[j];
                const long long rj = kj & 0xffffffffll;
                const long long dr = ri - rj, dq = qi - aq[j];
                if (((kj >> 32) & 1) != si || rj < cstart || dr <= 0 || dr > MAX_GAP || dq <= 0 || dq > MAX_GAP) continue;
                const int sc = ring[wid][(j - a0) & 63] + (int)min(min(dq, dr), (long long)k) -
                               gap_cost((int)(dr > dq ? dr - dq : dq - dr), k);
                if (sc > 0) {
                    const unsigned long long c = ((unsigned long long)sc << 32) | (unsigned)(j - a0 + 1);
                    best = c > best ? c : best;
                }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const unsigned long long v = __shfl_xor_sync(FULL, best, o);
                best = v > best ? v : best;
            }
            const int fi = k + (int)(best >> 32);
            if (lane == 0) {
                ring[wid][(i - a0) & 63] = fi;
                f[i] = fi;
                pred[i] = best ? (int)(a0 + (long long)(best & 0xffffffffu) - 1) : -1;
            }
            __syncwarp();
        }
    }
}

// one thread per read: the greedy extraction; out[rd] = n, f1, f2, strand, W, q0, r0, q1, r1 (int64) and the primary
// chain's (q, r) pairs at chain[2 * roff[rd] ..]
__global__ void extract_kernel(const long long* __restrict__ akey, const int* __restrict__ aq, const int* __restrict__ f,
                               const int* __restrict__ pred, const long long* __restrict__ order,
                               const long long* __restrict__ roff, const long long* __restrict__ seq_off, int n_reads, int k,
                               int max_band, uint8_t* __restrict__ taken, long long* __restrict__ chain,
                               long long* __restrict__ out) {
    for (int rd = blockIdx.x * blockDim.x + threadIdx.x; rd < n_reads; rd += gridDim.x * blockDim.x) {
        const long long a0 = roff[rd], a1 = roff[rd + 1], len = seq_off[rd + 1] - seq_off[rd];
        long long* o = out + 9ll * rd;
        long long n1 = 0, e1 = -1, f1 = 0, f2 = 0, ps = 0, pe = 0;
        for (long long t = a0; t < a1; ++t) {
            const long long e = order[t];
            if (taken[e]) continue;
            long long i = e, first = e, n = 0;
            while (i >= 0 && !taken[i]) {
                taken[i] = 1;
                ++n;
                first = i;
                i = pred[i];
            }
            const long long sc = f[e] - (i >= 0 ? f[i] : 0);
            long long qs = aq[first], qe = aq[e] + k;
            if ((akey[e] >> 32) & 1) {
                const long long tmp = qs;
                qs = len - qe, qe = len - tmp;
            }
            if (e1 < 0) {
                e1 = e, n1 = n, f1 = sc, ps = qs, pe = qe;
            } else {
                const long long ov = min(pe, qe) - max(ps, qs), shorter = min(pe - ps, qe - qs);
                if (ov > 0 && 2 * ov >= shorter && sc > f2) f2 = sc;
            }
        }
        long long band = 0;
        if (e1 >= 0) {
            long long i = e1, prev_d = 0;
            for (long long t = n1 - 1; t >= 0; --t) {
                const long long r = akey[i] & 0xffffffffll, q = aq[i], d = r - q;
                chain[2 * (a0 + t)] = q;
                chain[2 * (a0 + t) + 1] = r;
                if (t < n1 - 1) band = max(band, prev_d > d ? prev_d - d : d - prev_d);
                prev_d = d;
                i = pred[i];
            }
            band = min(64 + band, (long long)max_band);
        }
        o[0] = n1, o[1] = f1, o[2] = f2, o[3] = e1 >= 0 ? (akey[e1] >> 32) & 1 : 0, o[4] = band;
        o[5] = n1 ? chain[2 * a0] : 0, o[6] = n1 ? chain[2 * a0 + 1] : 0;
        o[7] = n1 ? chain[2 * (a0 + n1 - 1)] : 0, o[8] = n1 ? chain[2 * (a0 + n1 - 1) + 1] : 0;
    }
}

// ---------------------------------------------------------------------------- banded local alignment along a chain
// meta per pair (int64): qoff, m, toff, n, coff (chain pair index), clen, W, trace byte offset, ops slot offset (m + n)
constexpr int META = 9;

__device__ __forceinline__ int map_score(uint8_t a, uint8_t b) {
    const int ca = base_code(a), cb = base_code(b);
    return (ca < 0 || cb < 0) ? -1 : (ca == cb ? 2 : -4);
}

__host__ __device__ __forceinline__ int band_cells(int band) { return 8 * ((2 * band + 1 + 255) / 256); }   // C: cells per lane

// One warp per pair.  Lane l owns the band offsets b = 32 t + l of a row (t < C); a row is one pass over t with an
// inclusive max-scan across the warp for E (E[j] + 2j is the running max of H''[j'] + 2j' - 4 over the band cells left of
// j, H'' = max(0, diagonal, F): the terms where E itself won are strictly dominated by the extension they came from).
// Rows i-1 and i live in shared memory (H and F, NEG out of the band).  Traceback nibbles (bits 0-1: 0 diagonal,
// 1 start, 2 F, 3 E; bit 2: E opened; bit 3: F opened) go to row i - 1 of the pair's trace, word (t / 8) * 32 + l.
__global__ void __launch_bounds__(32)
align_kernel(const uint8_t* __restrict__ query, const uint8_t* __restrict__ target, const long long* __restrict__ chain,
             const long long* __restrict__ meta, int n_pairs, int C, int* __restrict__ cen_all, char* __restrict__ trace_all,
             uint8_t* __restrict__ ops_all, int* __restrict__ out) {
    extern __shared__ int smem[];
    const int lane = threadIdx.x, S = 32 * C;       // buffer pitch: the launch's widest band
    for (int p = blockIdx.x; p < n_pairs; p += gridDim.x) {
        const long long* mp = meta + (size_t)META * p;
        const uint8_t* qp = query + mp[0];
        const uint8_t* tp = target + mp[2];
        const int m = (int)mp[1], n = (int)mp[3], W = (int)mp[6];
        const long long* ch = chain + 2 * mp[4];
        const int nc = (int)mp[5];
        const long long toff = mp[2];
        int* cen = cen_all + mp[0];
        uint32_t* tb = reinterpret_cast<uint32_t*>(trace_all + mp[7]);
        const int cp = band_cells(W), sp = 32 * cp;     // this pair's cells per lane and per row
        const int rw = 4 * cp;                             // trace words per row
        // band centres
        for (int x = lane; x < m; x += 32) {
            long long c;
            if (x <= ch[0]) {
                c = ch[1] - toff + (x - ch[0]);
            } else if (x >= ch[2 * (nc - 1)]) {
                c = ch[2 * (nc - 1) + 1] - toff + (x - ch[2 * (nc - 1)]);
            } else {
                int lo = 0, hi = nc - 1;                   // largest a with q_a <= x
                while (lo < hi) {
                    const int mid = (lo + hi + 1) >> 1;
                    if (ch[2 * mid] <= x) lo = mid;
                    else hi = mid - 1;
                }
                const long long qa = ch[2 * lo], ra = ch[2 * lo + 1] - toff, qb = ch[2 * lo + 2], rb = ch[2 * lo + 3] - toff;
                c = ra + (x - qa) * (rb - ra) / (qb - qa);
            }
            cen[x] = (int)c;
        }
        __syncwarp();
        int* ph = smem;
        int* pf = smem + S;
        int* chh = smem + 2 * S;
        int* chf = smem + 3 * S;
        unsigned long long best = 0;
        int lo_prev = 0;
        for (int i = 1; i <= m; ++i) {
            const int lo = cen[i - 1] + 1 - W, shift = lo - lo_prev;
            lo_prev = lo;
            const uint8_t qc = qp[i - 1];
            int carry_a = lo == 1 ? -4 : MAP_NEGA;        // column 0 right before offset 0
            int ch_h = 0, ch_e = MAP_NEG;                  // the cell before offset 0 (used only when it is in the band)
            bool ch_in = false;
            uint32_t acc = 0;
            for (int t = 0; t < cp; ++t) {
                const int b = 32 * t + lane, j = lo + b;
                const bool inb = b <= 2 * W && j >= 1 && j <= n;
                int up_h, up_f, dg;
                if (i == 1) {
                    up_h = 0, up_f = MAP_NEG, dg = 0;
                } else {
                    const int ub = b + shift;
                    up_h = ub < sp ? ph[ub] : MAP_NEG;
                    up_f = ub < sp ? pf[ub] : MAP_NEG;
                    dg = j == 1 ? 0 : (ub - 1 >= 0 && ub - 1 < sp ? ph[ub - 1] : MAP_NEG);
                }
                const int s = inb ? map_score(qc, tp[j - 1]) : 0;
                const int d = dg + s;
                const bool fo = up_h - 6 >= up_f - 2;
                const int fv = fo ? up_h - 6 : up_f - 2;
                const int hpp = max(0, max(d, fv));
                const int a = inb ? hpp + 2 * j - 4 : ((j == 0 && b <= 2 * W) ? -4 : MAP_NEGA);
                int incl = a;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int v = __shfl_up_sync(FULL, incl, o);
                    if (lane >= o) incl = max(incl, v);
                }
                int excl = __shfl_up_sync(FULL, incl, 1);
                excl = lane == 0 ? carry_a : max(excl, carry_a);
                carry_a = max(carry_a, __shfl_sync(FULL, incl, 31));
                const int e = excl >= -4 ? excl - 2 * j : MAP_NEG;
                const int m3 = max(d, max(e, fv));
                uint32_t src;
                int h;
                if (m3 <= 0) h = 0, src = 1u;
                else h = m3, src = m3 == d ? 0u : (m3 == e ? 3u : 2u);
                if (!inb) h = MAP_NEG;
                // E opened: from the cell before (b - 1): lane - 1 at this t, or lane 31 at t - 1
                int p_h = __shfl_up_sync(FULL, h, 1), p_e = __shfl_up_sync(FULL, e, 1);
                bool p_in = __shfl_up_sync(FULL, inb, 1);
                if (lane == 0) p_h = ch_h, p_e = ch_e, p_in = ch_in;
                const bool eo = j == 1 ? true : (p_in && p_h - 6 >= p_e - 2);
                ch_h = __shfl_sync(FULL, h, 31), ch_e = __shfl_sync(FULL, e, 31), ch_in = __shfl_sync(FULL, inb, 31);
                chh[b] = h;
                chf[b] = inb ? fv : MAP_NEG;
                acc |= (src | (eo ? 4u : 0u) | (fo ? 8u : 0u)) << (4 * (t & 7));
                if ((t & 7) == 7) {
                    tb[(size_t)(i - 1) * rw + (t >> 3) * 32 + lane] = acc;
                    acc = 0;
                }
                if (inb && h > 0) {
                    const unsigned long long key =
                        ((unsigned long long)h << 44) | ((unsigned long long)i << 22) | (unsigned long long)j;
                    best = key > best ? key : best;
                }
            }
            __syncwarp();
            int* tmp = ph;
            ph = chh, chh = tmp;
            tmp = pf, pf = chf, chf = tmp;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long v = __shfl_xor_sync(FULL, best, o);
            best = v > best ? v : best;
        }
        if (lane == 0) {
            const int score = (int)(best >> 44);
            const int ei = (int)((best >> 22) & 0x3fffff), ej = (int)(best & 0x3fffff);
            uint8_t* op_end = ops_all + mp[8] + m + n;
            int i = ei, j = ej, cnt = 0, state = 0;
            while (score > 0 && i > 0 && j > 0) {
                const int b = j - (cen[i - 1] + 1 - W), t = b >> 5;
                const uint32_t nib = (tb[(size_t)(i - 1) * rw + (t >> 3) * 32 + (b & 31)] >> (4 * (t & 7))) & 15u;
                uint8_t op;
                if (state == 0) {
                    const uint32_t src = nib & 3u;
                    if (src == 1u) break;
                    if (src != 0u) {
                        state = src == 3u ? 1 : 2;
                        continue;
                    }
                    const int ca = base_code(qp[i - 1]);
                    op = (ca >= 0 && ca == base_code(tp[j - 1])) ? '=' : 'X';
                    --i, --j;
                } else if (state == 1) {
                    op = 'D';
                    --j;
                    if (nib & 4u) state = 0;
                } else {
                    op = 'I';
                    --i;
                    if (nib & 8u) state = 0;
                }
                op_end[-1 - cnt] = op;
                ++cnt;
            }
            int* o = out + 6 * p;
            o[0] = score, o[1] = score > 0 ? i : 0, o[2] = score > 0 ? ei : 0, o[3] = score > 0 ? j : 0;
            o[4] = score > 0 ? ej : 0, o[5] = cnt;
        }
        __syncwarp();
    }
}

int grid_for(long long n, int threads) {
    const long long blocks = (n + threads - 1) / threads;
    return (int)(blocks < 65536 ? (blocks > 0 ? blocks : 1) : 65536);
}

}  // namespace

extern "C" {

int b200_map_minimizers(const void* seq, long long n_bases, const long long* seq_off, int n_seqs, int k, int w, void* kmer,
                        void* mm, void* stream) {
    B200_REQUIRE(k >= 3 && k <= 31 && (k & 1) && w >= 1 && w <= 255, "map_minimizers: need odd k in [3, 31] and w in [1, 255] "
                 "(got k=%d w=%d)", k, w);
    B200_REQUIRE(n_bases >= 0 && n_seqs >= 0, "map_minimizers: bad sizes");
    if (n_bases == 0 || n_seqs == 0) return 0;
    B200_REQUIRE(seq && seq_off && kmer && mm, "map_minimizers: null pointer argument");
    cudaStream_t st = (cudaStream_t)stream;
    B200_CHECK_CUDA(cudaMemsetAsync(mm, 0xff, (size_t)n_bases * 8, st));
    const int grid = grid_for(n_bases, THREADS);
    kmer_kernel<<<grid, THREADS, 0, st>>>((const uint8_t*)seq, n_bases, seq_off, n_seqs, k, (long long*)kmer);
    window_kernel<<<grid, THREADS, 0, st>>>(n_bases, seq_off, n_seqs, k, w, (const long long*)kmer, (long long*)mm);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int b200_map_anchors(const void* mm, long long n_bases, const long long* seq_off, int n_seqs, int k, const void* uniq,
                     long long n_unique, const void* start, const void* val, int max_occ, void* count, const void* aoff,
                     void* akey, void* aq, void* stream) {
    B200_REQUIRE(n_bases >= 0 && n_seqs >= 0 && n_unique >= 0, "map_anchors: bad sizes");
    if (n_bases == 0 || n_seqs == 0) return 0;
    B200_REQUIRE(mm && seq_off && start && (uniq || !n_unique) && (val || !n_unique), "map_anchors: null pointer argument");
    B200_REQUIRE(count || (aoff && akey && aq), "map_anchors: need count, or aoff, akey and aq");
    anchor_kernel<<<grid_for(n_bases, THREADS), THREADS, 0, (cudaStream_t)stream>>>(
        (const long long*)mm, n_bases, seq_off, n_seqs, k, (const long long*)uniq, n_unique, (const long long*)start,
        (const long long*)val, max_occ, (int*)count, (const long long*)aoff, (long long*)akey, (int*)aq);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int b200_map_chain(const void* akey, const void* aq, const long long* read_aoff, int n_reads, const long long* ctg_off, int n_ctg,
                   int k, void* f, void* pred, void* stream) {
    B200_REQUIRE(n_reads >= 0 && n_ctg > 0, "map_chain: bad sizes");
    if (n_reads == 0) return 0;
    B200_REQUIRE(akey && aq && read_aoff && ctg_off && f && pred, "map_chain: null pointer argument");
    const int blocks = (n_reads + CHAIN_WARPS - 1) / CHAIN_WARPS;
    chain_kernel<<<blocks < 65536 ? blocks : 65536, 32 * CHAIN_WARPS, 0, (cudaStream_t)stream>>>(
        (const long long*)akey, (const int*)aq, read_aoff, n_reads, ctg_off, n_ctg, k, (int*)f, (int*)pred);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int b200_map_extract(const void* akey, const void* aq, const void* f, const void* pred, const void* order,
                     const long long* read_aoff, const long long* seq_off, int n_reads, int k, int max_band, void* taken,
                     void* chain, void* out, void* stream) {
    B200_REQUIRE(n_reads >= 0 && max_band >= 64, "map_extract: bad sizes");
    if (n_reads == 0) return 0;
    B200_REQUIRE(read_aoff && seq_off && taken && out, "map_extract: null pointer argument");
    extract_kernel<<<grid_for(n_reads, 128), 128, 0, (cudaStream_t)stream>>>(
        (const long long*)akey, (const int*)aq, (const int*)f, (const int*)pred, (const long long*)order, read_aoff, seq_off,
        n_reads, k, max_band, (uint8_t*)taken, (long long*)chain, (long long*)out);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

size_t b200_map_align_trace_bytes(int query_len, int band) {
    if (query_len <= 0 || band < 0) return 0;
    return (size_t)query_len * 16 * (size_t)band_cells(band);
}

int b200_map_align(const void* query, const void* target, const void* chain, const void* meta, int n_pairs, int max_band,
                   void* cen, void* trace, void* ops, void* out, void* stream) {
    B200_REQUIRE(n_pairs >= 0 && max_band >= 0 && max_band <= 4096, "map_align: bad sizes (n_pairs %d, max_band %d)", n_pairs,
                 max_band);
    if (n_pairs == 0) return 0;
    B200_REQUIRE(query && target && chain && meta && cen && trace && ops && out, "map_align: null pointer argument");
    const int C = band_cells(max_band);
    const size_t smem = (size_t)4 * 32 * C * sizeof(int);
    B200_CHECK_CUDA(cudaFuncSetAttribute(align_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int grid = n_pairs < 4096 ? n_pairs : 4096;
    align_kernel<<<grid, 32, smem, (cudaStream_t)stream>>>((const uint8_t*)query, (const uint8_t*)target,
                                                           (const long long*)chain, (const long long*)meta, n_pairs, C,
                                                           (int*)cen, (char*)trace, (uint8_t*)ops, (int*)out);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // extern "C"
