// BGZF compression (SAM specification section 4.1) for BAM output: one CTA per member of 65280 input bytes.
//
// Per member, in one CTA (the member staged in shared memory):
//   1. CRC32: a table CRC per thread over a contiguous slice, the slices combined by GF(2) shifts.
//   2. Hash chains: prev[p] = the last q < p whose next three bytes hash like p's.  Positions go through in chunks of
//      CHUNK; a stable block radix sort of each chunk by hash links equal hashes inside it, a head table links them to
//      earlier chunks.
//   3. Match search in parallel: every position follows its chain for up to CHAIN_DEPTH candidates within 32 KiB and
//      keeps the longest match (the nearest on ties).  A length-3 match further than 4 KiB costs more bits than three
//      literals and is dropped, as zlib does.
//   4. Greedy parse in one warp: from position 0, the match where there is one, else a literal.
//   5. Symbol histograms (shared-memory atomic adds: the counts do not depend on their order).
//   6. Canonical Huffman codes limited to 15 bits (literal/length, distance) and 7 bits (code lengths), built on one
//      thread each from a parallel rank sort.
//   7. Bits emitted in parallel: an exclusive scan of the symbols' bit counts gives every thread its bit offset, and the
//      bits are OR-ed into shared-memory words.  A stored block is written instead when it is not larger.
// The members land in per-member slots of the workspace; a scan launch computes their offsets and a copy launch packs them
// back to back into `out`.  Nothing depends on the order of atomics beyond the adds and ORs above, so the output is
// byte-identical from run to run.
#include <cub/block/block_radix_sort.cuh>

#include "common.cuh"

namespace {

constexpr int MEMBER_IN = B200_BGZF_MEMBER_INPUT;  // input bytes per member
constexpr int SLOT = 65536;                         // output bytes per member slot and per output member (stored: 65311)
constexpr int MEMBER_THREADS = 512;
constexpr int ITEMS = 2;
constexpr int CHUNK = MEMBER_THREADS * ITEMS;  // positions per hash-chain round
constexpr int HASH_BITS = 15;
constexpr int CHAIN_DEPTH = 4;
constexpr int WINDOW = 32768;
constexpr int MAX_MATCH = 258;
constexpr int FAR_MATCH3 = 4096;
constexpr uint16_t NONE = 0xffff;
constexpr int HEADER_BYTES = 18, TRAILER_BYTES = 8;
constexpr uint32_t CRC_POLY = 0xedb88320u;
constexpr int COPY_THREADS = 256, SCAN_THREADS = 1024;

constexpr int N_LIT = 286, N_DIST = 30, N_CL = 19;
constexpr int SEL = 0x8000, IS_MATCH = 0x4000;  // per-position code word after the parse: selected, match (else literal)

__constant__ uint8_t kClOrder[N_CL] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

using Sort = cub::BlockRadixSort<uint32_t, MEMBER_THREADS, ITEMS, uint16_t>;

// length 3..258 -> literal/length symbol - 257, extra bits, extra value (RFC 1951 section 3.2.5)
__device__ __forceinline__ void length_code(int len, int& idx, int& nbits, int& extra) {
    const int v = len - 3;
    if (len == MAX_MATCH) {
        idx = 28, nbits = 0, extra = 0;
    } else if (v < 8) {
        idx = v, nbits = 0, extra = 0;
    } else {
        const int lg = 31 - __clz(v);
        idx = 4 * (lg - 1) + ((v >> (lg - 2)) & 3);
        nbits = idx / 4 - 1;
        extra = v - ((4 + (idx & 3)) << nbits);
    }
}

// distance 1..32768 -> distance symbol, extra bits, extra value
__device__ __forceinline__ void dist_code(int dist, int& code, int& nbits, int& extra) {
    const int v = dist - 1;
    if (v < 4) {
        code = v, nbits = 0, extra = 0;
    } else {
        const int lg = 31 - __clz(v);
        code = 2 * lg + ((v >> (lg - 1)) & 1);
        nbits = code / 2 - 1;
        extra = v - ((2 + (code & 1)) << nbits);
    }
}

// a * b modulo the CRC polynomial, both reflected (the top bit is x^0)
__device__ uint32_t crc_multmod(uint32_t a, uint32_t b) {
    uint32_t p = 0;
    for (uint32_t m = 1u << 31; m; m >>= 1) {
        if (a & m) p ^= b;
        b = (b & 1) ? (b >> 1) ^ CRC_POLY : b >> 1;
    }
    return p;
}

// x^(8 * bytes) modulo the polynomial, what `bytes` zero bytes do to a CRC register; x2n[k] = x^(2^k)
__device__ uint32_t crc_shift_op(uint32_t bytes, const uint32_t* x2n) {
    uint32_t p = 1u << 31;
    for (int k = 3; bytes; bytes >>= 1, ++k)
        if (bytes & 1) p = crc_multmod(x2n[k], p);
    return p;
}

// ORs bits, LSB first, into 32-bit shared-memory words from an arbitrary bit offset
struct BitWriter {
    uint32_t* words;
    int w, nbits;
    uint64_t acc;
    __device__ BitWriter(uint32_t* out, int bitpos) : words(out), w(bitpos >> 5), nbits(bitpos & 31), acc(0) {}
    __device__ __forceinline__ void put(uint32_t v, int n) {  // n <= 32
        acc |= (uint64_t)v << nbits;
        nbits += n;
        if (nbits >= 32) {
            atomicOr(&words[w++], (uint32_t)acc);
            acc >>= 32;
            nbits -= 32;
        }
    }
    __device__ __forceinline__ void flush() {
        if (nbits > 0) atomicOr(&words[w], (uint32_t)acc);
    }
};

struct Shared {
    uint32_t lit_freq[N_LIT];
    uint32_t dist_freq[N_DIST];
    uint32_t cl_freq[N_CL];
    uint16_t lit_sorted[N_LIT];  // used symbols by ascending (frequency, symbol)
    uint16_t dist_sorted[N_DIST];
    uint16_t cl_sorted[N_CL];
    uint8_t lit_len[N_LIT];
    uint8_t dist_len[N_DIST];
    uint8_t cl_len[N_CL];
    uint16_t lit_code[N_LIT];  // bit-reversed canonical codes
    uint16_t dist_code[N_DIST];
    uint16_t cl_code[N_CL];
    uint8_t rle_sym[N_LIT + N_DIST];
    uint8_t rle_extra[N_LIT + N_DIST];
    int huff_scratch[2][N_LIT];
    uint32_t x2n[32];
    uint32_t crc_part[MEMBER_THREADS];
    int warp_sum[MEMBER_THREADS / 32];
    int n_lit_used, n_dist_used, n_rle, hlit, hdist, hclen, header_bits;
};

// Code lengths (<= limit) from the frequencies, given sorted[] = the n_used (>= 2) used symbols by ascending (frequency,
// symbol): minimum-redundancy lengths in place (Moffat and Katajainen), then the per-length counts brought under the limit
// with the Kraft sum kept at one.  One thread.
__device__ void huffman_lengths(const uint32_t* freq, const uint16_t* sorted, int n_used, int limit, uint8_t* len, int n,
                                int* a) {
    for (int i = 0; i < n; ++i) len[i] = 0;
    for (int i = 0; i < n_used; ++i) a[i] = (int)freq[sorted[i]];
    a[0] += a[1];
    int root = 0, leaf = 2;
    for (int next = 1; next < n_used - 1; ++next) {  // parent pointers
        if (leaf >= n_used || a[root] < a[leaf]) {
            a[next] = a[root];
            a[root++] = next;
        } else {
            a[next] = a[leaf++];
        }
        if (leaf >= n_used || (root < next && a[root] < a[leaf])) {
            a[next] += a[root];
            a[root++] = next;
        } else {
            a[next] += a[leaf++];
        }
    }
    a[n_used - 2] = 0;  // internal node depths
    for (int next = n_used - 3; next >= 0; --next) a[next] = a[a[next]] + 1;
    int avbl = 1, used = 0, depth = 0, next = n_used - 1;  // leaf depths
    root = n_used - 2;
    while (avbl > 0) {
        while (root >= 0 && a[root] == depth) {
            ++used;
            --root;
        }
        while (avbl > used) {
            a[next--] = depth;
            --avbl;
        }
        avbl = 2 * used;
        ++depth;
        used = 0;
    }
    int count[33];
    for (int i = 0; i <= 32; ++i) count[i] = 0;
    for (int i = 0; i < n_used; ++i) ++count[min(a[i], 32)];
    for (int i = limit + 1; i <= 32; ++i) count[limit] += count[i];
    uint32_t total = 0;
    for (int i = limit; i > 0; --i) total += (uint32_t)count[i] << (limit - i);
    while (total != (1u << limit)) {
        --count[limit];
        for (int i = limit - 1; i > 0; --i)
            if (count[i]) {
                --count[i];
                count[i + 1] += 2;
                break;
            }
        --total;
    }
    int j = n_used;  // the most frequent symbols get the shortest codes
    for (int l = 1; l <= limit; ++l)
        for (int c = count[l]; c > 0; --c) len[sorted[--j]] = (uint8_t)l;
}

// bit-reversed canonical codes of the lengths (RFC 1951 section 3.2.2).  One thread.
__device__ void canonical_codes(const uint8_t* len, int n, uint16_t* code) {
    int count[16] = {0}, next[16] = {0};
    for (int i = 0; i < n; ++i) ++count[len[i]];
    count[0] = 0;
    int c = 0;
    for (int l = 1; l < 16; ++l) {
        c = (c + count[l - 1]) << 1;
        next[l] = c;
    }
    for (int i = 0; i < n; ++i) {
        const int l = len[i];
        code[i] = l ? (uint16_t)(__brev((uint32_t)next[l]++) >> (32 - l)) : 0;
    }
}

// at least two used symbols, so that every code is complete (zlib's rule): the lowest unused symbols get a count of one
__device__ void force_two(uint32_t* freq, int n) {
    int used = 0;
    for (int i = 0; i < n; ++i) used += freq[i] != 0;
    for (int i = 0; i < n && used < 2; ++i)
        if (!freq[i]) freq[i] = 1, ++used;
}

// sorted[] = the symbols with nonzero freq[] by ascending (frequency, symbol), over threads [first, first + count)
__device__ void rank_sort(const uint32_t* freq, int n, uint16_t* sorted, int first, int count) {
    for (int i = (int)threadIdx.x - first; i >= 0 && i < n; i += count) {
        const uint32_t f = freq[i];
        if (!f) continue;
        int rank = 0;
        for (int j = 0; j < n; ++j) {
            const uint32_t g = freq[j];
            rank += g && (g < f || (g == f && j < i));
        }
        sorted[rank] = (uint16_t)i;
    }
}

__device__ __forceinline__ int n_used(const uint32_t* freq, int n) {
    int used = 0;
    for (int i = 0; i < n; ++i) used += freq[i] != 0;
    return used;
}

constexpr size_t SORT_REGION = (2u << HASH_BITS) + sizeof(Sort::TempStorage) + CHUNK * 6;
static_assert(SORT_REGION <= 2 * MEMBER_IN, "the hash-chain scratch must fit in the per-position code array");
constexpr size_t MEMBER_SMEM = SLOT + 2 * MEMBER_IN + sizeof(Shared);

__global__ void __launch_bounds__(MEMBER_THREADS, 1)
    bgzf_member_kernel(const uint8_t* __restrict__ in, int64_t in_bytes, uint8_t* __restrict__ slots,
                       int* __restrict__ sizes, uint16_t* __restrict__ prev_all, uint16_t* __restrict__ dist_all) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint8_t* buf = smem;                        // the member's bytes; after the parse, the DEFLATE bit stream
    uint32_t* words = (uint32_t*)smem;
    uint16_t* code = (uint16_t*)(smem + SLOT);  // per position: match length, then the parse's code word
    Shared& s = *(Shared*)(smem + SLOT + 2 * MEMBER_IN);
    // phase 2 scratch inside code[]: the hash head table, the sort's storage and the sorted chunk
    uint16_t* head = code;
    auto& sort_tmp = *(Sort::TempStorage*)(smem + SLOT + (2u << HASH_BITS));
    uint32_t* chunk_hash = (uint32_t*)(smem + SLOT + (2u << HASH_BITS) + sizeof(Sort::TempStorage));
    uint16_t* chunk_pos = (uint16_t*)(chunk_hash + CHUNK);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t member = blockIdx.x;
    const uint8_t* src = in + member * MEMBER_IN;
    const int n = (int)min((int64_t)MEMBER_IN, in_bytes - member * MEMBER_IN);
    uint16_t* prev = prev_all + member * MEMBER_IN;
    uint16_t* dist = dist_all + member * MEMBER_IN;
    uint8_t* slot = slots + member * SLOT;

    // ---- 1. stage the member, zero padded, and take its CRC32
    for (int i = tid; i < SLOT; i += MEMBER_THREADS) buf[i] = i < n ? src[i] : 0;
    for (int i = tid; i < (1 << HASH_BITS); i += MEMBER_THREADS) head[i] = NONE;
    for (int i = tid; i < N_LIT; i += MEMBER_THREADS) s.lit_freq[i] = i == 256;  // one end-of-block symbol
    for (int i = tid; i < N_DIST; i += MEMBER_THREADS) s.dist_freq[i] = 0;
    uint32_t* crc_table = chunk_hash;  // free until phase 2
    if (tid < 256) {
        uint32_t c = tid;
        for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ CRC_POLY : c >> 1;
        crc_table[tid] = c;
    }
    if (tid == 0) {
        uint32_t x = 1u << 30;  // x^1
        for (int k = 0; k < 32; ++k) {
            s.x2n[k] = x;
            x = crc_multmod(x, x);
        }
    }
    __syncthreads();
    {
        const int per = (n + MEMBER_THREADS - 1) / MEMBER_THREADS;
        const int lo = min(n, tid * per), hi = min(n, lo + per);
        uint32_t c = 0;  // the slice's CRC register from zero, then shifted over the bytes after it
        for (int i = lo; i < hi; ++i) c = crc_table[(c ^ buf[i]) & 0xff] ^ (c >> 8);
        s.crc_part[tid] = crc_multmod(crc_shift_op((uint32_t)(n - hi), s.x2n), c);
    }
    __syncthreads();
    if (warp == 0) {
        uint32_t c = 0;
        for (int i = lane; i < MEMBER_THREADS; i += 32) c ^= s.crc_part[i];
        for (int o = 16; o; o >>= 1) c ^= __shfl_xor_sync(0xffffffffu, c, o);
        if (lane == 0) s.crc_part[0] = c ^ crc_multmod(crc_shift_op((uint32_t)n, s.x2n), 0xffffffffu) ^ 0xffffffffu;
    }
    __syncthreads();
    const uint32_t crc = s.crc_part[0];

    // ---- 2. hash chains
    for (int base = 0; base < n; base += CHUNK) {
        uint32_t key[ITEMS];
        uint16_t pos[ITEMS];
        for (int k = 0; k < ITEMS; ++k) {
            const int p = base + tid * ITEMS + k;
            const uint32_t three = (uint32_t)buf[p] << 16 | (uint32_t)buf[p + 1] << 8 | buf[p + 2];
            key[k] = p < n ? (three * 2654435761u) >> (32 - HASH_BITS) : (1u << HASH_BITS);  // past the end: sorts last
            pos[k] = (uint16_t)p;
        }
        Sort(sort_tmp).Sort(key, pos, 0, HASH_BITS + 1);  // stable: equal hashes stay in position order
        for (int k = 0; k < ITEMS; ++k) {
            chunk_hash[tid * ITEMS + k] = key[k];
            chunk_pos[tid * ITEMS + k] = pos[k];
        }
        __syncthreads();
        for (int k = 0; k < ITEMS; ++k) {
            const int r = tid * ITEMS + k;
            const uint32_t h = key[k];
            if (h >> HASH_BITS) continue;
            prev[pos[k]] = (r > 0 && chunk_hash[r - 1] == h) ? chunk_pos[r - 1] : head[h];
        }
        __syncthreads();
        for (int k = 0; k < ITEMS; ++k) {
            const int r = tid * ITEMS + k;
            const uint32_t h = key[k];
            if (!(h >> HASH_BITS) && (r == CHUNK - 1 || chunk_hash[r + 1] != h)) head[h] = pos[k];
        }
        __syncthreads();
    }

    // ---- 3. longest match at every position (code[] takes over the phase 2 scratch)
    for (int p = tid; p < n; p += MEMBER_THREADS) {
        const int limit = min(MAX_MATCH, n - p);
        int best = 0, best_dist = 0;
        if (limit >= 3) {
            int q = prev[p];
            for (int d = 0; d < CHAIN_DEPTH && q != NONE && p - q <= WINDOW; ++d) {
                int l = 0;
                while (l < limit && buf[q + l] == buf[p + l]) ++l;
                if (l > best) {
                    best = l;
                    best_dist = p - q;
                    if (l == limit) break;
                }
                q = prev[q];
            }
            if (best < 3 || (best == 3 && best_dist > FAR_MATCH3)) best = 0;
        }
        code[p] = (uint16_t)best;
        dist[p] = (uint16_t)best_dist;
    }
    __syncthreads();

    // ---- 4. greedy parse in warp 0: code[p] becomes SEL | IS_MATCH | length, SEL | literal byte, or 0
    if (warp == 0) {
        int cur = 0;
        for (int base = 0; base < n; base += 32) {
            const int p = base + lane;
            const int len = p < n ? code[p] : 0;
            const int nx = p + max(len, 1);
            bool sel = false;
            while (cur < base + 32 && cur < n) {
                sel |= lane == cur - base;
                cur = __shfl_sync(0xffffffffu, nx, cur - base);
            }
            if (p < n) code[p] = sel ? (uint16_t)(SEL | (len ? IS_MATCH | len : buf[p])) : 0;
        }
    }
    __syncthreads();

    // ---- 5. histograms
    for (int p = tid; p < n; p += MEMBER_THREADS) {
        const int c = code[p];
        if (!(c & SEL)) continue;
        if (c & IS_MATCH) {
            int idx, nb, ex, dc;
            length_code(c & 0x1ff, idx, nb, ex);
            dist_code(dist[p], dc, nb, ex);
            atomicAdd(&s.lit_freq[257 + idx], 1u);
            atomicAdd(&s.dist_freq[dc], 1u);
        } else {
            atomicAdd(&s.lit_freq[c & 0xff], 1u);
        }
    }
    __syncthreads();

    // ---- 6. codes: literal/length on warp 0, distance on warp 1, then the code-length code on thread 0
    if (tid == 0) force_two(s.lit_freq, N_LIT);
    if (tid == 32) force_two(s.dist_freq, N_DIST);
    __syncthreads();
    rank_sort(s.lit_freq, N_LIT, s.lit_sorted, 0, MEMBER_THREADS / 2);
    rank_sort(s.dist_freq, N_DIST, s.dist_sorted, MEMBER_THREADS / 2, MEMBER_THREADS / 2);
    __syncthreads();
    if (tid == 0) {
        huffman_lengths(s.lit_freq, s.lit_sorted, n_used(s.lit_freq, N_LIT), 15, s.lit_len, N_LIT, s.huff_scratch[0]);
        canonical_codes(s.lit_len, N_LIT, s.lit_code);
    } else if (tid == 32) {
        huffman_lengths(s.dist_freq, s.dist_sorted, n_used(s.dist_freq, N_DIST), 15, s.dist_len, N_DIST, s.huff_scratch[1]);
        canonical_codes(s.dist_len, N_DIST, s.dist_code);
    }
    __syncthreads();
    if (tid == 0) {
        int hlit = N_LIT, hdist = N_DIST;
        while (hlit > 257 && !s.lit_len[hlit - 1]) --hlit;
        while (hdist > 1 && !s.dist_len[hdist - 1]) --hdist;
        // run-length code of the hlit + hdist lengths (runs may cross from one table into the other, RFC 1951 3.2.7)
        const int total = hlit + hdist;
        auto length_at = [&](int i) { return i < hlit ? s.lit_len[i] : s.dist_len[i - hlit]; };
        int m = 0;
        for (int i = 0; i < N_CL; ++i) s.cl_freq[i] = 0;
        for (int i = 0; i < total;) {
            const int v = length_at(i);
            int run = 1;
            while (i + run < total && length_at(i + run) == v) ++run;
            i += run;
            if (v == 0) {
                for (; run >= 11; m++) {
                    const int r = min(run, 138);
                    s.rle_sym[m] = 18, s.rle_extra[m] = (uint8_t)(r - 11), run -= r;
                }
                if (run >= 3) s.rle_sym[m] = 17, s.rle_extra[m++] = (uint8_t)(run - 3), run = 0;
            } else {
                s.rle_sym[m] = (uint8_t)v, s.rle_extra[m++] = 0, --run;
                for (; run >= 3; m++) {
                    const int r = min(run, 6);
                    s.rle_sym[m] = 16, s.rle_extra[m] = (uint8_t)(r - 3), run -= r;
                }
            }
            for (; run > 0; --run) s.rle_sym[m] = (uint8_t)v, s.rle_extra[m++] = 0;
        }
        for (int i = 0; i < m; ++i) ++s.cl_freq[s.rle_sym[i]];
        force_two(s.cl_freq, N_CL);
        int used = 0;
        for (int i = 0; i < N_CL; ++i)
            if (s.cl_freq[i]) {
                int j = used++;  // insertion sort by (frequency, symbol)
                for (; j > 0 && s.cl_freq[s.cl_sorted[j - 1]] > s.cl_freq[i]; --j) s.cl_sorted[j] = s.cl_sorted[j - 1];
                s.cl_sorted[j] = (uint16_t)i;
            }
        huffman_lengths(s.cl_freq, s.cl_sorted, used, 7, s.cl_len, N_CL, s.huff_scratch[0]);
        canonical_codes(s.cl_len, N_CL, s.cl_code);
        int hclen = N_CL;
        while (hclen > 4 && !s.cl_len[kClOrder[hclen - 1]]) --hclen;
        int bits = 3 + 5 + 5 + 4 + 3 * hclen;
        for (int i = 0; i < m; ++i) {
            const int sym = s.rle_sym[i];
            bits += s.cl_len[sym] + (sym == 16 ? 2 : sym == 17 ? 3 : sym == 18 ? 7 : 0);
        }
        s.n_rle = m, s.hlit = hlit, s.hdist = hdist, s.hclen = hclen, s.header_bits = bits;
    }

    // ---- 7. bit counts of each thread's contiguous range of positions, exclusive scan
    const int per = (n + MEMBER_THREADS - 1) / MEMBER_THREADS;
    const int lo = min(n, tid * per), hi = min(n, lo + per);
    __syncthreads();
    int mine = 0;
    for (int p = lo; p < hi; ++p) {
        const int c = code[p];
        if (!(c & SEL)) continue;
        if (c & IS_MATCH) {
            int idx, nb, ex, dc, dnb;
            length_code(c & 0x1ff, idx, nb, ex);
            dist_code(dist[p], dc, dnb, ex);
            mine += s.lit_len[257 + idx] + nb + s.dist_len[dc] + dnb;
        } else {
            mine += s.lit_len[c & 0xff];
        }
    }
    int incl = mine;
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) s.warp_sum[warp] = incl;
    __syncthreads();
    int before = incl - mine, body = 0;
    for (int w = 0; w < MEMBER_THREADS / 32; ++w) {
        before += w < warp ? s.warp_sum[w] : 0;
        body += s.warp_sum[w];
    }
    body += s.lit_len[256];
    const int header_bits = s.header_bits;
    const int dyn_bytes = (header_bits + body + 7) / 8;
    const bool stored = n + 5 <= dyn_bytes;
    const int deflate_bytes = stored ? n + 5 : dyn_bytes;

    if (!stored) {  // the member's bytes now live in code[] and src: buf becomes the bit stream
        for (int i = tid; i < SLOT / 4; i += MEMBER_THREADS) words[i] = 0;
        __syncthreads();
        if (tid == 0) {
            BitWriter bw(words, 0);
            bw.put(1, 1);  // BFINAL
            bw.put(2, 2);  // BTYPE 10: dynamic Huffman codes
            bw.put(s.hlit - 257, 5);
            bw.put(s.hdist - 1, 5);
            bw.put(s.hclen - 4, 4);
            for (int i = 0; i < s.hclen; ++i) bw.put(s.cl_len[kClOrder[i]], 3);
            for (int i = 0; i < s.n_rle; ++i) {
                const int sym = s.rle_sym[i];
                bw.put(s.cl_code[sym], s.cl_len[sym]);
                if (sym >= 16) bw.put(s.rle_extra[i], sym == 16 ? 2 : sym == 17 ? 3 : 7);
            }
            bw.flush();
            BitWriter eob(words, header_bits + body - s.lit_len[256]);
            eob.put(s.lit_code[256], s.lit_len[256]);
            eob.flush();
        }
        BitWriter bw(words, header_bits + before);
        for (int p = lo; p < hi; ++p) {
            const int c = code[p];
            if (!(c & SEL)) continue;
            if (c & IS_MATCH) {
                int idx, nb, ex, dc, dnb, dex;
                length_code(c & 0x1ff, idx, nb, ex);
                dist_code(dist[p], dc, dnb, dex);
                bw.put(s.lit_code[257 + idx], s.lit_len[257 + idx]);
                bw.put(ex, nb);
                bw.put(s.dist_code[dc], s.dist_len[dc]);
                bw.put(dex, dnb);
            } else {
                bw.put(s.lit_code[c & 0xff], s.lit_len[c & 0xff]);
            }
        }
        bw.flush();
        __syncthreads();
    }

    // ---- the member: gzip header with the BC subfield, DEFLATE data, CRC32, ISIZE
    const int size = HEADER_BYTES + deflate_bytes + TRAILER_BYTES;
    for (int i = tid; i < size; i += MEMBER_THREADS) {
        uint8_t b;
        if (i < HEADER_BYTES) {
            constexpr uint8_t fixed[16] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0};
            b = i < 16 ? fixed[i] : (uint8_t)((size - 1) >> (8 * (i - 16)));
        } else if (i < HEADER_BYTES + deflate_bytes) {
            const int j = i - HEADER_BYTES;
            if (!stored) {
                b = buf[j];
            } else if (j == 0) {
                b = 1;  // BFINAL, BTYPE 00, padding to the byte
            } else if (j < 5) {
                b = (uint8_t)((j < 3 ? n : ~n) >> (8 * ((j - 1) & 1)));  // LEN, NLEN
            } else {
                b = src[j - 5];
            }
        } else {
            const int j = i - HEADER_BYTES - deflate_bytes;
            b = (uint8_t)((j < 4 ? crc : (uint32_t)n) >> (8 * (j & 3)));
        }
        slot[i] = b;
    }
    if (tid == 0) sizes[member] = size;
}

// offsets[0..n] = exclusive prefix sums of the member sizes (one CTA)
__global__ void __launch_bounds__(SCAN_THREADS) bgzf_scan_kernel(const int* __restrict__ sizes, int64_t n,
                                                                 int64_t* __restrict__ offsets) {
    __shared__ int64_t warp_sum[SCAN_THREADS / 32];
    __shared__ int64_t carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) carry = 0;
    __syncthreads();
    for (int64_t base = 0; base < n; base += SCAN_THREADS) {
        const int64_t v = base + tid < n ? sizes[base + tid] : 0;
        int64_t incl = v;
        for (int o = 1; o < 32; o <<= 1) {
            const int64_t u = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += u;
        }
        if (lane == 31) warp_sum[warp] = incl;
        __syncthreads();
        int64_t before = carry + incl - v, total = carry;
        for (int w = 0; w < SCAN_THREADS / 32; ++w) {
            before += w < warp ? warp_sum[w] : 0;
            total += warp_sum[w];
        }
        if (base + tid < n) offsets[base + tid] = before;
        __syncthreads();
        if (tid == 0) carry = total;
        __syncthreads();
    }
    if (tid == 0) offsets[n] = carry;
}

__global__ void __launch_bounds__(COPY_THREADS) bgzf_copy_kernel(const uint8_t* __restrict__ slots,
                                                                 const int64_t* __restrict__ offsets,
                                                                 uint8_t* __restrict__ out) {
    const int64_t member = blockIdx.x;
    const uint8_t* from = slots + member * SLOT;
    uint8_t* to = out + offsets[member];
    const int size = (int)(offsets[member + 1] - offsets[member]);
    for (int i = threadIdx.x; i < size; i += COPY_THREADS) to[i] = from[i];
}

struct Layout {
    size_t sizes, slots, prev, dist, total;
};

Layout layout(int64_t in_bytes) {
    const int64_t members = (in_bytes + MEMBER_IN - 1) / MEMBER_IN;
    auto up = [](size_t x) { return (x + 255) & ~(size_t)255; };
    Layout l;
    l.sizes = 0;
    l.slots = up(members * sizeof(int));
    l.prev = l.slots + members * (size_t)SLOT;
    l.dist = l.prev + up(members * (size_t)MEMBER_IN * 2);
    l.total = l.dist + up(members * (size_t)MEMBER_IN * 2);
    return l;
}

}  // namespace

extern "C" {

size_t b200_bgzf_workspace_bytes(int64_t in_bytes) { return in_bytes > 0 ? layout(in_bytes).total : 0; }

int b200_bgzf_compress(const uint8_t* in, int64_t in_bytes, uint8_t* out, int64_t* out_offsets, void* workspace,
                       size_t workspace_bytes, void* stream) {
    B200_REQUIRE(in_bytes >= 0, "bgzf_compress: negative input size %lld", (long long)in_bytes);
    B200_REQUIRE(out_offsets, "bgzf_compress: null out_offsets");
    cudaStream_t st = (cudaStream_t)stream;
    if (in_bytes == 0) {
        B200_CHECK_CUDA(cudaMemsetAsync(out_offsets, 0, sizeof(int64_t), st));
        return 0;
    }
    B200_REQUIRE(in && out && workspace, "bgzf_compress: null pointer argument");
    const int64_t members = (in_bytes + MEMBER_IN - 1) / MEMBER_IN;
    B200_REQUIRE(members < (1ll << 31), "bgzf_compress: %lld members exceed one launch", (long long)members);
    const Layout l = layout(in_bytes);
    B200_REQUIRE(workspace_bytes >= l.total, "bgzf_compress: workspace has %zu bytes, %zu needed", workspace_bytes, l.total);
    uint8_t* ws = (uint8_t*)workspace;
    static_assert(MEMBER_SMEM <= 227 * 1024, "shared memory of the member kernel");
    B200_CHECK_CUDA(cudaFuncSetAttribute(bgzf_member_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)MEMBER_SMEM));
    bgzf_member_kernel<<<(unsigned)members, MEMBER_THREADS, MEMBER_SMEM, st>>>(
        in, in_bytes, ws + l.slots, (int*)(ws + l.sizes), (uint16_t*)(ws + l.prev), (uint16_t*)(ws + l.dist));
    bgzf_scan_kernel<<<1, SCAN_THREADS, 0, st>>>((const int*)(ws + l.sizes), members, out_offsets);
    bgzf_copy_kernel<<<(unsigned)members, COPY_THREADS, 0, st>>>(ws + l.slots, out_offsets, out);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // extern "C"
