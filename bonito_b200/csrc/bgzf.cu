// BGZF compression (SAM specification section 4.1) for BAM output: one CTA per member of 65280 input bytes; and BGZF
// decompression for BAM input: one warp per member (inflate_member, further down).
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

// the order of the code-length code's lengths in a dynamic block header (RFC 1951 section 3.2.7)
__host__ __device__ __forceinline__ int cl_order(int i) {
    constexpr uint8_t order[N_CL] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
    return order[i];
}

using Sort = cub::BlockRadixSort<uint32_t, MEMBER_THREADS, ITEMS, uint16_t>;

// The DEFLATE length and distance codes (RFC 1951 section 3.2.5), shared by the compressor and the inflater.
// literal/length symbol - 257 -> base length, extra bits
__host__ __device__ __forceinline__ void length_base(int idx, int& base, int& nbits) {
    if (idx == 28) {
        base = MAX_MATCH, nbits = 0;
    } else if (idx < 8) {
        base = 3 + idx, nbits = 0;
    } else {
        nbits = idx / 4 - 1;
        base = 3 + ((4 + (idx & 3)) << nbits);
    }
}

// distance symbol -> base distance, extra bits
__host__ __device__ __forceinline__ void dist_base(int code, int& base, int& nbits) {
    if (code < 4) {
        base = 1 + code, nbits = 0;
    } else {
        nbits = code / 2 - 1;
        base = 1 + ((2 + (code & 1)) << nbits);
    }
}

// length 3..258 -> literal/length symbol - 257, extra bits, extra value
__device__ __forceinline__ void length_code(int len, int& idx, int& nbits, int& extra) {
    const int v = len - 3;
    if (len == MAX_MATCH) {
        idx = 28;
    } else if (v < 8) {
        idx = v;
    } else {
        const int lg = 31 - __clz(v);
        idx = 4 * (lg - 1) + ((v >> (lg - 2)) & 3);
    }
    int base;
    length_base(idx, base, nbits);
    extra = len - base;
}

// distance 1..32768 -> distance symbol, extra bits, extra value
__device__ __forceinline__ void dist_code(int dist, int& code, int& nbits, int& extra) {
    const int v = dist - 1;
    if (v < 4) {
        code = v;
    } else {
        const int lg = 31 - __clz(v);
        code = 2 * lg + ((v >> (lg - 1)) & 1);
    }
    int base;
    dist_base(code, base, nbits);
    extra = dist - base;
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

// The CRC32 of n bytes from `parts` slices taken in parallel: crc_table_entry() and crc_powers() fill the tables once,
// crc_part() gives slice `part`'s contribution, and crc_finish() turns the XOR of every part into the CRC32.
__device__ __forceinline__ uint32_t crc_table_entry(uint32_t c) {
    for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ CRC_POLY : c >> 1;
    return c;
}

// x2n[k] = x^(2^k), k < 32 (one thread)
__device__ void crc_powers(uint32_t* x2n) {
    uint32_t x = 1u << 30;  // x^1
    for (int k = 0; k < 32; ++k) {
        x2n[k] = x;
        x = crc_multmod(x, x);
    }
}

// the slice's CRC register from zero, then shifted over the bytes after it
__device__ uint32_t crc_part(const uint8_t* buf, int n, int part, int parts, const uint32_t* table, const uint32_t* x2n) {
    const int per = (n + parts - 1) / parts;
    const int lo = min(n, part * per), hi = min(n, lo + per);
    uint32_t c = 0;
    for (int i = lo; i < hi; ++i) c = table[(c ^ buf[i]) & 0xff] ^ (c >> 8);
    return crc_multmod(crc_shift_op((uint32_t)(n - hi), x2n), c);
}

__device__ __forceinline__ uint32_t crc_finish(uint32_t parts_xor, int n, const uint32_t* x2n) {
    return parts_xor ^ crc_multmod(crc_shift_op((uint32_t)n, x2n), 0xffffffffu) ^ 0xffffffffu;
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
    if (tid < 256) crc_table[tid] = crc_table_entry(tid);
    if (tid == 0) crc_powers(s.x2n);
    __syncthreads();
    s.crc_part[tid] = crc_part(buf, n, tid, MEMBER_THREADS, crc_table, s.x2n);
    __syncthreads();
    if (warp == 0) {
        uint32_t c = 0;
        for (int i = lane; i < MEMBER_THREADS; i += 32) c ^= s.crc_part[i];
        for (int o = 16; o; o >>= 1) c ^= __shfl_xor_sync(0xffffffffu, c, o);
        if (lane == 0) s.crc_part[0] = crc_finish(c, n, s.x2n);
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
        while (hclen > 4 && !s.cl_len[cl_order(hclen - 1)]) --hclen;
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
            for (int i = 0; i < s.hclen; ++i) bw.put(s.cl_len[cl_order(i)], 3);
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

// ------------------------------------------------------------------------------------------------ inflate
// RFC 1951 inflation of one BGZF member, written once for the device (a warp, all lanes in lockstep) and the host (one
// "lane"): every lane reads the same bits and decodes the same symbols, so control flow stays uniform; lane 0 writes the
// literals, and the lanes share the Huffman table fills, match copies and stored-block copies.  A member's window is its
// own output (BGZF members share no history).  Every input read is bounded by in_len (bits peeked past it read as
// zeros; consuming them is an error), every output write by out_len.
constexpr int LIT_BITS = 10, DIST_BITS = 8;  // primary lookup bits; longer codes are decoded canonically
constexpr int N_LIT_SYMS = 288, N_DIST_SYMS = 32, MAX_BITS = 15;

struct InflateScratch {
    uint16_t lit_lut[1 << LIT_BITS];    // (symbol << 4) | length, 0 when the code is longer than LIT_BITS or unused
    uint16_t dist_lut[1 << DIST_BITS];  // the same; first the code-length code's table
    uint16_t lit_sym[N_LIT_SYMS];       // symbols in canonical order
    uint16_t dist_sym[N_DIST_SYMS];
    uint16_t lit_count[MAX_BITS + 1];   // codes of each length
    uint16_t dist_count[MAX_BITS + 1];
    uint16_t first[MAX_BITS + 1];       // while a table is built: the first code of each length,
    uint16_t start[MAX_BITS + 1];       // the canonical index of that code,
    uint16_t fill[MAX_BITS + 1];        // and the next free canonical index
    uint8_t lens[N_LIT_SYMS + N_DIST_SYMS];
};

__host__ __device__ __forceinline__ void lanes_sync(int lanes) {
#ifdef __CUDA_ARCH__
    __syncwarp(lanes >= 32 ? 0xffffffffu : (1u << lanes) - 1);
#endif
}

__host__ __device__ __forceinline__ uint8_t load_in(const uint8_t* p) {
#ifdef __CUDA_ARCH__
    return __ldg(p);
#else
    return *p;
#endif
}

__host__ __device__ __forceinline__ uint32_t reverse_bits(uint32_t v, int n) {
#ifdef __CUDA_ARCH__
    return __brev(v) >> (32 - n);
#else
    uint32_t r = 0;
    for (int i = 0; i < n; ++i, v >>= 1) r = r << 1 | (v & 1);
    return r;
#endif
}

struct Huff {
    uint16_t* lut;
    uint16_t* sym;
    uint16_t* count;
    int bits;
};

// Canonical code of lens[0..n): count[], sym[] and the primary table.  Returns 0 for a complete code or no code at all,
// 1 for the one incomplete code DEFLATE allows (a single code of length 1, when allow_single), -1 otherwise.  The counts
// and canonical offsets live in the warp's shared scratch, written by lane 0; the lanes then fill the table from the
// canonical order, each its own symbols.
__host__ __device__ int huff_build(const uint8_t* lens, int n, const Huff& h, bool allow_single, InflateScratch& s,
                                   int lane, int lanes) {
    lanes_sync(lanes);  // every lane is done with the table this one replaces
    if (lane == 0) {
        for (int l = 0; l <= MAX_BITS; ++l) h.count[l] = 0;
        for (int i = 0; i < n; ++i) ++h.count[lens[i]];
    }
    lanes_sync(lanes);
    const int used = n - h.count[0];
    int left = 1;
    for (int l = 1; l <= MAX_BITS; ++l) {
        left = (left << 1) - h.count[l];
        if (left < 0) return -1;  // over-subscribed
    }
    int status = 0;
    if (left > 0 && used > 0) {
        if (!(allow_single && used == 1 && h.count[1] == 1)) return -1;
        status = 1;
    }
    if (lane == 0) {
        int code = 0, pos = 0;
        for (int l = 1; l <= MAX_BITS; ++l) {
            code = (code + (l > 1 ? h.count[l - 1] : 0)) << 1;
            s.first[l] = (uint16_t)code;
            s.start[l] = s.fill[l] = (uint16_t)pos;
            pos += h.count[l];
        }
        for (int i = 0; i < n; ++i)
            if (lens[i]) h.sym[s.fill[lens[i]]++] = (uint16_t)i;
    }
    const int size = 1 << h.bits;
    for (int k = lane; k < size; k += lanes) h.lut[k] = 0;
    lanes_sync(lanes);
    for (int i = lane; i < used; i += lanes) {
        const int sym = h.sym[i], l = lens[sym];
        if (l > h.bits) break;  // canonical order: every later code is as long
        const int code = s.first[l] + i - s.start[l];
        const uint16_t e = (uint16_t)(sym << 4 | l);
        for (int k = (int)reverse_bits(code, l); k < size; k += 1 << l) h.lut[k] = e;
    }
    lanes_sync(lanes);
    return status;
}

struct BitReader {
    const uint8_t* in;
    int len, pos, cnt;  // pos: next byte to load (runs past len when zeros are peeked)
    uint64_t buf;
    __host__ __device__ void refill() {
        while (cnt <= 56) {
            buf |= (uint64_t)(pos < len ? load_in(in + pos) : 0) << cnt;
            ++pos;
            cnt += 8;
        }
    }
    __host__ __device__ __forceinline__ uint32_t take(int n) {
        const uint32_t v = (uint32_t)(buf & ((1ull << n) - 1));
        buf >>= n;
        cnt -= n;
        return v;
    }
    __host__ __device__ __forceinline__ bool overrun() const { return (int64_t)pos * 8 - cnt > (int64_t)len * 8; }
    // more than the 8 bytes the buffer can hold peeked past the end: the bits consumed have already passed it
    __host__ __device__ __forceinline__ bool far_overrun() const { return pos > len + 8; }
};

// one symbol, with at least MAX_BITS bits in the buffer; -1 for bits that match no code
__host__ __device__ __forceinline__ int huff_decode(BitReader& br, const Huff& h) {
    const uint16_t e = h.lut[br.buf & ((1u << h.bits) - 1)];
    if (e) {
        br.take(e & 15);
        return e >> 4;
    }
    int code = 0, first = 0, index = 0;  // canonical decode, one bit at a time
    for (int l = 1; l <= MAX_BITS; ++l) {
        code |= (int)((br.buf >> (l - 1)) & 1);
        const int c = h.count[l];
        if (code - c < first) {
            br.take(l);
            return h.sym[index + code - first];
        }
        index += c;
        first = (first + c) << 1;
        code <<= 1;
    }
    return -1;
}

// The dynamic block header: code lengths into lens[], then both tables.
__host__ __device__ int read_dynamic(BitReader& br, InflateScratch& s, const Huff& lit, const Huff& dist, int lane,
                                     int lanes) {
    br.refill();
    const int hlit = (int)br.take(5) + 257, hdist = (int)br.take(5) + 1, hclen = (int)br.take(4) + 4;
    if (hlit > 286 || hdist > 30) return B200_INFLATE_CODE_LENGTHS;
    lanes_sync(lanes);  // every lane is past the previous block's lengths
    if (lane == 0)
        for (int i = 0; i < N_CL; ++i) s.lens[i] = 0;
    br.refill();  // 3 * 19 bits: two refills
    for (int i = 0; i < hclen; ++i) {
        if (i == 16) br.refill();
        const uint8_t v = (uint8_t)br.take(3);
        if (lane == 0) s.lens[cl_order(i)] = v;
    }
    const Huff cl = {s.dist_lut, s.dist_sym, s.dist_count, 7};
    if (huff_build(s.lens, N_CL, cl, false, s, lane, lanes) != 0) return B200_INFLATE_CODE_LENGTHS;
    const int total = hlit + hdist;
    for (int i = 0; i < total;) {
        br.refill();
        if (br.far_overrun()) return B200_INFLATE_TRUNCATED;
        const int sym = huff_decode(br, cl);
        if (sym < 0) return B200_INFLATE_CODE_LENGTHS;
        if (sym < 16) {
            if (lane == 0) s.lens[i] = (uint8_t)sym;
            ++i;
            continue;
        }
        int len = 0, rep;
        if (sym == 16) {
            if (i == 0) return B200_INFLATE_REPEAT;
            lanes_sync(lanes);
            len = s.lens[i - 1];
            rep = 3 + (int)br.take(2);
        } else if (sym == 17) {
            rep = 3 + (int)br.take(3);
        } else {
            rep = 11 + (int)br.take(7);
        }
        if (i + rep > total) return B200_INFLATE_REPEAT;
        if (lane == 0)
            for (int k = 0; k < rep; ++k) s.lens[i + k] = (uint8_t)len;
        i += rep;
    }
    lanes_sync(lanes);
    if (s.lens[256] == 0) return B200_INFLATE_CODE_LENGTHS;  // no end-of-block code
    if (huff_build(s.lens, hlit, lit, true, s, lane, lanes) < 0) return B200_INFLATE_CODE_LENGTHS;
    if (huff_build(s.lens + hlit, hdist, dist, true, s, lane, lanes) < 0) return B200_INFLATE_CODE_LENGTHS;
    return B200_INFLATE_OK;
}

__host__ __device__ int read_fixed(InflateScratch& s, const Huff& lit, const Huff& dist, int lane, int lanes) {
    lanes_sync(lanes);
    if (lane == 0) {
        for (int i = 0; i < N_LIT_SYMS; ++i) s.lens[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8;
        for (int i = 0; i < N_DIST_SYMS; ++i) s.lens[N_LIT_SYMS + i] = 5;
    }
    lanes_sync(lanes);
    const int l = huff_build(s.lens, N_LIT_SYMS, lit, false, s, lane, lanes);
    const int d = huff_build(s.lens + N_LIT_SYMS, N_DIST_SYMS, dist, false, s, lane, lanes);
    return l || d ? B200_INFLATE_CODE_LENGTHS : B200_INFLATE_OK;
}

// Inflates the raw DEFLATE stream in[0..in_len) into exactly out[0..out_len); a B200_INFLATE_* status.  Every lane of
// the group [0, lanes) calls it with the same arguments and gets the same status.
__host__ __device__ int inflate_member(const uint8_t* in, int in_len, uint8_t* out, int out_len, InflateScratch& s,
                                       int lane, int lanes) {
    const Huff lit = {s.lit_lut, s.lit_sym, s.lit_count, LIT_BITS};
    const Huff dist = {s.dist_lut, s.dist_sym, s.dist_count, DIST_BITS};
    BitReader br = {in, in_len, 0, 0, 0};
    int op = 0;
    for (bool last = false; !last;) {
        br.refill();
        if (br.overrun()) return B200_INFLATE_TRUNCATED;
        last = br.take(1);
        const int type = (int)br.take(2);
        if (type == 0) {  // stored: to the byte boundary, LEN, NLEN, LEN bytes
            br.take(br.cnt & 7);
            int bp = br.pos - br.cnt / 8;
            if (bp + 4 > in_len) return B200_INFLATE_TRUNCATED;
            const int n = load_in(in + bp) | load_in(in + bp + 1) << 8;
            const int nn = load_in(in + bp + 2) | load_in(in + bp + 3) << 8;
            if (n != (~nn & 0xffff)) return B200_INFLATE_STORED_LENGTH;
            bp += 4;
            if (n > in_len - bp) return B200_INFLATE_TRUNCATED;
            if (n > out_len - op) return B200_INFLATE_OVERFLOW;
            for (int i = lane; i < n; i += lanes) out[op + i] = load_in(in + bp + i);
            op += n;
            br.pos = bp + n, br.cnt = 0, br.buf = 0;
            continue;
        }
        if (type == 3) return B200_INFLATE_BLOCK_TYPE;
        const int st = type == 1 ? read_fixed(s, lit, dist, lane, lanes) : read_dynamic(br, s, lit, dist, lane, lanes);
        if (st) return st;
        for (;;) {
            br.refill();  // >= 57 bits: a length code, its extra bits, a distance code and its extra bits
            if (br.far_overrun()) return B200_INFLATE_TRUNCATED;
            const int sym = huff_decode(br, lit);
            if (sym < 256) {
                if (sym < 0) return B200_INFLATE_SYMBOL;
                if (op >= out_len) return B200_INFLATE_OVERFLOW;
                if (lane == 0) out[op] = (uint8_t)sym;
                ++op;
                continue;
            }
            if (sym == 256) break;
            if (sym > 285) return B200_INFLATE_SYMBOL;
            int len, nb;
            length_base(sym - 257, len, nb);
            len += (int)br.take(nb);
            const int dsym = huff_decode(br, dist);
            if (dsym < 0 || dsym >= 30) return B200_INFLATE_SYMBOL;
            int d;
            dist_base(dsym, d, nb);
            d += (int)br.take(nb);
            if (d > op) return B200_INFLATE_DISTANCE;
            if (len > out_len - op) return B200_INFLATE_OVERFLOW;
            lanes_sync(lanes);  // the bytes before op are written
            // the match repeats out[op - d, op) with period d, so every byte reads from before op
            const uint8_t* from = out + op - d;
            const int step = lanes % d;
            for (int i = lane, j = lane % d; i < len; i += lanes) {
                out[op + i] = from[j];
                j += step;
                if (j >= d) j -= d;
            }
            op += len;
        }
        if (br.overrun()) return B200_INFLATE_TRUNCATED;
    }
    lanes_sync(lanes);
    return op == out_len ? B200_INFLATE_OK : B200_INFLATE_SHORT;
}

constexpr int INFLATE_WARPS = 4;

// one warp per member; meta[m] = raw DEFLATE start in `in`, its length, output offset, ISIZE, expected CRC32
__global__ void __launch_bounds__(INFLATE_WARPS * 32)
    bgzf_inflate_kernel(const uint8_t* __restrict__ in, int64_t in_bytes, const int64_t* __restrict__ meta, int n_members,
                        uint8_t* __restrict__ out, int64_t out_bytes, int32_t* __restrict__ status) {
    __shared__ InflateScratch scratch[INFLATE_WARPS];
    __shared__ uint32_t crc_table[256], x2n[32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int i = tid; i < 256; i += INFLATE_WARPS * 32) crc_table[i] = crc_table_entry(i);
    if (tid == 0) crc_powers(x2n);
    __syncthreads();
    const int64_t m = (int64_t)blockIdx.x * INFLATE_WARPS + warp;
    if (m >= n_members) return;
    const int64_t* mm = meta + 5 * m;
    const int64_t in_start = mm[0], in_len = mm[1], out_start = mm[2], isize = mm[3];
    const uint32_t crc = (uint32_t)mm[4];
    int st;
    if (in_start < 0 || in_len < 0 || in_len > in_bytes - in_start || isize < 0 || isize > SLOT || out_start < 0 ||
        isize > out_bytes - out_start) {
        st = B200_INFLATE_BOUNDS;
    } else {
        uint8_t* dst = out + out_start;
        st = inflate_member(in + in_start, (int)in_len, dst, (int)isize, scratch[warp], lane, 32);
        if (st == B200_INFLATE_OK) {
            uint32_t c = crc_part(dst, (int)isize, lane, 32, crc_table, x2n);
            for (int o = 16; o; o >>= 1) c ^= __shfl_xor_sync(0xffffffffu, c, o);
            if (crc_finish(c, (int)isize, x2n) != crc) st = B200_INFLATE_CRC;
        }
    }
    if (lane == 0) status[m] = st;
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

int b200_bgzf_decompress(const uint8_t* in, int64_t in_bytes, const int64_t* meta, int n_members, uint8_t* out,
                         int64_t out_bytes, int32_t* status, void* stream) {
    B200_REQUIRE(n_members >= 0 && in_bytes >= 0 && out_bytes >= 0, "bgzf_decompress: negative size");
    if (n_members == 0) return 0;
    B200_REQUIRE(meta && status && (in || in_bytes == 0) && (out || out_bytes == 0), "bgzf_decompress: null pointer argument");
    const unsigned blocks = (unsigned)((n_members + INFLATE_WARPS - 1) / INFLATE_WARPS);
    bgzf_inflate_kernel<<<blocks, INFLATE_WARPS * 32, 0, (cudaStream_t)stream>>>(in, in_bytes, meta, n_members, out, out_bytes,
                                                                               status);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // extern "C"
