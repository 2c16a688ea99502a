// Signal decompression for POD5 input.  POD5 stores each signal row as VBZ: the int16 samples delta-coded from 0 and
// zigzag-coded in 16-bit arithmetic, packed with StreamVByte-16 (svb16) and compressed as one zstd frame.  Two kernels undo
// it, one warp per row in each:
//
//   zstd (RFC 8878), zstd_stream: the lanes walk the same frame, block, literals and sequences headers in lockstep and
//     decode the sequence bit stream together (every lane holds the same states, so nothing has to be broadcast).  They
//     share the work that fans out: the Huffman table fill, the four Huffman literal streams (one lane each), the XXH64
//     accumulators (one lane each), and every literal, match, Raw and RLE copy.  The FSE tables and the Huffman weights are
//     built by lane 0 in the warp's shared scratch.  Matches read back from the stream's own output slot, so no window
//     buffer is needed; the literals of a compressed block are decoded into the end of the slot, where the block's
//     sequences consume them before its output reaches them.
//   svb16, svb16_row: 256 samples per warp step, one key byte (8 samples) per lane; a warp scan of the key bytes'
//     lengths places every lane's data bytes, and a second scan of the lanes' delta sums undoes the delta coding.
//
// Both kernels are __host__ __device__ at their core (lanes == 1 on the host), and every read is bounded by the row's
// input range and every write by its output slot, so a malformed row gets a status code and never faults.
#include "common.cuh"

namespace {

constexpr int ZSTD_WARPS = 4;
constexpr int SVB_WARPS = 4;
constexpr int BLOCK_MAX = 128 * 1024;  // largest block content (and compressed block) of a zstd frame
constexpr int HUF_MAX_BITS = 11;
constexpr int LL_MAX_LOG = 9, ML_MAX_LOG = 9, OF_MAX_LOG = 8, HW_MAX_LOG = 6;
constexpr int LL_MAX_SYM = 35, ML_MAX_SYM = 52, OF_MAX_SYM = 31, HW_MAX_SYM = 255;

struct FseEntry {
    uint16_t base;  // next state = base + the entry's bits
    uint8_t sym, bits;
};

struct HufEntry {
    uint8_t sym, bits;
};

// one warp's tables; the LL / OF / ML tables and the Huffman table persist across the blocks of a frame (Repeat, Treeless)
struct ZstdScratch {
    FseEntry ll[1 << LL_MAX_LOG], ml[1 << ML_MAX_LOG], of[1 << OF_MAX_LOG], hw[1 << HW_MAX_LOG];
    HufEntry huf[1 << HUF_MAX_BITS];
    int16_t norm[HW_MAX_SYM + 1];
    uint16_t next[HW_MAX_SYM + 1];
    uint16_t hstart[256];  // first Huffman table entry of each symbol
    uint8_t weights[256];
};

// the predefined distributions (RFC 8878 section 3.1.1.3.2.2)
__constant__ const int16_t LL_DEFAULT[36] = {4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2,
                                             2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1};
__constant__ const int16_t ML_DEFAULT[53] = {1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1,
                                             1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1,
                                             1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1};
__constant__ const int16_t OF_DEFAULT[29] = {1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1,
                                             1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1};
// literal length and match length codes 16.. / 32.. : baseline and extra bits (codes below are their own value)
__constant__ const int LL_BASE[20] = {16, 18, 20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384,
                                      32768, 65536};
__constant__ const uint8_t LL_BITS[20] = {1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};
__constant__ const int ML_BASE[21] = {35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195,
                                      16387, 32771, 65539};
__constant__ const uint8_t ML_BITS[21] = {1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};

#ifdef __CUDA_ARCH__
#define ZCONST(name) name
#else
#define ZCONST(name) host_##name
#endif
#ifndef __CUDA_ARCH__
// host copies of the tables (the host build decodes with lanes == 1)
const int16_t host_LL_DEFAULT[36] = {4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2,
                                     2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1};
const int16_t host_ML_DEFAULT[53] = {1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1,
                                     1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1};
const int16_t host_OF_DEFAULT[29] = {1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1,
                                     1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1};
const int host_LL_BASE[20] = {16, 18, 20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384,
                              32768, 65536};
const uint8_t host_LL_BITS[20] = {1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};
const int host_ML_BASE[21] = {35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195,
                              16387, 32771, 65539};
const uint8_t host_ML_BITS[21] = {1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};
#endif

__host__ __device__ __forceinline__ void lanes_sync(int lanes) {
#ifdef __CUDA_ARCH__
    __syncwarp(lanes >= 32 ? 0xffffffffu : (1u << lanes) - 1);
#endif
}

// every lane's flag or-ed (lanes is 32 on the device)
__host__ __device__ __forceinline__ int lanes_any(int v) {
#ifdef __CUDA_ARCH__
    return __any_sync(0xffffffffu, v);
#else
    return v;
#endif
}

// lane 0's value on every lane
__host__ __device__ __forceinline__ int from_lane0(int v) {
#ifdef __CUDA_ARCH__
    return __shfl_sync(0xffffffffu, v, 0);
#else
    return v;
#endif
}

__host__ __device__ __forceinline__ uint8_t load_in(const uint8_t* p) {
#ifdef __CUDA_ARCH__
    return __ldg(p);
#else
    return *p;
#endif
}

__host__ __device__ __forceinline__ int highbit(uint32_t v) {  // v > 0
#ifdef __CUDA_ARCH__
    return 31 - __clz(v);
#else
    return 31 - __builtin_clz(v);
#endif
}

__host__ __device__ __forceinline__ uint32_t le16(const uint8_t* p) { return load_in(p) | (uint32_t)load_in(p + 1) << 8; }
__host__ __device__ __forceinline__ uint32_t le24(const uint8_t* p) { return le16(p) | (uint32_t)load_in(p + 2) << 16; }
__host__ __device__ __forceinline__ uint32_t le32(const uint8_t* p) { return le24(p) | (uint32_t)load_in(p + 3) << 24; }

// A zstd backward bit stream (Huffman literal streams, FSE weights, sequences): the stream's bits are read from the top
// (the bit under the final byte's end marker) down to bit 0.  pos = bits not yet read; it goes negative when a malformed
// stream reads past its start, and those bits read as zeros.
struct BackBits {
    const uint8_t* p;
    int64_t len, pos, wlo;  // wlo: first bit of the cached 64-bit window w
    uint64_t w;

    // false for an empty stream or one whose last byte has no end marker
    __host__ __device__ bool init(const uint8_t* in, int64_t n) {
        p = in, len = n, wlo = -128, w = 0;  // the first read loads the window
        if (n <= 0) return false;
        const uint8_t last = load_in(in + n - 1);
        pos = (n - 1) * 8 + (last ? highbit(last) : 0);
        return last != 0;
    }
    // bits [lo, lo + n) of the stream, n <= 32
    __host__ __device__ uint32_t at(int64_t lo, int n) {
        if (n == 0) return 0;
        int shift = 0;
        if (lo < 0) {
            shift = (int)-lo;
            if (shift >= n) return 0;
            n -= shift;
            lo = 0;
        }
        if (lo < wlo || lo + n > wlo + 64) {
            int64_t b = ((lo + n + 7) >> 3) - 8;
            if (b < 0) b = 0;
            w = 0;
            for (int i = 0; i < 8; ++i)
                if (b + i < len) w |= (uint64_t)load_in(p + b + i) << (8 * i);
            wlo = b * 8;
        }
        const uint64_t v = (w >> (lo - wlo)) & ((1ull << n) - 1);
        return (uint32_t)(v << shift);
    }
    __host__ __device__ __forceinline__ uint32_t read(int n) {
        pos -= n;
        return at(pos, n);
    }
    __host__ __device__ __forceinline__ uint32_t peek(int n) { return at(pos - n, n); }
};

// 32 bits of a forward (LSB-first) bit stream from bit `bit`, zeros past n bytes
__host__ __device__ uint32_t fwd_bits(const uint8_t* in, int n, int bit) {
    const int b = bit >> 3;
    uint64_t v = 0;
    for (int i = 0; i < 5; ++i)
        if (b + i < n) v |= (uint64_t)load_in(in + b + i) << (8 * i);
    return (uint32_t)(v >> (bit & 7));
}

// An FSE table description (RFC 8878 section 4.1.1) into norm[0, *nsym): bytes used, or -1.  Lane 0 only.
__host__ __device__ int read_ncount(const uint8_t* in, int n, int max_sym, int max_log, int16_t* norm, int& nsym, int& log) {
    if (n < 1) return -1;
    for (int i = 0; i <= max_sym; ++i) norm[i] = 0;
    int bit = 0;
    log = (int)(fwd_bits(in, n, 0) & 15) + 5;
    bit = 4;
    if (log > max_log) return -1;
    int remaining = (1 << log) + 1, threshold = 1 << log, nb = log + 1, sym = 0;
    bool prev0 = false;
    while (remaining > 1 && sym <= max_sym) {
        if (prev0) {
            for (;;) {
                const int r = (int)(fwd_bits(in, n, bit) & 3);
                bit += 2;
                sym += r;
                if (r != 3) break;
                if (bit > 8 * n) return -1;
            }
            if (sym > max_sym) return -1;
        }
        const uint32_t v = fwd_bits(in, n, bit);
        const int max = (2 * threshold - 1) - remaining;
        int count;
        if ((int)(v & (threshold - 1)) < max) {
            count = (int)(v & (threshold - 1));
            bit += nb - 1;
        } else {
            count = (int)(v & (2 * threshold - 1));
            if (count >= threshold) count -= max;
            bit += nb;
        }
        --count;
        remaining -= count < 0 ? -count : count;
        norm[sym++] = (int16_t)count;
        prev0 = count == 0;
        while (remaining < threshold && threshold > 1) {
            --nb;
            threshold >>= 1;
        }
        if (bit > 8 * n) return -1;
    }
    if (remaining != 1 || bit > 8 * n) return -1;
    nsym = sym;
    return (bit + 7) >> 3;
}

// The decoding table of a distribution (RFC 8878 section 4.1.1): 0, or -1 for one that does not fill the table.  Lane 0.
__host__ __device__ int fse_build(const int16_t* norm, int nsym, int log, FseEntry* t, uint16_t* next) {
    const int size = 1 << log;
    int high = size - 1;
    for (int s = 0; s < nsym; ++s) {
        if (norm[s] == -1) {
            if (high < 0) return -1;
            t[high--].sym = (uint8_t)s;
            next[s] = 1;
        } else {
            next[s] = (uint16_t)norm[s];
        }
    }
    const int step = (size >> 1) + (size >> 3) + 3, mask = size - 1;
    int pos = 0, placed = 0;
    for (int s = 0; s < nsym; ++s)
        for (int i = 0; i < norm[s]; ++i) {
            if (++placed > high + 1) return -1;
            t[pos].sym = (uint8_t)s;
            do pos = (pos + step) & mask;
            while (pos > high);
        }
    if (pos != 0 || placed != high + 1) return -1;
    for (int u = 0; u < size; ++u) {
        const int s = t[u].sym, ns = next[s]++;
        const int bits = log - highbit((uint32_t)ns);
        t[u].bits = (uint8_t)bits;
        t[u].base = (uint16_t)((ns << bits) - size);
    }
    return 0;
}

// The Huffman tree description at in[0, n) (RFC 8878 section 4.2.1) into s.huf: bytes used, or -1; *bits = table log.
__host__ __device__ int read_huffman(const uint8_t* in, int n, ZstdScratch& s, int& bits, int lane, int lanes) {
    int used = -1, nw = 0, log = 0;
    lanes_sync(lanes);  // every lane is done with the table this one replaces
    if (lane == 0) {
        do {
            if (n < 1) break;
            const int hb = load_in(in);
            if (hb >= 128) {  // direct: 4 bits per weight
                nw = hb - 127;
                const int bytes = (nw + 1) / 2;
                if (1 + bytes > n) break;
                for (int i = 0; i < nw; ++i) {
                    const uint8_t b = load_in(in + 1 + i / 2);
                    s.weights[i] = (uint8_t)(i & 1 ? b & 15 : b >> 4);
                }
                used = 1 + bytes;
            } else {  // FSE-coded, two interleaved states
                if (hb == 0 || 1 + hb > n) break;
                int nsym, alog;
                const int c = read_ncount(in + 1, hb, HW_MAX_SYM, HW_MAX_LOG, s.norm, nsym, alog);
                if (c < 0 || fse_build(s.norm, nsym, alog, s.hw, s.next) < 0) break;
                BackBits br;
                if (!br.init(in + 1 + c, hb - c)) break;
                int s1 = (int)br.read(alog), s2 = (int)br.read(alog);
                bool ok = true;
                for (;;) {
                    if (nw >= 255) { ok = false; break; }
                    s.weights[nw++] = s.hw[s1].sym;
                    s1 = s.hw[s1].base + (int)br.read(s.hw[s1].bits);
                    if (br.pos < 0) {
                        if (nw >= 255) { ok = false; break; }
                        s.weights[nw++] = s.hw[s2].sym;
                        break;
                    }
                    if (nw >= 255) { ok = false; break; }
                    s.weights[nw++] = s.hw[s2].sym;
                    s2 = s.hw[s2].base + (int)br.read(s.hw[s2].bits);
                    if (br.pos < 0) {
                        if (nw >= 255) { ok = false; break; }
                        s.weights[nw++] = s.hw[s1].sym;
                        break;
                    }
                }
                if (!ok) break;
                used = 1 + hb;
            }
            // the implied last weight completes the code to a power of two
            uint32_t total = 0;
            int rank1 = 0;
            bool ok = true;
            for (int i = 0; i < nw; ++i) {
                const int w = s.weights[i];
                if (w > HUF_MAX_BITS + 1) ok = false;
                else if (w) total += 1u << (w - 1);
                rank1 += w == 1;
            }
            if (!ok || total == 0) { used = -1; break; }
            log = highbit(total) + 1;
            const uint32_t rest = (1u << log) - total;
            if (log > HUF_MAX_BITS || (rest & (rest - 1))) { used = -1; break; }
            const int lastw = highbit(rest) + 1;
            s.weights[nw] = (uint8_t)lastw;
            rank1 += lastw == 1;
            if (rank1 < 2 || (rank1 & 1)) { used = -1; break; }
            // entries of weight w: 2^(w-1) each, weights ascending, symbols ascending within a weight
            int start[HUF_MAX_BITS + 2], cnt[HUF_MAX_BITS + 2];
            for (int w = 0; w <= HUF_MAX_BITS + 1; ++w) cnt[w] = 0;
            for (int i = 0; i <= nw; ++i) ++cnt[s.weights[i]];
            int p = 0;
            for (int w = 1; w <= HUF_MAX_BITS + 1; ++w) {
                start[w] = p;
                p += cnt[w] << (w - 1);
            }
            for (int i = 0; i <= nw; ++i) {
                const int w = s.weights[i];
                if (w) {
                    s.hstart[i] = (uint16_t)start[w];
                    start[w] += 1 << (w - 1);
                }
            }
        } while (false);
    }
    used = from_lane0(used);
    if (used < 0) return -1;
    nw = from_lane0(nw);
    log = from_lane0(log);
    lanes_sync(lanes);
    for (int i = lane; i <= nw; i += lanes) {
        const int w = s.weights[i];
        if (!w) continue;
        const HufEntry e = {(uint8_t)i, (uint8_t)(log + 1 - w)};
        for (int k = 0, p = s.hstart[i]; k < 1 << (w - 1); ++k) s.huf[p + k] = e;
    }
    lanes_sync(lanes);
    bits = log;
    return used;
}

// one Huffman-coded literal stream of exactly n symbols, consuming the stream exactly
__host__ __device__ bool huf_stream(const uint8_t* in, int64_t len, uint8_t* dst, int n, const HufEntry* t, int bits) {
    BackBits br;
    if (!br.init(in, len)) return false;
    for (int i = 0; i < n; ++i) {
        const HufEntry e = t[br.peek(bits)];
        dst[i] = e.sym;
        br.pos -= e.bits;
        if (br.pos < 0) return false;
    }
    return br.pos == 0;
}

// dst[0, n) = src[0, n) where dst <= src (the regions may overlap): every group of lanes loads before it stores
__host__ __device__ void copy_down(uint8_t* dst, const uint8_t* src, int64_t n, int lane, int lanes) {
    for (int64_t base = 0; base < n; base += lanes) {
        const int64_t i = base + lane;
        const uint8_t v = i < n ? src[i] : 0;
        lanes_sync(lanes);
        if (i < n) dst[i] = v;
    }
    lanes_sync(lanes);
}

// a match of len bytes at distance d <= op; the bytes before out + op are written
__host__ __device__ void copy_match(uint8_t* out, int64_t op, int64_t d, int64_t len, int lane, int lanes) {
    const uint8_t* from = out + op - d;
    const int64_t step = lanes % d;
    int64_t j = lane % d;
    for (int64_t i = lane; i < len; i += lanes) {
        out[op + i] = from[j];
        j += step;
        if (j >= d) j -= d;
    }
    lanes_sync(lanes);
}

enum TableKind { LL = 0, OF = 1, ML = 2 };

// One symbol compression mode's table (mode: 0 predefined, 1 RLE, 2 FSE, 3 repeat): bytes used, or -1.
__host__ __device__ int seq_table(int kind, int mode, const uint8_t* in, int n, ZstdScratch& s, int& log, bool& have,
                                  int lane, int lanes) {
    FseEntry* t = kind == LL ? s.ll : kind == OF ? s.of : s.ml;
    const int max_sym = kind == LL ? LL_MAX_SYM : kind == OF ? OF_MAX_SYM : ML_MAX_SYM;
    const int max_log = kind == LL ? LL_MAX_LOG : kind == OF ? OF_MAX_LOG : ML_MAX_LOG;
    if (mode == 3) return have ? 0 : -1;
    int used = 0, nlog = 0;
    lanes_sync(lanes);  // every lane is done with the previous block's table
    if (lane == 0) {
        if (mode == 0) {
            const int16_t* d = kind == LL ? ZCONST(LL_DEFAULT) : kind == OF ? ZCONST(OF_DEFAULT) : ZCONST(ML_DEFAULT);
            const int nsym = kind == LL ? 36 : kind == OF ? 29 : 53;
            nlog = kind == OF ? 5 : 6;
            for (int i = 0; i < nsym; ++i) s.norm[i] = d[i];
            fse_build(s.norm, nsym, nlog, t, s.next);
        } else if (mode == 1) {
            if (n < 1 || load_in(in) > max_sym) {
                used = -1;
            } else {
                t[0] = {0, load_in(in), 0};
                used = 1;
            }
        } else {
            int nsym;
            used = read_ncount(in, n, max_sym, max_log, s.norm, nsym, nlog);
            if (used >= 0 && fse_build(s.norm, nsym, nlog, t, s.next) < 0) used = -1;
        }
    }
    used = from_lane0(used);
    log = from_lane0(nlog);
    lanes_sync(lanes);
    if (used >= 0) have = true;
    return used;
}

struct FrameState {
    bool have_huf, have_ll, have_of, have_ml;
    int huf_bits, ll_log, of_log, ml_log;
    int64_t rep[3];
};

// One compressed block b[0, n) appended at out + op (frame output from out + frame_start, capacity cap); a status.
__host__ __device__ int zstd_block(const uint8_t* b, int n, uint8_t* out, int64_t& op, int64_t frame_start, int64_t cap,
                                   uint64_t window, FrameState& f, ZstdScratch& s, int lane, int lanes) {
    // ---- literals section
    if (n < 1) return B200_ZSTD_LITERALS;
    const int b0 = load_in(b), type = b0 & 3, sf = (b0 >> 2) & 3;
    int64_t regen;
    int section;
    const uint8_t* lit;
    if (type < 2) {  // Raw or RLE
        const int lh = sf == 1 ? 2 : sf == 3 ? 3 : 1;
        if (n < lh) return B200_ZSTD_LITERALS;
        regen = lh == 1 ? b0 >> 3 : lh == 2 ? (b0 >> 4) + ((int)load_in(b + 1) << 4)
                                            : (b0 >> 4) + ((int)load_in(b + 1) << 4) + ((int)load_in(b + 2) << 12);
        if (type == 0) {
            if (regen > n - lh) return B200_ZSTD_LITERALS;
            lit = b + lh;
            section = lh + (int)regen;
        } else {
            if (n < lh + 1) return B200_ZSTD_LITERALS;
            if (regen > cap - op) return B200_ZSTD_OVERFLOW;
            uint8_t* dst = out + cap - regen;
            const uint8_t v = load_in(b + lh);
            for (int64_t i = lane; i < regen; i += lanes) dst[i] = v;
            lanes_sync(lanes);
            lit = dst;
            section = lh + 1;
        }
    } else {  // Huffman-coded, with a tree or Treeless
        const int lh = sf < 2 ? 3 : sf == 2 ? 4 : 5;
        if (n < lh) return B200_ZSTD_LITERALS;
        int64_t csize;
        if (lh == 3) {
            const uint32_t v = le24(b);
            regen = (v >> 4) & 0x3ff, csize = (v >> 14) & 0x3ff;
        } else if (lh == 4) {
            const uint32_t v = le32(b);
            regen = (v >> 4) & 0x3fff, csize = v >> 18;
        } else {
            const uint64_t v = le32(b) | (uint64_t)load_in(b + 4) << 32;
            regen = (v >> 4) & 0x3ffff, csize = (v >> 22) & 0x3ffff;
        }
        if (regen > BLOCK_MAX || csize > n - lh) return B200_ZSTD_LITERALS;
        if (regen > cap - op) return B200_ZSTD_OVERFLOW;
        const uint8_t* h = b + lh;
        int hs = 0;
        if (type == 2) {
            hs = read_huffman(h, (int)csize, s, f.huf_bits, lane, lanes);
            if (hs < 0) return B200_ZSTD_HUFFMAN;
            f.have_huf = true;
        } else if (!f.have_huf) {
            return B200_ZSTD_LITERALS;
        }
        const uint8_t* src = h + hs;
        const int64_t plen = csize - hs;
        uint8_t* dst = out + cap - regen;
        int bad = 0;
        if (sf == 0) {  // one stream
            if (lane == 0) bad = !huf_stream(src, plen, dst, (int)regen, s.huf, f.huf_bits);
        } else {  // four streams after a jump table of three sizes
            if (plen < 10) return B200_ZSTD_HUFFMAN;
            const int64_t l1 = le16(src), l2 = le16(src + 2), l3 = le16(src + 4);
            const int64_t l4 = plen - 6 - l1 - l2 - l3;
            const int64_t seg = (regen + 3) / 4, last = regen - 3 * seg;
            if (l4 < 1 || last < 0) return B200_ZSTD_HUFFMAN;
            for (int k = lane; k < 4; k += lanes) {
                const int64_t at = 6 + (k > 0 ? l1 : 0) + (k > 1 ? l2 : 0) + (k > 2 ? l3 : 0);
                const int64_t len = k == 0 ? l1 : k == 1 ? l2 : k == 2 ? l3 : l4;
                bad |= !huf_stream(src + at, len, dst + k * seg, (int)(k == 3 ? last : seg), s.huf, f.huf_bits);
            }
        }
        lanes_sync(lanes);
        if (lanes_any(bad)) return B200_ZSTD_HUFFMAN;
        lit = dst;
        section = lh + (int)csize;
    }
    // ---- sequences section
    const uint8_t* q = b + section;
    int m = n - section;
    if (m < 1) return B200_ZSTD_SEQUENCES;
    int nseq = load_in(q), hl = 1;
    if (nseq >= 128) {
        if (m < 2) return B200_ZSTD_SEQUENCES;
        if (nseq < 255) {
            nseq = ((nseq - 128) << 8) + load_in(q + 1), hl = 2;
        } else {
            if (m < 3) return B200_ZSTD_SEQUENCES;
            nseq = (int)le16(q + 1) + 0x7f00, hl = 3;
        }
    }
    q += hl, m -= hl;
    int64_t lp = 0;  // literals consumed
    if (nseq > 0) {
        if (m < 1) return B200_ZSTD_SEQUENCES;
        const int modes = load_in(q);
        if (modes & 3) return B200_ZSTD_SEQUENCES;
        ++q, --m;
        const int mode[3] = {modes >> 6, (modes >> 4) & 3, (modes >> 2) & 3};
        int* logs[3] = {&f.ll_log, &f.of_log, &f.ml_log};
        bool* have[3] = {&f.have_ll, &f.have_of, &f.have_ml};
        for (int k = 0; k < 3; ++k) {
            int lg = *logs[k];
            const int u = seq_table(k, mode[k], q, m, s, lg, *have[k], lane, lanes);
            if (u < 0) return B200_ZSTD_FSE;
            if (mode[k] != 3) *logs[k] = lg;
            q += u, m -= u;
        }
        BackBits br;
        if (!br.init(q, m)) return B200_ZSTD_SEQUENCES;
        int sll = (int)br.read(f.ll_log), sof = (int)br.read(f.of_log), sml = (int)br.read(f.ml_log);
        for (int i = 0; i < nseq; ++i) {
            const int ofc = s.of[sof].sym, mlc = s.ml[sml].sym, llc = s.ll[sll].sym;
            const uint64_t ofv = (1ull << ofc) + br.read(ofc);
            const int64_t ml = mlc < 32 ? mlc + 3 : ZCONST(ML_BASE)[mlc - 32] + br.read(ZCONST(ML_BITS)[mlc - 32]);
            const int64_t ll = llc < 16 ? llc : ZCONST(LL_BASE)[llc - 16] + br.read(ZCONST(LL_BITS)[llc - 16]);
            int64_t off;
            if (ofv > 3) {
                off = (int64_t)(ofv - 3);
                f.rep[2] = f.rep[1], f.rep[1] = f.rep[0], f.rep[0] = off;
            } else {
                const int idx = (int)ofv - (ll != 0);
                if (idx == 0) {
                    off = f.rep[0];
                } else if (idx == 1) {
                    off = f.rep[1];
                    f.rep[1] = f.rep[0], f.rep[0] = off;
                } else {
                    off = idx == 2 ? f.rep[2] : f.rep[0] - 1;
                    if (off <= 0) return B200_ZSTD_OFFSET;
                    f.rep[2] = f.rep[1], f.rep[1] = f.rep[0], f.rep[0] = off;
                }
            }
            if (i + 1 < nseq) {
                sll = s.ll[sll].base + (int)br.read(s.ll[sll].bits);
                sml = s.ml[sml].base + (int)br.read(s.ml[sml].bits);
                sof = s.of[sof].base + (int)br.read(s.of[sof].bits);
            }
            if (br.pos < 0 || ll > regen - lp) return B200_ZSTD_SEQUENCES;
            if (ll + ml > cap - op) return B200_ZSTD_OVERFLOW;
            copy_down(out + op, lit + lp, ll, lane, lanes);
            op += ll, lp += ll;
            if (off > op - frame_start || (uint64_t)off > window) return B200_ZSTD_OFFSET;
            copy_match(out, op, off, ml, lane, lanes);
            op += ml;
        }
        if (br.pos != 0) return B200_ZSTD_SEQUENCES;
    } else if (m != 0) {
        return B200_ZSTD_SEQUENCES;
    }
    if (regen - lp > cap - op) return B200_ZSTD_OVERFLOW;
    copy_down(out + op, lit + lp, regen - lp, lane, lanes);
    op += regen - lp;
    return B200_ZSTD_OK;
}

__host__ __device__ __forceinline__ uint64_t rotl64(uint64_t x, int r) { return x << r | x >> (64 - r); }

constexpr uint64_t XP1 = 0x9E3779B185EBCA87ull, XP2 = 0xC2B2AE3D27D4EB4Full, XP3 = 0x165667B19E3779F9ull,
                   XP4 = 0x85EBCA77C2B2AE63ull, XP5 = 0x27D4EB2F165667C5ull;

__host__ __device__ __forceinline__ uint64_t xxh_round(uint64_t acc, uint64_t in) { return rotl64(acc + in * XP2, 31) * XP1; }

__host__ __device__ __forceinline__ uint64_t load64(const uint8_t* p) {
    uint64_t v = 0;
    for (int i = 0; i < 8; ++i) v |= (uint64_t)p[i] << (8 * i);
    return v;
}

// XXH64 (seed 0) of p[0, n), written by the lanes before the call: one lane per accumulator
__host__ __device__ uint64_t xxh64(const uint8_t* p, int64_t n, int lane, int lanes) {
    uint64_t h;
    const int64_t stripes = n / 32;
    if (stripes) {
        const uint64_t init[4] = {XP1 + XP2, XP2, 0, 0 - XP1};
        uint64_t v[4] = {0, 0, 0, 0};
        for (int k = lane; k < 4; k += lanes) {
            uint64_t a = init[k];
            for (int64_t i = 0; i < stripes; ++i) a = xxh_round(a, load64(p + 32 * i + 8 * k));
            v[k] = a;
        }
#ifdef __CUDA_ARCH__
        for (int k = 0; k < 4; ++k) v[k] = __shfl_sync(0xffffffffu, v[k], k);
#endif
        h = rotl64(v[0], 1) + rotl64(v[1], 7) + rotl64(v[2], 12) + rotl64(v[3], 18);
        for (int k = 0; k < 4; ++k) h = (h ^ xxh_round(0, v[k])) * XP1 + XP4;
    } else {
        h = XP5;
    }
    h += (uint64_t)n;
    int64_t i = stripes * 32;
    for (; i + 8 <= n; i += 8) h = rotl64(h ^ xxh_round(0, load64(p + i)), 27) * XP1 + XP4;
    if (i + 4 <= n) {
        const uint64_t w = p[i] | (uint64_t)p[i + 1] << 8 | (uint64_t)p[i + 2] << 16 | (uint64_t)p[i + 3] << 24;
        h = rotl64(h ^ w * XP1, 23) * XP2 + XP3;
        i += 4;
    }
    for (; i < n; ++i) h = rotl64(h ^ p[i] * XP5, 11) * XP1;
    h ^= h >> 33;
    h *= XP2;
    h ^= h >> 29;
    h *= XP3;
    h ^= h >> 32;
    return h;
}

// One zstd frame starting at in[ip] (its magic already checked); appends at out + op.  A status.
__host__ __device__ int zstd_frame(const uint8_t* in, int64_t n, int64_t& ip, uint8_t* out, int64_t& op, int64_t cap,
                                   ZstdScratch& s, int lane, int lanes) {
    ip += 4;
    if (ip >= n) return B200_ZSTD_TRUNCATED;
    const int fhd = load_in(in + ip++);
    const int fcs_flag = fhd >> 6, single = (fhd >> 5) & 1, checksum = (fhd >> 2) & 1, did_flag = fhd & 3;
    if (fhd & 8) return B200_ZSTD_FRAME_HEADER;
    const int did_size = did_flag == 3 ? 4 : did_flag, fcs_size = fcs_flag == 0 ? single : 1 << fcs_flag;
    if (n - ip < !single + did_size + fcs_size) return B200_ZSTD_TRUNCATED;
    uint64_t window = 0;
    if (!single) {
        const int wd = load_in(in + ip++), wlog = 10 + (wd >> 3);
        if (wlog > 31) return B200_ZSTD_FRAME_HEADER;
        window = (1ull << wlog) + ((1ull << wlog) >> 3) * (wd & 7);
    }
    uint32_t did = 0;
    for (int i = 0; i < did_size; ++i) did |= (uint32_t)load_in(in + ip++) << (8 * i);
    if (did) return B200_ZSTD_FRAME_HEADER;
    uint64_t fcs = 0;
    for (int i = 0; i < fcs_size; ++i) fcs |= (uint64_t)load_in(in + ip++) << (8 * i);
    if (fcs_size == 2) fcs += 256;
    if (single) window = fcs;
    const int64_t frame_start = op;
    if (fcs_size && fcs > (uint64_t)(cap - op)) return B200_ZSTD_OVERFLOW;
    FrameState f = {false, false, false, false, 0, 0, 0, 0, {1, 4, 8}};
    for (bool last = false; !last;) {
        if (n - ip < 3) return B200_ZSTD_TRUNCATED;
        const uint32_t bh = le24(in + ip);
        ip += 3;
        last = bh & 1;
        const int type = (bh >> 1) & 3;
        const int64_t size = bh >> 3;
        if (type == 3) return B200_ZSTD_BLOCK_TYPE;
        if (type == 1) {  // RLE
            if (n - ip < 1) return B200_ZSTD_TRUNCATED;
            if (size > cap - op) return B200_ZSTD_OVERFLOW;
            const uint8_t v = load_in(in + ip++);
            for (int64_t i = lane; i < size; i += lanes) out[op + i] = v;
            op += size;
            lanes_sync(lanes);
            continue;
        }
        if (size > n - ip) return B200_ZSTD_TRUNCATED;
        if (type == 0) {  // Raw
            if (size > cap - op) return B200_ZSTD_OVERFLOW;
            for (int64_t i = lane; i < size; i += lanes) out[op + i] = load_in(in + ip + i);
            op += size;
            lanes_sync(lanes);
        } else {
            if (size > BLOCK_MAX) return B200_ZSTD_BLOCK_TYPE;
            const int st = zstd_block(in + ip, (int)size, out, op, frame_start, cap, window, f, s, lane, lanes);
            if (st) return st;
        }
        ip += size;
    }
    if (fcs_size && (uint64_t)(op - frame_start) != fcs) return B200_ZSTD_CONTENT_SIZE;
    if (checksum) {
        if (n - ip < 4) return B200_ZSTD_TRUNCATED;
        const uint32_t want = le32(in + ip);
        ip += 4;
        if ((uint32_t)xxh64(out + frame_start, op - frame_start, lane, lanes) != want) return B200_ZSTD_CHECKSUM;
    }
    return B200_ZSTD_OK;
}

// A whole stream in[0, n): frames and skippable frames back to back, as ZSTD_decompress takes them.  A status; *len =
// bytes written to out[0, cap).
__host__ __device__ int zstd_stream(const uint8_t* in, int64_t n, uint8_t* out, int64_t cap, int64_t& len, ZstdScratch& s,
                                    int lane, int lanes) {
    int64_t ip = 0, op = 0;
    int st = B200_ZSTD_OK;
    while (n - ip >= 5) {
        const uint32_t magic = le32(in + ip);
        if ((magic & 0xfffffff0u) == 0x184d2a50u) {  // skippable frame
            if (n - ip < 8) {
                st = B200_ZSTD_TRUNCATED;
                break;
            }
            const int64_t size = le32(in + ip + 4);
            if (size > n - ip - 8) {
                st = B200_ZSTD_TRUNCATED;
                break;
            }
            ip += 8 + size;
            continue;
        }
        if (magic != 0xfd2fb528u) {
            st = B200_ZSTD_MAGIC;
            break;
        }
        st = zstd_frame(in, n, ip, out, op, cap, s, lane, lanes);
        if (st) break;
    }
    if (st == B200_ZSTD_OK && ip != n) st = B200_ZSTD_TRUNCATED;
    lanes_sync(lanes);
    len = op;
    return st;
}

// one warp per stream; meta[i] = input offset, input length, output offset, output capacity
__global__ void __launch_bounds__(ZSTD_WARPS * 32)
    zstd_kernel(const uint8_t* __restrict__ in, int64_t in_bytes, const int64_t* __restrict__ meta, int n, uint8_t* out,
                int64_t out_bytes, int64_t* __restrict__ out_len, int32_t* __restrict__ status) {
    __shared__ ZstdScratch scratch[ZSTD_WARPS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t r = (int64_t)blockIdx.x * ZSTD_WARPS + warp;
    if (r >= n) return;
    const int64_t* mm = meta + 4 * r;
    const int64_t in_start = mm[0], in_len = mm[1], out_start = mm[2], cap = mm[3];
    int64_t len = 0;
    int st;
    if (in_start < 0 || in_len < 0 || in_start > in_bytes || in_len > in_bytes - in_start || out_start < 0 || cap < 0 ||
        out_start > out_bytes || cap > out_bytes - out_start) {
        st = B200_ZSTD_BOUNDS;
    } else {
        st = zstd_stream(in + in_start, in_len, out + out_start, cap, len, scratch[warp], lane, 32);
    }
    if (lane == 0) {
        status[r] = st;
        out_len[r] = len;
    }
}

// svb16: one warp per row; meta[i] = svb offset in `in`, svb length, sample count, sample offset in `out`
__global__ void __launch_bounds__(SVB_WARPS * 32)
    svb16_kernel(const uint8_t* __restrict__ in, int64_t in_bytes, const int64_t* __restrict__ meta, int n,
                 int16_t* __restrict__ out, int64_t out_samples, int32_t* __restrict__ status) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t r = (int64_t)blockIdx.x * SVB_WARPS + warp;
    if (r >= n) return;
    const int64_t* mm = meta + 4 * r;
    const int64_t start = mm[0], len = mm[1], count = mm[2], o = mm[3];
    if (start < 0 || len < 0 || start > in_bytes || len > in_bytes - start || count < 0 || o < 0 || o > out_samples ||
        count > out_samples - o) {
        if (lane == 0) status[r] = B200_SVB16_BOUNDS;
        return;
    }
    const int64_t keys = (count + 7) >> 3;
    if (len < keys) {
        if (lane == 0) status[r] = B200_SVB16_LENGTH;
        return;
    }
    const uint8_t* key = in + start;
    const uint8_t* data = key + keys;
    const int64_t dlen = len - keys;
    int16_t* dst = out + o;
    int64_t dpos = 0;     // data bytes before this step
    uint32_t carry = 0;   // the last sample before this step
    for (int64_t base = 0; base < count; base += 256) {
        const int64_t kb = (base >> 3) + lane, j0 = kb * 8;
        const int nv = j0 >= count ? 0 : count - j0 >= 8 ? 8 : (int)(count - j0);
        const uint32_t k = nv ? load_in(key + kb) & ((1u << nv) - 1) : 0;
        const int nbytes = nv + __popc(k);
        int incl = nbytes;  // inclusive scan of the lanes' byte counts
        for (int d = 1; d < 32; d <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += v;
        }
        int64_t p = dpos + incl - nbytes;
        uint32_t v[8], sum = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            if (i < nv) {
                uint32_t z = p < dlen ? load_in(data + p) : 0;
                if (k >> i & 1) z |= (p + 1 < dlen ? (uint32_t)load_in(data + p + 1) : 0u) << 8;
                p += 1 + (k >> i & 1);
                sum += (z >> 1) ^ (0u - (z & 1));  // unzigzag; sums are taken mod 2^16
            }
            v[i] = sum;
        }
        uint32_t acc = sum;  // inclusive scan of the lanes' delta sums
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, acc, d);
            if (lane >= d) acc += t;
        }
        const uint32_t before = carry + acc - sum;
#pragma unroll
        for (int i = 0; i < 8; ++i)
            if (i < nv) dst[j0 + i] = (int16_t)(uint16_t)(before + v[i]);
        carry += __shfl_sync(0xffffffffu, acc, 31);
        dpos += __shfl_sync(0xffffffffu, incl, 31);
    }
    if (lane == 0) status[r] = dpos == dlen ? B200_SVB16_OK : B200_SVB16_LENGTH;
}

}  // namespace

extern "C" {

int b200_zstd_decompress(const uint8_t* in, int64_t in_bytes, const int64_t* meta, int n, uint8_t* out, int64_t out_bytes,
                         int64_t* out_len, int32_t* status, void* stream) {
    B200_REQUIRE(n >= 0 && in_bytes >= 0 && out_bytes >= 0, "zstd_decompress: negative size");
    if (n == 0) return 0;
    B200_REQUIRE(meta && status && out_len && (in || in_bytes == 0) && (out || out_bytes == 0),
                 "zstd_decompress: null pointer argument");
    const unsigned blocks = (unsigned)((n + ZSTD_WARPS - 1) / ZSTD_WARPS);
    zstd_kernel<<<blocks, ZSTD_WARPS * 32, 0, (cudaStream_t)stream>>>(in, in_bytes, meta, n, out, out_bytes, out_len, status);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int b200_svb16_decode(const uint8_t* in, int64_t in_bytes, const int64_t* meta, int n, int16_t* out, int64_t out_samples,
                      int32_t* status, void* stream) {
    B200_REQUIRE(n >= 0 && in_bytes >= 0 && out_samples >= 0, "svb16_decode: negative size");
    if (n == 0) return 0;
    B200_REQUIRE(meta && status && (in || in_bytes == 0) && (out || out_samples == 0), "svb16_decode: null pointer argument");
    const unsigned blocks = (unsigned)((n + SVB_WARPS - 1) / SVB_WARPS);
    svb16_kernel<<<blocks, SVB_WARPS * 32, 0, (cudaStream_t)stream>>>(in, in_bytes, meta, n, out, out_samples, status);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // extern "C"
