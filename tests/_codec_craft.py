"""
Hand-built zstd frames (RFC 8878) and DEFLATE streams (RFC 1951) in which the caller picks every encoding: frame header
fields, block types, literals modes and size formats, Huffman weights and code lengths, FSE table descriptions and the
table mode of each sequence code, the parse itself, DEFLATE block types, HLIT / HDIST / HCLEN and the code-length runs.
Encoders at their usual settings never reach many of the decoders' branches; these streams do.

Every builder returns (stream, expected bytes, features); `features` names the format branches the stream uses, and
zstd_valid(), zstd_malformed(), inflate_valid() and inflate_malformed() are the named lists the tests run.  Pure Python
and numpy, so the lists build anywhere the tests run.
"""
import heapq
import struct
import zlib

import numpy as np

M64 = (1 << 64) - 1

# B200_ZSTD_* and B200_INFLATE_* status codes (include/bonito_b200.h)
Z_OK, Z_MAGIC, Z_FRAME_HEADER, Z_BLOCK_TYPE, Z_LITERALS, Z_HUFFMAN, Z_FSE, Z_SEQUENCES, Z_OFFSET, Z_OVERFLOW, \
    Z_CONTENT_SIZE, Z_TRUNCATED, Z_CHECKSUM, Z_BOUNDS = range(14)
I_OK, I_BLOCK_TYPE, I_STORED_LENGTH, I_CODE_LENGTHS, I_REPEAT, I_SYMBOL, I_DISTANCE, I_OVERFLOW, I_SHORT, I_TRUNCATED, \
    I_CRC, I_BOUNDS = range(12)


class Bits:
    """An LSB-first bit writer: DEFLATE fields, zstd FSE table descriptions, and zstd backward streams (see back())."""

    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def put(self, v, n):
        assert n >= 0 and 0 <= v < (1 << n) or (n == 0 and v == 0), (v, n)
        self.acc |= v << self.n
        self.n += n
        while self.n >= 8:
            self.out.append(self.acc & 255)
            self.acc >>= 8
            self.n -= 8
        return self

    def code(self, c, n):
        """A DEFLATE Huffman code: most significant bit first."""
        return self.put(int(format(c, f"0{n}b")[::-1], 2) if n else 0, n)

    def align(self):
        return self.put(0, -self.n % 8)

    @property
    def nbits(self):
        return 8 * len(self.out) + self.n

    def bytes(self):
        return bytes(self.out) + (bytes([self.acc]) if self.n else b"")


def back(fields):
    """A zstd backward bit stream whose reader meets fields [(value, nbits)] in this order; the end marker included."""
    w = Bits()
    for v, n in reversed(fields):
        w.put(v, n)
    return w.put(1, 1).bytes()


# ================================================================================================================ zstd
MAGIC = struct.pack("<I", 0xFD2FB528)
LL, OF, ML = 0, 1, 2
LL_DEFAULT = [4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1]
ML_DEFAULT = [1, 4, 3, 2, 2, 2, 2, 2, 2] + [1] * 37 + [-1] * 7
OF_DEFAULT = [1, 1, 1, 1, 1, 1, 2, 2, 2] + [1] * 15 + [-1] * 5
LL_BASE = list(range(16)) + [16, 18, 20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768,
                             65536]
LL_BITS = [0] * 16 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
ML_BASE = list(range(3, 35)) + [35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195, 16387,
                                32771, 65539]
ML_BITS = [0] * 32 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
MAX_SYM = {LL: 35, OF: 31, ML: 52}
MAX_LOG = {LL: 9, OF: 8, ML: 9}
BLOCK_MAX = 128 * 1024

XP1, XP2, XP3, XP4, XP5 = (0x9E3779B185EBCA87, 0xC2B2AE3D27D4EB4F, 0x165667B19E3779F9, 0x85EBCA77C2B2AE63,
                           0x27D4EB2F165667C5)


def _rotl(x, r):
    return ((x << r) | (x >> (64 - r))) & M64


def _round(acc, lane):
    return _rotl((acc + lane * XP2) & M64, 31) * XP1 & M64


def xxh64(data, seed=0):
    """XXH64 of data (the zstd content checksum is its low 32 bits)."""
    data = bytes(data)
    n, i = len(data), 0
    if n >= 32:
        words = np.frombuffer(data[:n - n % 32], dtype="<u8").reshape(-1, 4).tolist()
        v = [(seed + XP1 + XP2) & M64, (seed + XP2) & M64, seed, (seed - XP1) & M64]
        for row in words:
            v = [_round(a, w) for a, w in zip(v, row)]
        h = (_rotl(v[0], 1) + _rotl(v[1], 7) + _rotl(v[2], 12) + _rotl(v[3], 18)) & M64
        for a in v:
            h = ((h ^ _round(0, a)) * XP1 + XP4) & M64
        i = n - n % 32
    else:
        h = (seed + XP5) & M64
    h = (h + n) & M64
    while i + 8 <= n:
        h = (_rotl(h ^ _round(0, struct.unpack_from("<Q", data, i)[0]), 27) * XP1 + XP4) & M64
        i += 8
    if i + 4 <= n:
        h = (_rotl(h ^ (struct.unpack_from("<I", data, i)[0] * XP1 & M64), 23) * XP2 + XP3) & M64
        i += 4
    for b in data[i:]:
        h = _rotl(h ^ (b * XP5 & M64), 11) * XP1 & M64
    h ^= h >> 33
    h = h * XP2 & M64
    h ^= h >> 29
    h = h * XP3 & M64
    return h ^ (h >> 32)


def fse_table(norm, log):
    """The decoding table [(symbol, bits, base)] of a normalized distribution (RFC 8878 section 4.1.1)."""
    size = 1 << log
    assert sum(abs(c) for c in norm) == size, (sum(abs(c) for c in norm), size)
    high, sym, nxt = size - 1, [0] * size, {}
    for s, c in enumerate(norm):
        if c == -1:
            sym[high] = s
            high -= 1
            nxt[s] = 1
        else:
            nxt[s] = c
    step, pos = (size >> 1) + (size >> 3) + 3, 0
    for s, c in enumerate(norm):
        for _ in range(max(c, 0)):
            sym[pos] = s
            pos = (pos + step) & (size - 1)
            while pos > high:
                pos = (pos + step) & (size - 1)
    assert pos == 0
    table = []
    for u in range(size):
        s = sym[u]
        ns = nxt[s]
        nxt[s] += 1
        bits = log - (ns.bit_length() - 1)
        table.append((s, bits, (ns << bits) - size))
    return table


def fse_states(table, symbols):
    """Decoder states s_0.. that emit `symbols` (s_i+1 = base_i + the bits read after s_i).  The last state is the one of
    its symbol with the most bits, so that a reader updating it past the stream's start runs out of bits."""
    by_sym = {}
    for u, (s, _, _) in enumerate(table):
        by_sym.setdefault(s, []).append(u)
    states = [0] * len(symbols)
    states[-1] = max(by_sym[symbols[-1]], key=lambda u: table[u][1])
    for i in range(len(symbols) - 2, -1, -1):
        nxt = states[i + 1]
        states[i] = next(u for u in by_sym[symbols[i]] if table[u][2] <= nxt < table[u][2] + (1 << table[u][1]))
    return states


def ncount(norm, log):
    """An FSE table description (RFC 8878 section 4.1.1) of norm (counts, -1 for "less than 1"): the bytes."""
    w = Bits().put(log - 5, 4)
    remaining, threshold, nb = (1 << log) + 1, 1 << log, log + 1
    last = max(s for s, c in enumerate(norm) if c)
    s = 0
    while s <= last:
        c = norm[s]
        value = c + 1
        mx = (2 * threshold - 1) - remaining
        if value >= threshold:
            value += mx
        if value < mx:
            w.put(value, nb - 1)
        else:
            w.put(value, nb)
        remaining -= abs(c)
        while remaining < threshold:
            nb -= 1
            threshold >>= 1
        s += 1
        if c == 0:   # repeat flags: how many more zero counts follow, 3 at a time
            z = 0
            while s + z <= last and norm[s + z] == 0:
                z += 1
            s += z
            while z >= 3:
                w.put(3, 2)
                z -= 3
            w.put(z, 2)
    assert remaining == 1
    return w.bytes()


def normalize(counts, log, below_one=()):
    """counts {symbol: n} scaled to a distribution over 2^log (symbols in below_one get -1): a list by symbol."""
    size, syms = 1 << log, sorted(counts)
    norm = [0] * (max(syms) + 1)
    for s in below_one:
        norm[s] = -1
    rest = [s for s in syms if s not in below_one]
    left, total = size - len(below_one), sum(counts[s] for s in rest)
    for s in rest:
        norm[s] = max(1, counts[s] * left // total)
    big = max(rest, key=lambda s: norm[s])
    norm[big] += left - sum(norm[s] for s in rest)
    assert norm[big] > 0
    return norm


def ll_code(ll):
    c = max(i for i, b in enumerate(LL_BASE) if b <= ll)
    assert ll - LL_BASE[c] < (1 << LL_BITS[c])
    return c, LL_BITS[c], ll - LL_BASE[c]


def ml_code(ml):
    c = max(i for i, b in enumerate(ML_BASE) if b <= ml)
    assert ml - ML_BASE[c] < (1 << ML_BITS[c])
    return c, ML_BITS[c], ml - ML_BASE[c]


def huf_codes(lengths):
    """zstd's canonical Huffman codes of lengths {symbol: bits} (a complete code): ({symbol: (code, bits)}, weights).
    Table entries go by weight, then symbol; weight = max bits + 1 - bits; the weights list stops before the last
    symbol, whose weight the decoder infers."""
    top = max(lengths.values())
    assert sum(2 ** (top - l) for l in lengths.values()) == 2 ** top, "the code must be complete"
    p, codes = 0, {}
    for s in sorted(lengths, key=lambda s: (top + 1 - lengths[s], s)):
        w = top + 1 - lengths[s]
        codes[s] = (p >> (w - 1), lengths[s])
        p += 1 << (w - 1)
    last = max(lengths)
    return codes, [top + 1 - lengths[s] if s in lengths else 0 for s in range(last)]


def lengths_for(data, max_bits):
    """Length-limited Huffman code lengths of data's bytes (a complete code of at least two symbols)."""
    counts = np.bincount(np.frombuffer(bytes(data), np.uint8), minlength=256)
    freq = {s: int(c) for s, c in enumerate(counts) if c}
    if len(freq) == 1:
        freq[(next(iter(freq)) + 1) % 256] = 1
    while True:
        lens = huffman_depths(freq)
        if max(lens.values()) <= max_bits:
            return lens
        freq = {s: (c + 1) // 2 for s, c in freq.items()}


def huffman_depths(freq):
    """Optimal (unlimited) prefix code lengths of {symbol: frequency}."""
    if len(freq) == 1:
        return {next(iter(freq)): 1}
    heap = [(f, i, (s,)) for i, (s, f) in enumerate(sorted(freq.items()))]
    heapq.heapify(heap)
    depth = dict.fromkeys(freq, 0)
    k = len(heap)
    while len(heap) > 1:
        f1, _, a = heapq.heappop(heap)
        f2, _, b = heapq.heappop(heap)
        for s in a + b:
            depth[s] += 1
        heapq.heappush(heap, (f1 + f2, k, a + b))
        k += 1
    return depth


class Frame:
    """One zstd frame under construction, with the decoder's state mirrored: the output so far, the repeat offsets and
    the tables that Repeat mode and Treeless literals reuse."""

    def __init__(self, fcs=None, fcs_bytes=None, single=False, window_log=17, window_mantissa=0, checksum=False,
                 dict_id=0, did_bytes=0):
        self.fcs, self.fcs_bytes, self.single = fcs, fcs_bytes, single
        self.window_log, self.window_mantissa, self.checksum = window_log, window_mantissa, checksum
        self.dict_id, self.did_bytes = dict_id, did_bytes
        self.blocks, self.out, self.rep = [], bytearray(), [1, 4, 8]
        self.tables = {LL: None, OF: None, ML: None}
        self.huf = None
        self.features = set()
        self.invalid = False

    @property
    def window(self):
        if self.single:
            return self.fcs
        return (1 << self.window_log) + ((1 << self.window_log) >> 3) * self.window_mantissa

    def header(self):
        f = self.features
        fcs_bytes = self.fcs_bytes
        if fcs_bytes is None:
            fcs_bytes = 0 if self.fcs is None else 1 if self.fcs < 256 else 2 if self.fcs < 65792 else 4 if \
                self.fcs < 1 << 32 else 8
        assert not (self.single and fcs_bytes == 0)
        flag = {0: 0, 1: 0, 2: 1, 4: 2, 8: 3}[fcs_bytes]
        assert fcs_bytes != 1 or self.single
        did_flag = {0: 0, 1: 1, 2: 2, 4: 3}[self.did_bytes]
        h = bytearray(MAGIC + bytes([flag << 6 | self.single << 5 | self.checksum << 2 | did_flag]))
        if not self.single:
            h.append((self.window_log - 10) << 3 | self.window_mantissa)
            f.add(("window", "descriptor"))
        else:
            f.add(("window", "single_segment"))
        h += self.dict_id.to_bytes(self.did_bytes, "little")
        if self.did_bytes:
            f.add(("dict_id", self.did_bytes))
        if fcs_bytes:
            f.add(("fcs", fcs_bytes))
            h += (self.fcs - (256 if fcs_bytes == 2 else 0)).to_bytes(fcs_bytes, "little")
        if self.checksum:
            f.add("checksum")
        return bytes(h)

    # ---- blocks
    def raw(self, data):
        self.blocks.append((0, bytes(data), len(data)))
        self.out += data
        self.features.add(("block", "raw"))
        return self

    def rle(self, byte, n):
        self.blocks.append((1, bytes([byte]), n))
        self.out += bytes([byte]) * n
        self.features.add(("block", "rle"))
        return self

    def compressed(self, literals, seqs=(), modes=("predef", "predef", "predef"), nseq_bytes=None):
        """A compressed block: `literals` a section from one of the lit_* methods (the section, the literal bytes),
        then the sequences [(literal length, match length, Offset_Value)] with table modes (LL, OF, ML), each
        "predef", "rle", "repeat" or ("fse", norm, log)."""
        section, lits = literals
        body = section + self._sequences(list(seqs), modes, nseq_bytes)
        assert len(body) <= BLOCK_MAX
        if len(body) == BLOCK_MAX:
            self.features.add(("block", "compressed_128k"))
        self.blocks.append((2, body, len(body)))
        self.features.add(("block", "compressed"))
        self._apply(lits, seqs)
        return self

    def _apply(self, lits, seqs):
        lp = 0
        for ll, ml, ofv in seqs:
            self.out += lits[lp:lp + ll]
            lp += ll
            if ofv > 3:
                off = ofv - 3
                self.rep = [off, self.rep[0], self.rep[1]]
            else:
                idx = ofv - (ll != 0)
                if idx == 0:
                    off = self.rep[0]
                elif idx == 1:
                    off = self.rep[1]
                    self.rep = [off, self.rep[0], self.rep[2]]
                else:
                    off = self.rep[2] if idx == 2 else self.rep[0] - 1
                    self.rep = [off, self.rep[0], self.rep[1]]
                self.features.add(("repeat", ofv, ll == 0))
            if not 0 < off <= len(self.out) or lp > len(lits):
                self.invalid = True     # a malformed stream on purpose: the expected output is moot
                return
            while ml:
                n = min(ml, off)
                self.out += self.out[len(self.out) - off:len(self.out) - off + n]
                ml -= n
        self.out += lits[lp:]

    # ---- literals sections
    @staticmethod
    def _raw_header(btype, n, hl):
        if hl == 1:
            assert n < 32
            return bytes([btype | n << 3])
        if hl == 2:
            assert n < 4096
            return bytes([btype | 1 << 2 | (n & 15) << 4, n >> 4])
        assert n < 1 << 20
        return bytes([btype | 3 << 2 | (n & 15) << 4, (n >> 4) & 255, n >> 12])

    def lit_raw(self, data, hl=None):
        hl = hl or (1 if len(data) < 32 else 2 if len(data) < 4096 else 3)
        self.features.add(("lit", "raw", hl))
        return self._raw_header(0, len(data), hl) + bytes(data), bytes(data)

    def lit_rle(self, byte, n, hl=None):
        hl = hl or (1 if n < 32 else 2 if n < 4096 else 3)
        self.features.add(("lit", "rle", hl))
        return self._raw_header(1, n, hl) + bytes([byte]), bytes([byte]) * n

    def lit_huffman(self, data, lengths=None, streams=4, sf=None, weights="fse", wlog=6, below_one=()):
        """Huffman-coded literals: with a tree description of `lengths` ({byte: bits}; weights "direct" or "fse" at
        accuracy log wlog), or Treeless (lengths None: the previous block's tree).  streams 1 or 4; sf the size format
        (0: 1 stream and 10-bit sizes, 1 / 2 / 3: 4 streams and 10 / 14 / 18-bit sizes)."""
        data = bytes(data)
        f = self.features
        if lengths is None:
            assert self.huf is not None
            tree = b""
            f.add(("lit", "treeless"))
        else:
            codes, wts = huf_codes(lengths)
            self.huf = codes
            if weights == "direct":
                assert len(wts) <= 128
                wts2 = wts + [0] * (len(wts) % 2)
                tree = bytes([127 + len(wts)]) + bytes(wts2[i] << 4 | wts2[i + 1] for i in range(0, len(wts2), 2))
                f.add(("huf_weights", "direct"))
            else:
                tree = self._fse_weights(wts, wlog, below_one)
                f.add(("huf_weights", "fse"))
            f.add(("huf_weight_count", len(wts)))
            f.add(("huf_max_bits", max(lengths.values())))
        codes = self.huf
        n = len(data)
        if streams == 1:
            payload = back([codes[b] for b in data])
        else:
            seg = (n + 3) // 4
            parts = [data[:seg], data[seg:2 * seg], data[2 * seg:3 * seg], data[3 * seg:]]
            assert len(parts[3]) == n - 3 * seg >= 0
            if not parts[3]:
                f.add(("lit", "4stream_empty_last"))
            enc = [back([codes[b] for b in p]) for p in parts]
            payload = struct.pack("<HHH", *(len(e) for e in enc[:3])) + b"".join(enc)
        csize = len(tree) + len(payload)
        if sf is None:
            sf = 0 if streams == 1 else 1 if max(n, csize) < 1024 else 2 if max(n, csize) < 16384 else 3
        assert (sf == 0) == (streams == 1)
        bits = 10 if sf < 2 else 14 if sf == 2 else 18
        assert n < 1 << bits and csize < 1 << bits
        v = (3 if lengths is None else 2) | sf << 2 | n << 4 | csize << (4 + bits)
        f.add(("lit", "huffman", f"{streams}stream", f"sf{bits}"))
        return v.to_bytes((4 + 2 * bits + 7) // 8, "little") + tree + payload, data

    def _fse_weights(self, wts, log, below_one):
        """Weights FSE-coded with two interleaved states (RFC 8878 section 4.2.1.2): header byte, table, stream."""
        counts = {}
        for w in wts:
            counts[w] = counts.get(w, 0) + 1
        norm = normalize(counts, log, below_one)
        table = fse_table(norm, log)
        chains = [fse_states(table, wts[0::2]), fse_states(table, wts[1::2])]
        fields = [(chains[0][0], log), (chains[1][0], log)]
        for i in range(len(wts) - 2):   # the update after weight i; the one after the next-to-last runs dry
            u, nxt = chains[i % 2][i // 2], chains[i % 2][i // 2 + 1]
            fields.append((nxt - table[u][2], table[u][1]))
        assert table[chains[len(wts) % 2][-1]][1] > 0
        body = ncount(norm, log) + back(fields)
        assert len(body) < 128, len(body)
        if -1 in norm:
            self.features.add(("fse", "below_one"))
        return bytes([len(body)]) + body

    # ---- sequences section
    def _sequences(self, seqs, modes, nseq_bytes):
        f = self.features
        n = len(seqs)
        if nseq_bytes is None:
            nseq_bytes = 1 if n < 128 else 2 if n < 0x7F00 else 3
        if nseq_bytes == 1:
            head = bytes([n])
        elif nseq_bytes == 2:
            assert n < 0x7F00
            head = bytes([128 + (n >> 8), n & 255])
        else:
            head = bytes([255]) + struct.pack("<H", n - 0x7F00)
        f.add(("seq", f"nseq{nseq_bytes}"))
        if not n:
            return head
        codes = {LL: [], OF: [], ML: []}
        extra = []
        for ll, ml, ofv in seqs:
            lc, lb, lx = ll_code(ll)
            mc, mb, mx = ml_code(ml)
            oc = ofv.bit_length() - 1
            codes[LL].append(lc)
            codes[ML].append(mc)
            codes[OF].append(oc)
            extra.append(((ofv - (1 << oc), oc), (mx, mb), (lx, lb)))
            f.update({("ll_code", lc), ("ml_code", mc), ("of_code", oc)})
        mode_bits, desc, tabs = 0, b"", {}
        for k, name in ((LL, "ll"), (OF, "of"), (ML, "ml")):
            m = modes[k]
            if m == "predef":
                dflt = {LL: (LL_DEFAULT, 6), OF: (OF_DEFAULT, 5), ML: (ML_DEFAULT, 6)}[k]
                self.tables[k] = (fse_table(*dflt), dflt[1])
                mb = 0
            elif m == "rle":
                assert len(set(codes[k])) == 1
                desc += bytes([codes[k][0]])
                self.tables[k] = ([(codes[k][0], 0, 0)], 0)
                mb = 1
                if (LL_BITS if k == LL else ML_BITS if k == ML else range(32))[codes[k][0]]:
                    f.add(("rle_table_with_extra_bits", name))
            elif m == "repeat":
                assert self.tables[k] is not None
                mb = 3
            else:
                _, norm, log = m
                assert log <= MAX_LOG[k] and len(norm) - 1 <= MAX_SYM[k]
                desc += ncount(norm, log)
                self.tables[k] = (fse_table(norm, log), log)
                mb = 2
                f.add(("fse_log", name, log))
                if -1 in norm:
                    f.add(("fse", "below_one"))
                zeros = max((len(r) for r in "".join("0" if c == 0 else "x" for c in norm).split("x")), default=0)
                if zeros > 3:
                    f.add(("fse", "zero_run_gt3"))
            f.add(("table_mode", name, ("predef", "rle", "fse", "repeat")[mb]))
            mode_bits |= mb << (6 - 2 * k)
            tabs[k] = self.tables[k]
        states = {k: fse_states(tabs[k][0], codes[k]) for k in (LL, OF, ML)}
        fields = [(states[LL][0], tabs[LL][1]), (states[OF][0], tabs[OF][1]), (states[ML][0], tabs[ML][1])]
        for i in range(n):
            fields += list(extra[i])
            if i + 1 < n:
                for k in (LL, ML, OF):
                    u, nxt = states[k][i], states[k][i + 1]
                    sym, bits, base = tabs[k][0][u]
                    fields.append((nxt - base, bits))
        per_seq = max(sum(b for _, b in e) for e in extra) + sum(t[1] for t in tabs.values())
        if per_seq > 64:
            f.add(("seq", "bits_gt64"))
        return head + bytes([mode_bits]) + desc + back(fields)

    # ---- the frame
    def bytes(self):
        data = self.header()
        for i, (btype, body, size) in enumerate(self.blocks):
            last = i == len(self.blocks) - 1
            data += struct.pack("<I", int(last) | btype << 1 | size << 3)[:3] + body
        if self.checksum:
            data += struct.pack("<I", xxh64(self.out) & 0xffffffff)
        return data

    def build(self):
        assert not self.invalid
        return self.bytes(), bytes(self.out), frozenset(self.features)


def _rng(seed):
    return np.random.default_rng(seed)


def _text(rng, n, alphabet=b"ACGT"):
    return bytes(np.frombuffer(alphabet, np.uint8)[rng.integers(0, len(alphabet), n)])


def fib_lengths(symbols, top):
    """A complete code with lengths 1, 2, .., top - 1, top, top on the given top + 1 symbols."""
    assert len(symbols) == top + 1
    return {s: min(i + 1, top) for i, s in enumerate(symbols)}


def zstd_valid():
    """[(name, stream, expected, features)]: valid frames over every branch the decoder has."""
    out = []

    def add(name, fr):
        out.append((name,) + fr.build())

    rng = _rng(1)
    # frame headers: every Frame_Content_Size width and its edges, window descriptors, checksums, skippable frames
    for fcs, nb, single in ((0, 1, True), (255, 1, True), (256, 2, False), (65791, 2, True), (65792, 4, True),
                            (300, 8, False), (70000, 8, True), (1000, 4, False)):
        data = _text(rng, fcs)
        fr = Frame(fcs=fcs, fcs_bytes=nb, single=single, checksum=fcs % 2 == 1, window_log=17)
        if fcs > BLOCK_MAX // 2:
            fr.raw(data[:fcs // 2]).raw(data[fcs // 2:])
        else:
            fr.raw(data)
        add(f"fcs {fcs} in {nb} bytes", fr)
    add("no fcs, window 2^10 * 1.875, checksum", Frame(window_log=10, window_mantissa=7, checksum=True)
        .raw(b"x" * 5).rle(ord("y"), 3000).raw(b"z"))
    add("empty frame", Frame(fcs=0, single=True).raw(b""))
    add("rle block", Frame(fcs=BLOCK_MAX, single=True).rle(7, BLOCK_MAX))
    two = Frame(checksum=True).raw(b"first frame").build()
    three = Frame(fcs=4, single=True).rle(1, 4).build()
    skip = struct.pack("<II", 0x184D2A5A, 5) + b"skip!"
    out.append(("two frames around a skippable frame", two[0] + skip + three[0], two[1] + three[1],
                two[2] | three[2] | {("skippable",), ("frames", 2)}))

    # literals: raw and RLE with 1-, 2- and 3-byte headers, then matches over them
    fr = Frame(checksum=True)
    for hl, n in ((1, 20), (2, 31), (2, 4000), (3, 5000)):
        fr.compressed(fr.lit_raw(_text(rng, n), hl), [(n // 2, 7, 1 + 3)])
    for hl, n in ((1, 31), (2, 1000), (3, 70000)):
        fr.compressed(fr.lit_rle(65 + hl, n, hl), [(n // 3, 40, 2), (0, 5, 1)])
    add("raw and rle literals, all header sizes", fr)

    # Huffman literals: direct and FSE weights, 1 and 4 streams, 10-, 14- and 18-bit sizes, 11-bit codes, Treeless
    syms = list(range(97, 109))
    eleven = fib_lengths(syms, 11)                                        # codes of 1 .. 11 bits, direct weights
    lits = rng.choice(syms, 900, p=np.array([2.0 ** -eleven[s] for s in syms])).astype(np.uint8).tobytes()
    lits += bytes(syms)                                                   # every code once at least
    fr = Frame(checksum=True)
    fr.compressed(fr.lit_huffman(lits, eleven, streams=1, weights="direct"), [(100, 20, 50 + 3)])
    fr.compressed(fr.lit_huffman(lits[:500], None, streams=4, sf=1), [(0, 30, 1)])   # Treeless, same block order
    fr.raw(b"raw block between")
    fr.compressed(fr.lit_raw(b"abc"), [(3, 4, 2)])                        # a block that leaves the tree alone
    fr.compressed(fr.lit_huffman(lits[::-1], None, streams=1), [])        # Treeless two blocks after the tree
    add("11-bit huffman codes, direct weights, treeless later", fr)

    wide = dict(zip(rng.permutation(256).tolist(), [7] * 64 + [8] * 64 + [9] * 128))   # 255 FSE-coded weights
    lits = rng.integers(0, 256, 12000, dtype=np.uint8).tobytes()
    fr = Frame(checksum=True)
    fr.compressed(fr.lit_huffman(lits, wide, streams=4, sf=2, wlog=6), [(1000, 300, 3 + 200)])
    fr.compressed(fr.lit_huffman(lits[:9], wide, streams=4, sf=3, wlog=5, below_one=(2,)), [])  # last stream empty
    fr.compressed(fr.lit_huffman(lits[:6], None, streams=4, sf=3), [])
    add("255 fse weights, 14- and 18-bit sizes, empty 4th stream", fr)

    fr = Frame(checksum=True)
    big = _text(rng, 100000, b"ACGTN")
    fr.compressed(fr.lit_huffman(big, lengths_for(big, 11), streams=4, sf=3), [(70000, 50, 3 + 1)])
    add("18-bit literal sizes, 100 kB of literals", fr)

    # sequences: every literal-length and match-length code with extra bits, the 3-byte count, long bit budgets
    fr = Frame(window_log=18, checksum=True)
    fr.raw(_text(rng, 16))
    seqs = []
    for c in range(16, 36):
        ll = LL_BASE[c] + (1 << LL_BITS[c]) - 1 if c < 33 else LL_BASE[c] + 1234
        seqs.append((ll, 3, 1))
    lits = _text(rng, sum(s[0] for s in seqs))
    seqs_a = seqs[:17]
    seqs_b = seqs[17:]
    la = sum(s[0] for s in seqs_a)
    fr.compressed(fr.lit_raw(lits[:la]), seqs_a)
    for ll, ml, ofv in seqs_b:     # LL codes 33..35 need a block each: 16 KiB .. 66 KiB of literals
        fr.compressed(fr.lit_raw(lits[la:la + ll]), [(ll, ml, ofv)])
        la += ll
    add("literal-length codes 16..35", fr)

    fr = Frame(window_log=18, checksum=True)
    fr.raw(_text(rng, 64))
    for group in (range(32, 44), range(44, 49), range(49, 51), (51,), (52,)):
        seqs = [(1, ML_BASE[c] + (1 << ML_BITS[c]) - 1 if c < 52 else ML_BASE[c] + 777, 3 + 64) for c in group]
        fr.compressed(fr.lit_raw(_text(rng, len(seqs))), seqs)
    add("match-length codes 32..52", fr)

    fr = Frame(window_log=18, checksum=True)
    fr.raw(rng.integers(0, 256, BLOCK_MAX, dtype=np.uint8).tobytes()).raw(rng.integers(0, 256, 70000, dtype=np.uint8).tobytes())
    lits = _text(rng, 65600 * 2)
    seqs = [(65536 + 60000, 65539 + 60000, 3 + 190000)]    # OF 17 + ML 16 + LL 16 extra bits and three updates
    fr.compressed(fr.lit_raw(lits[:125536]), seqs, modes=("predef", ("fse", normalize({0: 1, 17: 5}, 8), 8),
                                                          "predef"))
    add("one sequence over more than 64 bits", fr)

    fr = Frame(checksum=True)
    fr.raw(b"01234567")
    nseq = 0x7F00 + 5
    fr.compressed(fr.lit_raw(b""), [(0, 3, 1)] * nseq, modes=("rle", "rle", "rle"))
    fr.compressed(fr.lit_raw(_text(rng, 300)), [(1, 3, 3 + 2)] * 300 + [(0, 4, 1)], nseq_bytes=2)
    add("3-byte sequence count", fr)

    # the four table modes; FSE tables at every accuracy log up to the maximum, zero runs and "less than 1" counts
    fr = Frame(checksum=True)
    fr.raw(_text(rng, 600))
    for log in range(5, 10):
        lcodes = [0, 1, 3, 17, 25]
        mcodes = [0, 5, 33, 40, 43]
        ocodes = [4, 8, 1]
        seqs = []
        for i in range(40):
            lc, mc, oc = lcodes[i % 5], mcodes[(i * 3) % 5], ocodes[i % 3]
            ofv = (1 << oc) + int(rng.integers(0, 1 << oc))
            seqs.append((LL_BASE[lc] + int(rng.integers(0, 1 << LL_BITS[lc])),
                         ML_BASE[mc] + int(rng.integers(0, 1 << ML_BITS[mc])), ofv))
        lits = _text(rng, sum(s[0] for s in seqs))
        lnorm = normalize({c: 3 for c in lcodes}, log, below_one=(25,))
        mnorm = normalize({c: 3 for c in mcodes} | {52: 1}, log, below_one=(52,))
        onorm = normalize({c: 3 for c in ocodes} | {0: 1}, min(log, 8), below_one=(0,))
        fr.compressed(fr.lit_raw(lits), seqs, modes=(("fse", lnorm, log), ("fse", onorm, min(log, 8)),
                                                     ("fse", mnorm, log)))
        if log == 7:
            fr.compressed(fr.lit_raw(lits), seqs, modes=("repeat", "repeat", "repeat"))
    add("fse tables at accuracy logs 5..9, repeat mode", fr)

    fr = Frame(checksum=True)
    fr.raw(_text(rng, 100))
    fr.compressed(fr.lit_raw(_text(rng, 120)), [(40, 70, 3 + 50)] * 3, modes=("rle", "rle", "rle"))  # LL 28 ML 38
    fr.compressed(fr.lit_raw(b""), [(0, 3, 3 + 50)], modes=("rle", "repeat", "predef"))
    add("rle tables with extra bits, repeat of rle", fr)

    # repeat offsets: every Offset_Value 1..3 with and without literals, the LL == 0, value 3 rule (Rep1 - 1)
    fr = Frame(checksum=True)
    fr.raw(_text(rng, 64))
    seqs = [(2, 4, 3 + 10), (3, 5, 3 + 20), (1, 4, 3 + 30), (1, 3, 1), (1, 3, 2), (1, 3, 3), (0, 3, 1), (0, 3, 2),
            (0, 3, 3), (2, 3, 3 + 7), (0, 4, 3), (0, 5, 1), (4, 6, 2)]
    fr.compressed(fr.lit_raw(_text(rng, sum(s[0] for s in seqs))), seqs)
    add("repeat offsets", fr)

    # offsets at the window: exactly the window size (descriptor 2^10), and from blocks before a block's literals
    fr = Frame(window_log=10, checksum=True)
    fr.raw(_text(rng, 1024))
    fr.compressed(fr.lit_raw(b"q"), [(1, 8, 3 + 1024)])
    fr.features.add(("offset", "window"))
    add("offset of exactly the window size", fr)
    fr = Frame(fcs=2900, single=True)
    fr.raw(_text(rng, 2000))
    fr.compressed(fr.lit_raw(b"w" * 500), [(500, 400, 3 + 2500)])
    fr.features.add(("offset", "window"))
    add("single-segment offset of the whole output", fr)

    # an exactly sized output: compressed-block literals staged at the slot's end while matches read earlier blocks
    fr = Frame()
    first = _text(rng, 3000)
    fr.compressed(fr.lit_huffman(first, lengths_for(first, 11), streams=4), [])
    lits = _text(rng, 2000)
    fr.compressed(fr.lit_huffman(lits, None, streams=4), [(100, 2900, 3 + 2500), (500, 1000, 3 + 4000), (1000, 50, 1)])
    fr.compressed(fr.lit_rle(9, 300), [(200, 3000, 3 + 9000)])
    fr.features.add(("exact_slot", "staged_literals"))
    add("matches from earlier blocks under staged literals", fr)

    # a compressed block of exactly 128 KiB
    fr = Frame(checksum=True)
    body = rng.integers(0, 256, BLOCK_MAX - 3 - 1, dtype=np.uint8).tobytes()
    fr.compressed(fr.lit_raw(body, 3), [])
    add("compressed block of 128 KiB", fr)
    return out


def zstd_malformed():
    """[(name, stream, capacity, status, libzstd_rejects)]: each stream fails one check of the decoder.
    libzstd_rejects is False where the decoder is deliberately stricter than libzstd."""
    rng = _rng(2)
    out = []

    def add(name, fr_or_bytes, status, cap=None, libzstd=True):
        stream = fr_or_bytes if isinstance(fr_or_bytes, bytes) else fr_or_bytes.bytes()
        out.append((name, stream, 4096 if cap is None else cap, status, libzstd))

    good = Frame(fcs=5, single=True).raw(b"hello").bytes()
    add("bad magic", b"\x27" + good[1:], Z_MAGIC)
    add("reserved header bit", good[:4] + bytes([good[4] | 8]) + good[5:], Z_FRAME_HEADER)
    add("dictionary id", Frame(fcs=5, single=True, dict_id=7, did_bytes=1).raw(b"hello"), Z_FRAME_HEADER)
    add("dictionary id, 4 bytes", Frame(dict_id=1 << 31, did_bytes=4).raw(b"hello"), Z_FRAME_HEADER)
    wide = Frame().raw(b"hello").bytes()
    add("window above 2^31", wide[:5] + bytes([(32 - 10) << 3]) + wide[6:], Z_FRAME_HEADER)
    blk = Frame(fcs=5, single=True).raw(b"hello").bytes()
    add("block type 3", blk[:6] + bytes([blk[6] | 6]) + blk[7:], Z_BLOCK_TYPE)
    fr = Frame()
    fr.blocks.append((2, bytes(BLOCK_MAX + 1), BLOCK_MAX + 1))
    add("compressed block over 128 KiB", fr, Z_BLOCK_TYPE, cap=1 << 18)
    fr = Frame()
    fr.blocks.append((2, bytes([0x03 | 5 << 4, 1 << 6, 0]) + b"\0\0", 5))
    add("treeless with no tree", fr, Z_LITERALS)
    fr = Frame()
    fr.blocks.append((2, bytes([10 << 3]) + b"abc", 4))
    add("raw literals past the block", fr, Z_LITERALS)
    fr = Frame()
    head = (2 | 3 << 2 | 0x3ffff << 4 | 1 << 22).to_bytes(5, "little")     # 18-bit sizes: 262143 literals
    fr.blocks.append((2, head + b"\0\0", 7))
    add("huffman literals past 128 KiB", fr, Z_LITERALS)
    lens = fib_lengths(list(range(97, 109)), 11)
    fr = Frame()
    fr.compressed(fr.lit_huffman(b"abcdefghijkl" * 3, lens, streams=1, weights="direct"), [])
    s = bytearray(fr.bytes())
    s[len(fr.header()) + 3 + 3 + 1] = 0xcc     # past the block and literals headers and the weights' header byte:
    #                                            weights 12, 12 make codes longer than 11 bits
    add("huffman weights above 11 bits", bytes(s), Z_HUFFMAN)
    fr = Frame()
    fr.compressed(fr.lit_huffman(b"abcdefghijkl" * 3, lens, streams=1, weights="direct"), [])
    bad = bytearray(fr.blocks[0][1])
    bad[-2] ^= 0x80                    # the stream's last byte (before the sequence count): its end marker moves
    fr2 = Frame()
    fr2.blocks.append((2, bytes(bad), len(bad)))
    add("huffman stream not consumed exactly", fr2, Z_HUFFMAN)
    fr = Frame()
    fr.blocks.append((2, bytes([0x00, 0x01, 0x80, 0x0f, 0x00]), 5))
    add("fse accuracy log 20", fr, Z_FSE)
    fr = Frame()
    fr.blocks.append((2, bytes([0x00, 0x01, 0xfc, 0x01]), 4))
    add("repeat mode with no table", fr, Z_FSE)
    fr = Frame()
    fr.blocks.append((2, bytes([0x00, 0x01, 0x55, 0, 5, 0, 0x20]), 7))
    add("reserved mode bits", fr, Z_SEQUENCES)
    fr = Frame()
    fr.blocks.append((2, bytes([0x00, 0x00, 0x77]), 3))
    add("bytes after a zero sequence count", fr, Z_SEQUENCES)
    fr = Frame()
    fr.blocks.append((2, bytes([0x00, 0xff, 0x00]), 3))
    add("3-byte sequence count cut short", fr, Z_SEQUENCES)
    fr = Frame()
    fr.raw(b"abcdefgh")
    fr.blocks.append((2, bytes([8 << 3]) + b"abcdefgh" + bytes([0x01, 0x54, 8, 0, 0, 0x03]), 15))
    add("sequence bits left over", fr, Z_SEQUENCES)
    fr = Frame()
    fr.blocks.append((2, bytes([2 << 3]) + b"ab" + bytes([0x01, 0x54, 8, 0, 0, 0x01]), 9))
    add("literal length past the literals", fr, Z_SEQUENCES)
    fr = Frame()
    fr.blocks.append((2, bytes([0x00, 0x01, 0x54, 0, 5, 0, 0x20]), 7))
    add("offset before the frame", fr, Z_OFFSET)
    fr = Frame(window_log=10)
    fr.raw(_text(rng, 1100))
    fr.compressed(fr.lit_raw(b"q"), [(1, 8, 3 + 1025)])
    add("offset one past the window", fr, Z_OFFSET, libzstd=False)
    add("repeat offset Rep1 - 1 of zero", Frame().raw(b"a").compressed(Frame().lit_raw(b""), [(0, 3, 3)]), Z_OFFSET,
        libzstd=False)
    add("output past capacity", Frame(fcs=10, single=True).raw(b"0123456789"), Z_OVERFLOW, cap=9)
    add("output past capacity, no fcs", Frame().rle(1, 50), Z_OVERFLOW, cap=49)
    add("content size differs", Frame(fcs=11, single=True).raw(b"0123456789"), Z_CONTENT_SIZE)
    add("frame cut short", Frame(fcs=10, single=True).raw(b"0123456789").bytes()[:-3], Z_TRUNCATED)
    add("no last block", Frame(fcs=10, single=True).raw(b"0123456789").bytes()[:-13] + struct.pack("<I", 10 << 3)[:3]
        + b"0123456789", Z_TRUNCATED)
    add("skippable frame cut short", struct.pack("<II", 0x184D2A50, 10) + b"abc", Z_TRUNCATED)
    chk = Frame(checksum=True).raw(b"0123456789").bytes()
    add("checksum differs", chk[:-1] + bytes([chk[-1] ^ 1]), Z_CHECKSUM)
    add("checksum cut short", chk[:-2], Z_TRUNCATED)
    return out


# ============================================================================================================= DEFLATE
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227,
            258]
LEN_BITS = [0] * 8 + [1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577]
DIST_BITS = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 30


def canonical(lengths):
    """Canonical codes (RFC 1951 section 3.2.2) of a list of code lengths: [code or None]."""
    count = [0] * 16
    for l in lengths:
        count[l] += 1
    count[0] = 0
    nxt, c = [0] * 16, 0
    for l in range(1, 16):
        c = (c + count[l - 1]) << 1
        nxt[l] = c
    out = []
    for l in lengths:
        out.append(nxt[l] if l else None)
        if l:
            nxt[l] += 1
    return out


def len_symbol(n):
    i = 28 if n == 258 else max(i for i in range(28) if LEN_BASE[i] <= n)
    return 257 + i, LEN_BITS[i], n - LEN_BASE[i]


def dist_symbol(d):
    i = max(i for i in range(30) if DIST_BASE[i] <= d)
    return i, DIST_BITS[i], d - DIST_BASE[i]


def rle_tokens(lengths, style="zlib"):
    """Code-length tokens [(symbol, extra)] of the concatenated lit/len and distance lengths.  style "zlib": runs of
    16 / 17 / 18 where they fit; "plain": every length written alone."""
    toks, i, n = [], 0, len(lengths)
    while i < n:
        v, run = lengths[i], 1
        while i + run < n and lengths[i + run] == v:
            run += 1
        i += run
        if style == "plain":
            toks += [(v, 0)] * run
            continue
        if v == 0:
            while run >= 11:
                r = min(run, 138)
                toks.append((18, r - 11))
                run -= r
            if run >= 3:
                toks.append((17, run - 3))
                run = 0
        else:
            toks.append((v, 0))
            run -= 1
            while run >= 3:
                r = min(run, 6)
                toks.append((16, r - 3))
                run -= r
        toks += [(v, 0)] * run
    return toks


def expand_tokens(tokens):
    out = []
    for sym, ex in tokens:
        if sym < 16:
            out.append(sym)
        elif sym == 16:
            out += [out[-1]] * (3 + ex)
        elif sym == 17:
            out += [0] * (3 + ex)
        else:
            out += [0] * (11 + ex)
    return out


class Deflate:
    """A raw DEFLATE stream under construction; parse items are a byte (literal) or (length, distance)."""

    def __init__(self):
        self.w, self.out, self.features = Bits(), bytearray(), set()

    def _body(self, parse, lit_codes, dist_codes):
        syms = [len_symbol(i[0])[0] if isinstance(i, tuple) else i for i in parse] + [256]
        dsyms = [dist_symbol(i[1])[0] for i in parse if isinstance(i, tuple)]
        assert all(lit_codes[s][1] for s in syms) and all(dist_codes[s][1] for s in dsyms), "a symbol with no code"
        for item in parse:
            if isinstance(item, int):
                self.w.code(*lit_codes[item])
                self.out.append(item)
                continue
            n, d = item
            s, nb, ex = len_symbol(n)
            self.w.code(*lit_codes[s]).put(ex, nb)
            ds, dnb, dex = dist_symbol(d)
            self.w.code(*dist_codes[ds]).put(dex, dnb)
            assert 0 < d <= len(self.out)
            for _ in range(n):
                self.out.append(self.out[-d])
            self.features.update({("inflate_dist_len", dist_codes[ds][1]), ("inflate_dist_sym", ds)})
            self.features.add(("inflate_len_sym", s))
            if d == 32768:
                self.features.add(("inflate", "distance_32768"))
        for item in parse:
            if isinstance(item, int):
                self.features.add(("inflate_lit_len", lit_codes[item][1]))
            else:
                self.features.add(("inflate_lit_len", lit_codes[len_symbol(item[0])[0]][1]))
        self.w.code(*lit_codes[256])
        self.features.add(("inflate_lit_len", lit_codes[256][1]))

    def stored(self, data, last=False):
        if self.w.n:
            self.features.add(("inflate", "stored_after_midbyte"))
        self.w.put(int(last), 1).put(0, 2).align()
        self.w.put(len(data), 16).put(len(data) ^ 0xffff, 16)
        for b in data:
            self.w.put(b, 8)
        self.out += data
        self.features.add(("inflate", "stored_empty" if not data else "stored"))
        return self

    def fixed(self, parse, last=False):
        self.w.put(int(last), 1).put(1, 2)
        self._body(parse, list(zip(canonical(FIXED_LIT), FIXED_LIT)), list(zip(canonical(FIXED_DIST), FIXED_DIST)))
        self.features.add(("inflate", "fixed"))
        return self

    def dynamic(self, parse, lit_lens=None, dist_lens=None, tokens=None, style="zlib", hclen=None, last=False):
        """A dynamic block: lit_lens (HLIT of them) and dist_lens (HDIST) default to Huffman codes of the parse's
        symbols; tokens (the code-length runs) default to rle_tokens(style); hclen to the fewest that cover them."""
        if lit_lens is None or dist_lens is None:
            lf, df = {256: 1}, {}
            for item in parse:
                if isinstance(item, int):
                    lf[item] = lf.get(item, 0) + 1
                else:
                    s = len_symbol(item[0])[0]
                    lf[s] = lf.get(s, 0) + 1
                    ds = dist_symbol(item[1])[0]
                    df[ds] = df.get(ds, 0) + 1
            if lit_lens is None:
                ll = limited(lf, 15)
                lit_lens = [ll.get(s, 0) for s in range(max(257, max(ll) + 1))]
            if dist_lens is None:
                dl = limited(df, 15) if df else {}
                dist_lens = [dl.get(s, 0) for s in range(max(1, max(dl, default=0) + 1))]
        self.header(lit_lens, dist_lens, tokens, style, hclen, last)
        self._body(parse, list(zip(canonical(lit_lens), lit_lens)), list(zip(canonical(dist_lens), dist_lens)))
        return self

    def header(self, lit_lens, dist_lens, tokens=None, style="zlib", hclen=None, last=False, hdist=None):
        """A dynamic block's header.  tokens, when given, are written as they are (valid or not); hdist overrides
        the HDIST field."""
        hlit = len(lit_lens)
        if tokens is None:
            tokens = rle_tokens(list(lit_lens) + list(dist_lens), style)
            assert expand_tokens(tokens) == list(lit_lens) + list(dist_lens)
        hdist = len(dist_lens) if hdist is None else hdist
        cf = {}
        for s, _ in tokens:
            cf[s] = cf.get(s, 0) + 1
        cl = limited(cf, 7)
        cl_lens = [cl.get(s, 0) for s in range(19)]
        if hclen is None:
            hclen = max(4, max(i + 1 for i, s in enumerate(CL_ORDER) if cl_lens[s]))
        assert all(cl_lens[s] == 0 for s in CL_ORDER[hclen:])
        self.w.put(int(last), 1).put(2, 2).put(hlit - 257, 5).put(hdist - 1, 5).put(hclen - 4, 4)
        for s in CL_ORDER[:hclen]:
            self.w.put(cl_lens[s], 3)
        cl_codes = list(zip(canonical(cl_lens), cl_lens))
        at = 0
        for s, ex in tokens:
            self.w.code(*cl_codes[s])
            n = 1
            if s >= 16:
                self.w.put(ex, (2, 3, 7)[s - 16])
                n = 3 + ex if s < 18 else 11 + ex
                if at < hlit < at + n:
                    self.features.add(("inflate_repeat_across", s))
            at += n
        f = self.features
        f.update({("hlit", hlit), ("hdist", hdist), ("hclen", hclen), ("inflate", "dynamic")})
        if not any(dist_lens):
            f.add(("inflate", "no_distance_codes"))
        if sum(1 for l in dist_lens if l) == 1 and max(dist_lens) == 1:
            f.add(("inflate", "single_distance_code"))
        return self

    def build(self):
        return self.w.bytes(), bytes(self.out), frozenset(self.features)


def limited(freq, limit):
    """Huffman code lengths {symbol: bits} of {symbol: frequency} no longer than limit (frequencies halved until they
    fit); a lone symbol gets a 1-bit code."""
    if len(freq) == 1:
        return {next(iter(freq)): 1}
    while True:
        d = huffman_depths(freq)
        if max(d.values()) <= limit:
            return d
        freq = {s: (c + 1) // 2 for s, c in freq.items()}


def inflate_valid():
    """[(name, raw DEFLATE, expected, features)]: valid streams over every branch of the inflater."""
    rng = _rng(3)
    out = []

    def add(name, d):
        out.append((name,) + d.build())

    # lit/len codes of 1 .. 15 bits and distance codes of 1 .. 15 bits (Fibonacci-shaped sets), every code used
    lit_syms = [65, 66, 67, 68, 69, 70, 71, 72, 256, 257, 265, 270, 280, 284, 285, 90]
    lit_lens = [0] * 286
    for i, s in enumerate(lit_syms):
        lit_lens[s] = min(i + 1, 15)
    dist_syms = [0, 3, 4, 8, 10, 13, 15, 17, 19, 21, 23, 25, 26, 27, 28, 29]
    dist_lens = [0] * 30
    for i, s in enumerate(dist_syms):
        dist_lens[s] = min(i + 1, 15)
    d = Deflate()
    d.stored(rng.integers(65, 73, 33000).astype(np.uint8).tobytes())
    parse = list(b"ABCDEFGHZ")
    length_of = {257: 3, 265: 12, 270: 24, 280: 130, 284: 257, 285: 258}
    for i, ds in enumerate(dist_syms):
        parse.append((length_of[[257, 265, 270, 280, 284, 285][i % 6]],
                      DIST_BASE[ds] + (1 << DIST_BITS[ds]) - 1 if ds < 29 else 32768))
    parse += [(258, 1), (3, 32768), 90, 72]
    d.dynamic(parse, lit_lens, dist_lens, last=True)
    add("lit/len and distance codes of 1..15 bits, distance 32768, length 258", d)

    # HLIT / HDIST / HCLEN at the ends of their ranges; code-length runs 16, 17 and 18 across the lit/len-distance edge
    data = _text(rng, 3000, b"ACGTacgt")
    d = Deflate()
    lf = limited({b: 1 + data.count(b) for b in set(data)} | {256: 1, 275: 1}, 15)
    ll = [lf.get(s, 0) for s in range(286)]                            # HLIT 286: a zero run from 276 into dist
    dl = [0] * 5 + [1, 1] + [0] * 23                                    # HDIST 30: codes 5 and 6 only
    d.dynamic(list(data[:50]) + [(55, 7)] + list(data[50:]), ll, dl, hclen=19)
    # HLIT 257, HDIST 1 and no distance code at all, HCLEN 5: lengths 8 only (symbols 1..256)
    d.dynamic(list(b"no distance codes"), [0] + [8] * 256, [0])
    # HLIT 258: a 16 run from lengths 256/257 into eight distance codes of 3 bits
    ll = [0] * 258
    ll[97], ll[98], ll[256], ll[257] = 1, 2, 3, 3
    parse = list(b"ab" * 10) + [(3, dd) for dd in (1, 2, 3, 4, 6, 8, 12, 16)]
    d.dynamic(parse, ll, [3] * 8)
    # HLIT 260: a 17 run from lengths 258/259 into three zero distance lengths
    ll = [0] * 260
    ll[97], ll[98], ll[256], ll[257] = 1, 2, 3, 3
    d.dynamic(list(b"ba") + [(3, 9)] * 2, ll, [0, 0, 0, 0, 0, 0, 1])  # one distance code of length 1 (code 6)
    # a fixed block that ends mid-byte, an empty stored block, a stored block after it
    d.fixed(list(b"fixed") + [(258, 3), (3, 1)])
    d.stored(b"")
    d.stored(b"stored after fixed", last=True)
    add("header ranges, runs across the lit/len-distance edge, no or one distance code, stored blocks", d)

    d = Deflate()
    d.stored(bytes(range(256)) * 130)
    d.fixed([(258, 32768), (258, 1), 7, (3, 32768)], last=True)
    add("fixed codes at distance 32768 and length 258", d)

    d = Deflate()
    d.stored(b"", last=True)
    add("one empty stored block", d)
    return out


def _raw(bits_fn):
    w = Bits()
    bits_fn(w)
    return w.bytes()


def inflate_malformed():
    """[(name, raw DEFLATE, ISIZE, CRC32, status)]: each a member that one check of the inflater rejects (BOUNDS, a meta
    row outside the buffers, is the test's to build)."""
    text = b"malformed members " * 4
    good = Deflate().dynamic(list(text), last=True).build()[0]
    crc = zlib.crc32(text)
    out = [("block type 3", _raw(lambda w: w.put(1, 1).put(3, 2).put(0, 16)), 4, 0, I_BLOCK_TYPE),
           ("stored LEN/NLEN", b"\x01" + struct.pack("<HH", 5, 0xfffa ^ 1) + b"hello", 5, zlib.crc32(b"hello"),
            I_STORED_LENGTH)]

    def dyn(lit_lens, dist_lens, tail, hdist=None, tokens=None):
        d = Deflate()
        d.header(lit_lens, dist_lens, tokens=tokens, last=True, hdist=hdist)
        tail(d.w)
        return d.w.put(0, 32).bytes()

    ok_lit = [0] * 97 + [1, 2] + [0] * 157 + [3, 3]   # 'a' 'b', EOB, length 3
    out.append(("HDIST 31", dyn(ok_lit, [1, 1] + [0] * 29, lambda w: None, hdist=31), 4, 0, I_CODE_LENGTHS))
    out.append(("over-subscribed lit/len code", dyn([1, 1, 1] + [0] * 253 + [2], [1, 1], lambda w: None), 4, 0,
                I_CODE_LENGTHS))
    out.append(("incomplete lit/len code", dyn([0] * 97 + [2, 2] + [0] * 157 + [3], [1, 1], lambda w: None), 4, 0,
                I_CODE_LENGTHS))
    out.append(("no end-of-block code", dyn([0] * 97 + [1, 1] + [0] * 158, [1, 1], lambda w: None), 4, 0,
                I_CODE_LENGTHS))
    out.append(("incomplete code-length code", _raw(lambda w: w.put(1, 1).put(2, 2).put(0, 10).put(0, 4).put(1, 3)
                                                    .put(0, 9).put(0, 16)), 4, 0, I_CODE_LENGTHS))
    out.append(("repeat with no previous length", dyn(ok_lit, [1, 1], lambda w: None, tokens=[(16, 0)] + [(0, 0)] * 256),
                4, 0, I_REPEAT))
    out.append(("repeat past HLIT + HDIST", dyn(ok_lit, [1, 1], lambda w: None,
                                               tokens=rle_tokens(ok_lit + [1]) + [(16, 3)]), 4, 0, I_REPEAT))
    out.append(("fixed symbol 286", _raw(lambda w: w.put(1, 1).put(1, 2).code(0xc6, 8).put(0, 16)), 4, 0, I_SYMBOL))
    out.append(("fixed distance code 31", _raw(lambda w: w.put(1, 1).put(1, 2).code(0x30 + 65, 8).code(1, 7)
                                               .code(31, 5).put(0, 16)), 4, 0, I_SYMBOL))
    one_dist = [0, 0, 0, 1]                           # a single distance code of length 1: bit 1 matches nothing
    cl_a = canonical(ok_lit)
    out.append(("unused half of a one-code distance table",
                dyn(ok_lit, one_dist, lambda w: w.code(cl_a[97], 1).code(cl_a[257], 3).code(1, 1)), 4, 0, I_SYMBOL))
    out.append(("length with no distance codes",
                dyn(ok_lit, [0], lambda w: w.code(cl_a[97], 1).code(cl_a[257], 3).put(0, 8)), 4, 0, I_SYMBOL))
    out.append(("distance past the output", dyn(ok_lit, [1, 1], lambda w: w.code(cl_a[97], 1).code(cl_a[257], 3)
                                                .code(1, 1).code(cl_a[256], 3)), 4, 0, I_DISTANCE))
    out.append(("output past ISIZE", good, len(text) - 1, crc, I_OVERFLOW))
    out.append(("output short of ISIZE", good, len(text) + 1, crc, I_SHORT))
    out.append(("stream cut short", good[:len(good) // 2], len(text), crc, I_TRUNCATED))
    out.append(("stored block cut short", b"\x01" + struct.pack("<HH", 10, 0xfff5) + b"abc", 10, 0, I_TRUNCATED))
    out.append(("CRC differs", good, len(text), crc ^ 1, I_CRC))
    return out


def read_dynamic_block(raw):
    """The first block of raw DEFLATE data, a dynamic one: {"lit_lens", "dist_lens", "cl_lens", "cl_counts",
    "lit_counts", "dist_counts"}, the counts being how often the header's runs and the block's body use each symbol."""
    bits = np.unpackbits(np.frombuffer(bytes(raw), np.uint8), bitorder="little").tolist()
    pos = 0

    def take(n):
        nonlocal pos
        v = sum(b << i for i, b in enumerate(bits[pos:pos + n]))
        pos += n
        return v

    def decoder(lens):
        return {(l, c): s for s, (c, l) in enumerate(zip(canonical(lens), lens)) if l}

    def symbol(dec):
        c = 0
        for l in range(1, 16):
            c = c << 1 | take(1)
            if (l, c) in dec:
                return dec[(l, c)]
        raise ValueError("bits that match no code")

    take(1)
    assert take(2) == 2, "not a dynamic block"
    hlit, hdist, hclen = take(5) + 257, take(5) + 1, take(4) + 4
    cl_lens = [0] * 19
    for s in CL_ORDER[:hclen]:
        cl_lens[s] = take(3)
    cl_dec, lens, cl_counts = decoder(cl_lens), [], [0] * 19
    while len(lens) < hlit + hdist:
        s = symbol(cl_dec)
        cl_counts[s] += 1
        lens += [s] if s < 16 else [lens[-1]] * (3 + take(2)) if s == 16 else [0] * (3 + take(3)) if s == 17 else \
            [0] * (11 + take(7))
    lit_lens, dist_lens = lens[:hlit], lens[hlit:]
    lit_dec, dist_dec = decoder(lit_lens), decoder(dist_lens)
    lit_counts, dist_counts = [0] * hlit, [0] * hdist
    while True:
        s = symbol(lit_dec)
        lit_counts[s] += 1
        if s == 256:
            break
        if s > 256:
            take(LEN_BITS[s - 257])
            d = symbol(dist_dec)
            dist_counts[d] += 1
            take(DIST_BITS[d])
    return {"lit_lens": lit_lens, "dist_lens": dist_lens, "cl_lens": cl_lens, "cl_counts": cl_counts,
            "lit_counts": lit_counts, "dist_counts": dist_counts}


def deep_code_payload(seed=0, n=65280, n_fib=14, n_flat=128):
    """n shuffled bytes whose optimal literal/length code is deeper than 15 bits: n_fib bytes with the Fibonacci-shaped
    counts 1, 2, 3, 5, .. (with the end-of-block symbol's count of one they make a chain one level deeper per symbol)
    and n_flat bytes sharing the rest evenly.  Bytes are then swapped until no 3 bytes recur within 4096 and no 4 within
    32768, so that an LZ77 parse finds no match and the literal counts stay exactly these."""
    rng = _rng(seed)
    fib = [1, 2]
    while len(fib) < n_fib:
        fib.append(fib[-1] + fib[-2])
    rest = n - sum(fib)
    counts = fib + [rest // n_flat + (i < rest % n_flat) for i in range(n_flat)]
    data = np.concatenate([np.full(c, s, np.uint8) for s, c in zip(rng.permutation(256), counts)])
    rng.shuffle(data)
    for _ in range(100):
        a = data.astype(np.int64)
        k3 = (a[:-2] << 16 | a[1:-1] << 8 | a[2:]).tolist()
        k4 = (a[:-3] << 24 | a[1:-2] << 16 | a[2:-1] << 8 | a[3:]).tolist()
        seen3, seen4, bad = {}, {}, []
        for i, k in enumerate(k3):
            if i - seen3.get(k, -1 << 20) <= 4096 or (i < len(k4) and i - seen4.get(k4[i], -1 << 20) <= 32768):
                bad.append(i)
            seen3[k] = i
            if i < len(k4):
                seen4[k4[i]] = i
        if not bad:
            return data.tobytes()
        for i in bad:
            j = int(rng.integers(0, n))
            data[i + 1], data[j] = data[j], data[i + 1]
    raise AssertionError("no match-free arrangement found")
