"""
DEFLATE test members for the BGZF reader: valid raw streams from zlib over the settings htslib and libdeflate use and
the edges of RFC 1951, and one crafted malformed stream per B200_INFLATE_* status.  zlib, struct and numpy only.
"""
import struct
import zlib

import numpy as np

OK, BLOCK_TYPE, STORED_LENGTH, CODE_LENGTHS, REPEAT, SYMBOL, DISTANCE, OVERFLOW, SHORT, TRUNCATED, CRC, BOUNDS = range(12)
EOF_MARKER = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


class Bits:
    """A DEFLATE bit stream: fields LSB first, Huffman codes MSB first."""

    def __init__(self):
        self.bits = []

    def put(self, value, n):
        self.bits += [(value >> i) & 1 for i in range(n)]
        return self

    def code(self, code, n):
        self.bits += [(code >> (n - 1 - i)) & 1 for i in range(n)]
        return self

    def bytes(self):
        b = self.bits + [0] * (-len(self.bits) % 8)
        return bytes(sum(b[i + k] << k for k in range(8)) for i in range(0, len(b), 8))


def fixed_lit(bw, sym):
    """A literal/length symbol with the fixed code (RFC 1951 section 3.2.6)."""
    if sym < 144:
        return bw.code(0x30 + sym, 8)
    if sym < 256:
        return bw.code(0x190 + sym - 144, 9)
    if sym < 280:
        return bw.code(sym - 256, 7)
    return bw.code(0xc0 + sym - 280, 8)


def deflate(data, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, flush_at=()):
    """Raw DEFLATE of data, with Z_FULL_FLUSH / Z_SYNC_FLUSH (alternating) at the offsets in flush_at."""
    c = zlib.compressobj(level, zlib.DEFLATED, -15, 9, strategy)
    out, prev = [], 0
    for k, cut in enumerate(sorted(flush_at)):
        out.append(c.compress(data[prev:cut]) + c.flush(zlib.Z_FULL_FLUSH if k % 2 else zlib.Z_SYNC_FLUSH))
        prev = cut
    out.append(c.compress(data[prev:]) + c.flush())
    return b"".join(out)


def payloads(seed=0):
    """{name: bytes}: random bytes, the two farthest periods, single-byte runs, SAM text and BAM records."""
    rng = np.random.default_rng(seed)
    rand = rng.integers(0, 256, 65536, dtype=np.uint8).tobytes()
    p32768 = rng.integers(0, 256, 32768, dtype=np.uint8).tobytes()
    p32769 = rng.integers(0, 256, 32769, dtype=np.uint8).tobytes()
    runs = b"".join(bytes([int(b)]) * int(n) for b, n in zip(rng.integers(0, 256, 400), rng.integers(1, 700, 400)))
    sam, bam = [], []
    for i in range(60):
        n = int(rng.integers(50, 1500))
        seq = "".join(rng.choice(list("ACGT"), n))
        qual = bytes((np.clip(rng.normal(20, 6, n), 1, 50)).astype(np.uint8))
        sam.append(f"read_{i}\t{16 * (i % 2)}\t*\t0\t0\t*\t*\t0\t0\t{seq}\t{(np.frombuffer(qual, np.uint8) + 33).tobytes().decode()}"
                   f"\tqs:i:20\n")
        name = f"read_{i}".encode() + b"\0"
        nt = np.frombuffer(seq.encode(), np.uint8)
        code = np.zeros(256, np.uint8)
        code[[ord(c) for c in "ACGT"]] = [1, 2, 4, 8]
        nib = np.append(code[nt], np.uint8(0)) if n % 2 else code[nt]
        packed = (nib[0::2] << 4 | nib[1::2]).astype(np.uint8).tobytes()
        body = struct.pack("<iiBBHHHIiii", -1, -1, len(name), 0, 4680, 0, 4, n, -1, -1, 0) + name + packed + qual
        bam.append(struct.pack("<i", len(body)) + body)
    return {"random": rand, "period32768": (p32768 * 3)[:65536], "period32769": (p32769 * 2)[:65536],
            "runs": runs[:65536], "sam": "".join(sam).encode()[:65536], "bam": b"".join(bam)[:65536]}


def valid_members(seed=0):
    """[(name, raw DEFLATE, uncompressed bytes)] over levels, strategies, flushes, sizes and random cut points."""
    rng = np.random.default_rng(seed + 1)
    out = []
    strategies = {"default": zlib.Z_DEFAULT_STRATEGY, "fixed": zlib.Z_FIXED, "huffman": zlib.Z_HUFFMAN_ONLY,
                  "rle": zlib.Z_RLE, "filtered": zlib.Z_FILTERED}
    for pname, data in payloads(seed).items():
        sizes = sorted({0, 1, 65280, 65536, int(rng.integers(2, 65280)), int(rng.integers(2, 65280))})
        for size in sizes:
            d = data[:size]
            for level in (0, 1, 6, 9):
                out.append((f"{pname}-{size}-l{level}", deflate(d, level), d))
            for sname, strategy in strategies.items():
                if sname != "default":
                    out.append((f"{pname}-{size}-{sname}", deflate(d, 6, strategy), d))
            cuts = sorted(int(c) for c in rng.integers(0, size + 1, 3))
            out.append((f"{pname}-{size}-flush", deflate(d, 6, flush_at=cuts + [size]), d))
    return out


def malformed():
    """[(name, raw DEFLATE, ISIZE, status)]: each a stream one check rejects."""
    out = [("block type 3", Bits().put(1, 1).put(3, 2).put(0, 16).bytes(), 4, BLOCK_TYPE),
           ("stored LEN/NLEN", b"\x01" + struct.pack("<HH", 5, 0xfffe ^ 1) + b"hello", 5, STORED_LENGTH)]
    # dynamic headers: BFINAL 1, BTYPE 2, HLIT - 257, HDIST - 1, HCLEN - 4, then 3-bit code-length code lengths
    out.append(("HLIT 287", Bits().put(1, 1).put(2, 2).put(30, 5).put(0, 5).put(0, 4).put(0, 24).bytes(), 4, CODE_LENGTHS))
    over = Bits().put(1, 1).put(2, 2).put(0, 5).put(0, 5).put(15, 4)
    for _ in range(19):
        over.put(1, 3)                    # nineteen codes of length 1: over-subscribed
    out.append(("over-subscribed", over.bytes(), 4, CODE_LENGTHS))

    def two_symbol_cl(a, b):
        """A header whose code-length code is {a: 0, b: 1} (one bit each); symbols in the order of RFC 1951 3.2.7."""
        order = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
        bw = Bits().put(1, 1).put(2, 2).put(0, 5).put(0, 5).put(15, 4)
        for s in order:
            bw.put(1 if s in (a, b) else 0, 3)
        return bw

    out.append(("repeat first", two_symbol_cl(0, 16).code(1, 1).put(0, 2).put(0, 32).bytes(), 4, REPEAT))
    past = two_symbol_cl(0, 18)
    for _ in range(2):
        past.code(1, 1).put(127, 7)       # 138 + 138 zeros > HLIT + HDIST = 258
    out.append(("repeat past end", past.put(0, 16).bytes(), 4, REPEAT))
    incomplete = Bits().put(1, 1).put(2, 2).put(0, 5).put(0, 5).put(0, 4).put(1, 3).put(0, 9).put(0, 16)
    out.append(("incomplete cl code", incomplete.bytes(), 4, CODE_LENGTHS))
    out.append(("symbol 286", fixed_lit(Bits().put(1, 1).put(1, 2), 286).put(0, 16).bytes(), 4, SYMBOL))
    d30 = fixed_lit(fixed_lit(Bits().put(1, 1).put(1, 2), 65), 257).code(30, 5).put(0, 16)
    out.append(("distance code 30", d30.bytes(), 4, SYMBOL))
    far = fixed_lit(fixed_lit(Bits().put(1, 1).put(1, 2), 65), 257).code(1, 5)    # length 3, distance 2, after 1 byte
    out.append(("distance too far", fixed_lit(far, 256).bytes(), 4, DISTANCE))
    text = bytes(range(100))
    out.append(("output past ISIZE", deflate(text), 50, OVERFLOW))
    out.append(("output short of ISIZE", deflate(text), 150, SHORT))
    out.append(("stored block cut", b"\x01" + struct.pack("<HH", 10, 0xfff5) + b"abc", 10, TRUNCATED))
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    out.append(("no final block", c.compress(text) + c.flush(zlib.Z_SYNC_FLUSH), 100, TRUNCATED))
    return out


def member(raw, data=None, isize=None, crc=None, extra=b""):
    """One BGZF member around raw DEFLATE data: the BC subfield after the optional extra subfields."""
    xlen = len(extra) + 6
    bsize = 12 + xlen + len(raw) + 8
    head = b"\x1f\x8b\x08\x04" + struct.pack("<IBBH", 0, 0, 0xff, xlen) + extra + b"BC" + struct.pack("<HH", 2, bsize - 1)
    isize = len(data) if isize is None else isize
    crc = zlib.crc32(data) if crc is None else crc
    return head + raw + struct.pack("<II", crc & 0xffffffff, isize)


def bgzf_file(data, rng, max_member=65280, level=6, empty_at=None):
    """A BGZF file from zlib: members of random sizes, an empty member after member `empty_at`, the EOF marker."""
    out, pos, k = [], 0, 0
    while pos < len(data):
        n = int(rng.integers(1, max_member + 1))
        out.append(member(deflate(data[pos:pos + n], level), data[pos:pos + n]))
        pos += n
        if k == empty_at:
            out.append(member(deflate(b"", level), b""))
        k += 1
    return b"".join(out) + EOF_MARKER
