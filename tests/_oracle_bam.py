"""
Independent BAM reader for the tests, from gzip / zlib / struct only: checks every BGZF member (header fields, BSIZE,
CRC32, ISIZE) and the EOF marker, and turns the records back into SAM text lines the way `samtools view` prints them
(a `<l_seq>S<ref_len>N` placeholder CIGAR with a CG:B:I tag becomes the real CIGAR again), floats excepted: those are
printed with every digit float32 needs.
"""
import struct
import zlib

EOF_MARKER = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


def bgzf_members(data):
    """[(raw DEFLATE bytes, uncompressed bytes)] of every member; the last member must be the EOF marker."""
    members, off = [], 0
    while off < len(data):
        head = data[off:off + 18]
        assert head[:4] == b"\x1f\x8b\x08\x04", f"member at {off}: bad gzip magic / method / flags {head[:4].hex()}"
        mtime, xfl, os_, xlen = struct.unpack("<IBBH", head[4:12])
        assert (mtime, xfl, os_, xlen) == (0, 0, 0xff, 6), (off, mtime, xfl, os_, xlen)
        assert head[12:16] == b"BC\x02\x00", f"member at {off}: no BC subfield"
        bsize = struct.unpack("<H", head[16:18])[0] + 1
        cdata = data[off + 18:off + bsize - 8]
        crc, isize = struct.unpack("<II", data[off + bsize - 8:off + bsize])
        raw = zlib.decompress(cdata, wbits=-15)
        assert len(raw) == isize and zlib.crc32(raw) == crc, f"member at {off}: ISIZE / CRC32 mismatch"
        members.append((cdata, raw))
        off += bsize
    assert off == len(data)
    return members


def bgzf_decompress(data):
    """The uncompressed stream of a BGZF file that ends with the EOF marker."""
    assert data.endswith(EOF_MARKER), "no BGZF EOF marker"
    members = bgzf_members(data[:-len(EOF_MARKER)])
    return b"".join(raw for _, raw in members)


def _fmt_float(v):
    """The shortest text that reads back as the same float32 (samtools prints %g, which can lose digits)."""
    import numpy as np
    return str(np.float32(v))


_INT = {"c": "b", "C": "B", "s": "h", "S": "H", "i": "i", "I": "I"}


def _aux(buf, off):
    tags = []
    while off < len(buf):
        tag, typ = buf[off:off + 2].decode(), chr(buf[off + 2])
        off += 3
        if typ == "A":
            tags.append((tag, f"{tag}:A:{chr(buf[off])}"))
            off += 1
        elif typ in _INT:
            size = struct.calcsize(_INT[typ])
            tags.append((tag, f"{tag}:i:{struct.unpack_from('<' + _INT[typ], buf, off)[0]}"))
            off += size
        elif typ == "f":
            tags.append((tag, f"{tag}:f:{_fmt_float(struct.unpack_from('<f', buf, off)[0])}"))
            off += 4
        elif typ in "ZH":
            end = buf.index(b"\0", off)
            tags.append((tag, f"{tag}:{typ}:{buf[off:end].decode()}"))
            off = end + 1
        elif typ == "B":
            sub = chr(buf[off])
            count = struct.unpack_from("<i", buf, off + 1)[0]
            code = "f" if sub == "f" else _INT[sub]
            vals = struct.unpack_from(f"<{count}{code}", buf, off + 5)
            off += 5 + count * struct.calcsize(code)
            text = ",".join(_fmt_float(v) if sub == "f" else str(v) for v in vals)
            tags.append((tag, f"{tag}:B:{sub}" + ("," + text if count else ""), vals))
        else:
            raise AssertionError(f"unknown aux type {typ!r}")
    return tags


def decode_record(buf, refs):
    """One record (without block_size) -> (SAM line, fields dict)."""
    ref_id, pos, l_name, mapq, bin_, n_cigar, flag, l_seq, next_ref, next_pos, tlen = struct.unpack_from("<iiBBHHHIiii", buf)
    off = 32
    name = buf[off:off + l_name - 1].decode()
    assert buf[off + l_name - 1] == 0
    off += l_name
    cigar = list(struct.unpack_from(f"<{n_cigar}I", buf, off))
    off += 4 * n_cigar
    packed = buf[off:off + (l_seq + 1) // 2]
    off += (l_seq + 1) // 2
    seq = "".join("=ACMGRSVTWYHKDBN"[(packed[i // 2] >> (4 * (1 - i % 2))) & 15] for i in range(l_seq))
    qual = buf[off:off + l_seq]
    off += l_seq
    tags = _aux(buf, off)
    cg = [t for t in tags if t[0] == "CG"]
    if len(cigar) == 2 and cigar[0] == (l_seq << 4 | 4) and cigar[1] & 15 == 3 and cg:
        cigar = list(cg[0][2])
        tags = [t for t in tags if t[0] != "CG"]
    cigar_str = "".join(f"{c >> 4}{'MIDNSHP=X'[c & 15]}" for c in cigar) or "*"
    rname = "*" if ref_id < 0 else refs[ref_id][0]
    rnext = "*" if next_ref < 0 else "=" if next_ref == ref_id else refs[next_ref][0]
    qual_str = "*" if not l_seq or qual[0] == 0xff else "".join(chr(q + 33) for q in qual)
    fields = [name, str(flag), rname, str(pos + 1), str(mapq), cigar_str, rnext, str(next_pos + 1), str(tlen),
              seq or "*", qual_str] + [t[1] for t in tags]
    return "\t".join(fields), {"bin": bin_, "n_cigar": n_cigar, "raw_cigar": cigar, "tags": tags}


def decode_bam(raw):
    """(header text, [(name, length)], [SAM lines], [fields dicts]) of an uncompressed BAM stream."""
    assert raw[:4] == b"BAM\1"
    l_text = struct.unpack_from("<i", raw, 4)[0]
    text = raw[8:8 + l_text].decode()
    off = 8 + l_text
    n_ref = struct.unpack_from("<i", raw, off)[0]
    off += 4
    refs = []
    for _ in range(n_ref):
        l_name = struct.unpack_from("<i", raw, off)[0]
        name = raw[off + 4:off + 4 + l_name - 1].decode()
        assert raw[off + 4 + l_name - 1] == 0
        refs.append((name, struct.unpack_from("<i", raw, off + 4 + l_name)[0]))
        off += 8 + l_name
    lines, info = [], []
    while off < len(raw):
        size = struct.unpack_from("<i", raw, off)[0]
        line, fields = decode_record(raw[off + 4:off + 4 + size], refs)
        lines.append(line)
        info.append(fields)
        off += 4 + size
    assert off == len(raw)
    return text, refs, lines, info


def same_sam_line(bam_line, sam_line):
    """Equal SAM lines, with `f` tags compared as float32."""
    import numpy as np
    a, b = bam_line.split("\t"), sam_line.split("\t")
    if len(a) != len(b):
        return False
    for x, y in zip(a, b):
        if x == y:
            continue
        if len(x) > 5 and x[:5] == y[:5] and x[3:5] == "f:":
            if np.float32(float(x[5:])) != np.float32(float(y[5:])):
                return False
            continue
        return False
    return True
