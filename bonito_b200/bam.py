"""
BAM output: the binary encoding of the SAM header and records that bonito_b200.io builds as text, following htslib's
`sam_parse1` (what the reference's `AlignedSegment.fromstring` runs, bonito/io.py:400-503), and a BGZF writer whose
DEFLATE compression runs on the GPU (b200_bgzf_compress).

BAM input (`duplex reads.bam`, what the reference reads through pysam in bonito/cli/duplex.py:45-105): a BGZF reader
whose inflation runs on the GPU (b200_bgzf_decompress) and accepts any valid BGZF file (htslib's, libdeflate's, this
module's), a record parser that checks every field, and `read_records`, which returns what the SAM reader of
`duplex` returns for the same records.

`sam_record` and `read_tags` in bonito_b200.io decide what a record holds; this module only encodes SAM lines.
"""

import re
import struct

import numpy as np
import torch

from bonito_b200 import native

MAGIC = b"BAM\1"
# the empty BGZF member that ends every BGZF file (SAM specification section 4.1.2)
EOF_MARKER = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")
MAX_CIGAR_OPS = 0xffff
MAX_READ_NAME = 254

_CIGAR = re.compile(r"(\d+)([MIDNSHP=X])")
_CIGAR_OPS = {op: i for i, op in enumerate("MIDNSHP=X")}
_REF_OPS = {0, 2, 3, 7, 8}            # M D N = X consume the reference
_NT16 = np.full(256, 15, dtype=np.uint8)
for _i, _c in enumerate("=ACMGRSVTWYHKDBN"):
    _NT16[ord(_c)] = _NT16[ord(_c.lower())] = _i
_B_TYPES = {"c": "b", "C": "B", "s": "h", "S": "H", "i": "i", "I": "I", "f": "f"}
_SEQ_CHARS = np.frombuffer(b"=ACMGRSVTWYHKDBN", dtype=np.uint8)
_AUX_SIZES = {ord(t): n for t, n in zip("AcCsSiIf", (1, 1, 1, 2, 2, 4, 4, 4))}
_B_DTYPES = {"c": np.int8, "C": np.uint8, "s": np.int16, "S": np.uint16, "i": np.int32, "I": np.uint32, "f": np.float32}


def reg2bin(beg, end, min_shift=14, n_lvls=5):
    """htslib's hts_reg2bin: the smallest bin that holds [beg, end)."""
    end -= 1
    s, t = min_shift, ((1 << ((n_lvls << 1) + n_lvls)) - 1) // 7
    for level in range(n_lvls - 1, -1, -1):
        if beg >> s == end >> s:
            return t + (beg >> s)
        s += 3
        t -= 1 << ((level << 1) + level)
    return 0


def encode_header(text, contigs=()):
    """BAM header: magic, the SAM header text, then each contig's name and length."""
    text = text.encode()
    out = [MAGIC, struct.pack("<i", len(text)), text, struct.pack("<i", len(contigs))]
    for name, length in contigs:
        name = name.encode() + b"\0"
        out += [struct.pack("<i", len(name)), name, struct.pack("<i", int(length))]
    return b"".join(out)


def _int_tag(tag, value):
    v = int(value)
    if v < 0:
        t = "c" if v >= -0x80 else "s" if v >= -0x8000 else "i"
    else:
        t = "C" if v <= 0xff else "S" if v <= 0xffff else "I"
    return tag + t.encode() + struct.pack("<" + _B_TYPES[t], v)


def _array_values(sub, text):
    """The values of a B-array; single-digit integer lists (the move table) skip the per-value parse."""
    if not text:
        return np.zeros(0, dtype=_B_DTYPES[sub])
    if sub != "f":
        raw = np.frombuffer(text.encode(), dtype=np.uint8)
        if raw.size % 2 and np.all(raw[1::2] == ord(",")) and np.all((raw[::2] >= ord("0")) & (raw[::2] <= ord("9"))):
            return (raw[::2] - ord("0")).astype(_B_DTYPES[sub])
        return np.array([int(v) for v in text.split(",")], dtype=np.int64).astype(_B_DTYPES[sub])
    return np.array([float(v) for v in text.split(",")], dtype=np.float32)


def encode_tag(field):
    """One SAM optional field `TG:T:value` as BAM aux bytes (sam_parse1's type choices)."""
    tag, typ, value = field[:2].encode(), field[3], field[5:]
    if typ == "i":
        return _int_tag(tag, value)
    if typ == "Z" or typ == "H":
        return tag + typ.encode() + value.encode() + b"\0"
    if typ == "A":
        return tag + b"A" + value.encode()
    if typ == "f":
        return tag + b"f" + struct.pack("<f", float(value))
    if typ == "B":
        sub, _, rest = value.partition(",")
        if sub not in _B_DTYPES:
            raise ValueError(f"unknown B-array subtype in SAM field {field[:32]!r}")
        if sub != "f" and rest:
            head, _, tail = rest.partition(",")      # a move table starts with the stride, which may have two digits
            vals = np.concatenate([np.array([int(head)]), _array_values(sub, tail)]).astype(_B_DTYPES[sub])
        else:
            vals = _array_values(sub, rest)
        return tag + b"B" + sub.encode() + struct.pack("<i", vals.size) + vals.astype(vals.dtype.newbyteorder("<")).tobytes()
    raise ValueError(f"unknown type {typ!r} in SAM field {field[:32]!r}")


def encode_record(line, ref_ids=None):
    """One SAM text line (no newline) as a BAM record, block_size included.  ref_ids: {contig name: index}."""
    f = line.split("\t")
    qname, flag, rname, pos, mapq, cigar, rnext, pnext, tlen, seq, qual = f[:11]
    name = qname.encode()
    if len(name) > MAX_READ_NAME:
        raise ValueError(f"read name of {len(name)} bytes: BAM allows at most {MAX_READ_NAME} ({qname[:40]}...)")
    ref_ids = ref_ids or {}
    ref_id = -1 if rname == "*" else ref_ids[rname]
    pos = int(pos) - 1
    next_ref = -1 if rnext == "*" else ref_id if rnext == "=" else ref_ids[rnext]
    ops = np.zeros(0, dtype=np.uint32)
    ref_len = 0
    if cigar != "*":
        parsed = _CIGAR.findall(cigar)
        lens = np.array([int(n) for n, _ in parsed], dtype=np.uint32)
        codes = np.array([_CIGAR_OPS[op] for _, op in parsed], dtype=np.uint32)
        ops = lens << 4 | codes
        ref_len = int(lens[np.isin(codes, list(_REF_OPS))].sum())
    l_seq = 0 if seq == "*" else len(seq)
    bin_ = reg2bin(pos, pos + ref_len if ref_len > 0 else pos + 1)
    aux = [encode_tag(t) for t in f[11:]]
    if ops.size > MAX_CIGAR_OPS:          # htslib's convention: a placeholder CIGAR, the real one in CG:B:I
        aux.append(b"CGBI" + struct.pack("<i", ops.size) + ops.astype("<u4").tobytes())
        ops = np.array([l_seq << 4 | 4, ref_len << 4 | 3], dtype=np.uint32)
    if l_seq:
        nt = _NT16[np.frombuffer(seq.encode(), dtype=np.uint8)]
        if l_seq % 2:
            nt = np.append(nt, np.uint8(0))
        packed = (nt[0::2] << 4 | nt[1::2]).astype(np.uint8).tobytes()
        quals = b"\xff" * l_seq if qual == "*" else (np.frombuffer(qual.encode(), dtype=np.uint8) - 33).astype(np.uint8).tobytes()
    else:
        packed = quals = b""
    fixed = struct.pack("<iiBBHHHIiii", ref_id, pos, len(name) + 1, int(mapq), bin_, ops.size, int(flag), l_seq,
                        next_ref, int(pnext) - 1, int(tlen))
    body = b"".join([fixed, name, b"\0", ops.astype("<u4").tobytes(), packed, quals, *aux])
    return struct.pack("<i", len(body)) + body


class BgzfWriter:
    """
    A BGZF stream to the binary file `fd`, compressed on the GPU: the uncompressed bytes gather in a pinned staging buffer,
    and whenever `members_per_launch` full members (of 65280 bytes) are waiting they are compressed by one
    b200_bgzf_compress launch on a stream of the writer's own and written out; the rest carries forward.  close()
    compresses the tail and appends the EOF marker.  Members are cut at fixed offsets of the uncompressed stream, so the
    file does not depend on `members_per_launch`.
    """

    def __init__(self, fd, device="cuda", members_per_launch=256):
        if members_per_launch < 1:
            raise ValueError(f"members_per_launch must be at least 1, got {members_per_launch}")
        native.require()
        self.fd, self.members = fd, int(members_per_launch)
        device = torch.device(device)
        self.device = device if device.index is not None else torch.device("cuda", torch.cuda.current_device())
        m = native.BGZF_MEMBER_INPUT
        self.cap = (self.members + 1) * m
        slots = self.members + 1
        self.stage = torch.empty(self.cap, dtype=torch.uint8, pin_memory=True)
        self.view = self.stage.numpy()
        self.fill = 0
        self.stream = native.new_stream(self.device)
        self.d_in = torch.empty(self.cap, dtype=torch.uint8, device=self.device)
        self.d_out = torch.empty(slots * native.BGZF_MEMBER_MAX, dtype=torch.uint8, device=self.device)
        self.d_off = torch.empty(slots + 1, dtype=torch.int64, device=self.device)
        self.d_ws = torch.empty(native.bgzf_workspace_bytes(self.cap), dtype=torch.uint8, device=self.device)
        self.h_out = torch.empty(slots * native.BGZF_MEMBER_MAX, dtype=torch.uint8, pin_memory=True)
        self.h_off = torch.empty(slots + 1, dtype=torch.int64, pin_memory=True)

    def write(self, data):
        data = memoryview(data).cast("B")
        full = self.members * native.BGZF_MEMBER_INPUT
        while len(data):
            take = min(len(data), self.cap - self.fill)
            self.view[self.fill:self.fill + take] = np.frombuffer(data[:take], dtype=np.uint8)
            self.fill += take
            data = data[take:]
            if self.fill >= full:
                self._compress(self.fill - self.fill % native.BGZF_MEMBER_INPUT)

    def _compress(self, nbytes):
        """Compress the first `nbytes` staged bytes, write the members, keep the rest staged."""
        n = native.bgzf_members(nbytes)
        with torch.cuda.device(self.device), torch.cuda.stream(self.stream):
            self.d_in[:nbytes].copy_(self.stage[:nbytes], non_blocking=True)
            native.bgzf_compress(self.d_in[:nbytes], self.d_out, self.d_off, self.d_ws, stream=self.stream)
            self.h_off[:n + 1].copy_(self.d_off[:n + 1], non_blocking=True)
            self.stream.synchronize()
            total = int(self.h_off[n])
            self.h_out[:total].copy_(self.d_out[:total], non_blocking=True)
            self.stream.synchronize()
        self.fd.write(memoryview(self.h_out.numpy())[:total])
        rest = self.fill - nbytes
        self.view[:rest] = self.view[nbytes:self.fill]
        self.fill = rest

    def close(self):
        if self.fill:
            self._compress(self.fill)
        self.fd.write(EOF_MARKER)
        self.fd.flush()


class BamOutput:
    """A BAM file on `fd`: the header from the SAM header text and contigs, then one record per SAM line."""

    def __init__(self, fd, header_text, contigs=None, device="cuda", members_per_launch=256):
        contigs = list(contigs or ())
        self.ref_ids = {name: i for i, (name, _) in enumerate(contigs)}
        self.bgzf = BgzfWriter(fd, device=device, members_per_launch=members_per_launch)
        self.bgzf.write(encode_header(header_text, contigs))

    def write_sam(self, line):
        self.bgzf.write(encode_record(line, self.ref_ids))

    def close(self):
        self.bgzf.close()


# ------------------------------------------------------------------------------------------------ BAM input
def check_bgzf_file(path):
    """Cheap host check that `path` can be a BGZF file: a gzip magic and the 28-byte EOF marker at the end."""
    with open(path, "rb") as fh:
        head = fh.read(4)
        fh.seek(0, 2)
        size = fh.tell()
        tail = b""
        if size >= len(EOF_MARKER):
            fh.seek(size - len(EOF_MARKER))
            tail = fh.read()
    if head[:3] != b"\x1f\x8b\x08" or tail != EOF_MARKER:
        raise ValueError(f"{path} is not a BAM file: empty, or missing the BGZF EOF marker that htslib writes")


def next_member(fh, where):
    """(member bytes, raw DEFLATE start and length in them, CRC32, ISIZE) of the BGZF member at the file position
    `where` of the binary file `fh`, or None at the end of the file."""
    def bad(what):
        return ValueError(f"BGZF member at byte {where}: {what}")

    head = fh.read(12)
    if not head:
        return None
    if len(head) < 12:
        raise bad("truncated header")
    if head[:3] != b"\x1f\x8b\x08" or head[3] != 4:
        raise bad(f"not a BGZF member header (magic, method, flags {head[:4].hex()})")
    xlen = head[10] | head[11] << 8
    extra = fh.read(xlen)
    if len(extra) < xlen:
        raise bad("truncated extra field")
    bsize, p = None, 0
    while p < xlen:                                  # subfields: SI1 SI2 SLEN data
        slen = extra[p + 2] | extra[p + 3] << 8 if xlen - p >= 4 else None
        if slen is None or xlen - p - 4 < slen:
            raise bad("malformed extra subfield")
        if extra[p:p + 2] == b"BC" and slen == 2:
            bsize = (extra[p + 4] | extra[p + 5] << 8) + 1
        p += 4 + slen
    if bsize is None:
        raise bad("no BC subfield")
    if bsize < 12 + xlen + 8:
        raise bad(f"BSIZE {bsize - 1} is smaller than its header and trailer")
    rest = fh.read(bsize - 12 - xlen)
    if len(rest) < bsize - 12 - xlen:
        raise bad("truncated member")
    crc, isize = struct.unpack_from("<II", rest, len(rest) - 8)
    if isize > native.BGZF_MEMBER_MAX:
        raise bad(f"ISIZE {isize} exceeds {native.BGZF_MEMBER_MAX}")
    return head + extra + rest, 12 + xlen, bsize - 20 - xlen, crc, isize


class BgzfReader:
    """
    The uncompressed bytes of the BGZF file `path`, inflated on the GPU: iterating yields one bytes object per window of
    up to `members_per_launch` members.  For each window the host walks the member headers, then one host-to-device copy,
    one b200_bgzf_decompress launch on a stream of the reader's own and one device-to-host copy bring the bytes back.
    Memory stays bounded by the window whatever the file's size, and the bytes do not depend on `members_per_launch`.
    A malformed member is a ValueError naming its byte offset in the file; so is a file without the EOF marker.
    """

    def __init__(self, path, device="cuda", members_per_launch=1024):
        if members_per_launch < 1:
            raise ValueError(f"members_per_launch must be at least 1, got {members_per_launch}")
        native.require()
        self.path, self.members = path, int(members_per_launch)
        device = torch.device(device)
        self.device = device if device.index is not None else torch.device("cuda", torch.cuda.current_device())
        self.meta_bytes = self.members * 5 * 8
        cap_in = self.meta_bytes + self.members * native.BGZF_MEMBER_MAX
        cap_out = self.members * (native.BGZF_MEMBER_MAX + 4)
        self.h_in = torch.empty(cap_in, dtype=torch.uint8, pin_memory=True)
        self.h_out = torch.empty(cap_out, dtype=torch.uint8, pin_memory=True)
        self.d_in = torch.empty(cap_in, dtype=torch.uint8, device=self.device)
        self.d_out = torch.empty(cap_out, dtype=torch.uint8, device=self.device)
        self.stream = native.new_stream(self.device)

    def _windows(self):
        """Lists of up to `members` (file offset, raw start, raw length, CRC32, ISIZE) rows, the raw start an offset into
        the window's raw bytes, which come with them; the EOF marker is checked at the end."""
        with open(self.path, "rb") as fh:
            where, last = 0, None
            while True:
                window, raws, at = [], [], 0
                while len(window) < self.members:
                    m = next_member(fh, where)
                    if m is None:
                        break
                    member, raw, n_raw, crc, isize = m
                    window.append((where, at, n_raw, crc, isize))
                    raws.append(member[raw:raw + n_raw])
                    at += n_raw
                    where += len(member)
                    last = member
                if not window:
                    break
                yield window, b"".join(raws)
        if last != EOF_MARKER:
            raise ValueError(f"{self.path} does not end with the BGZF EOF marker (truncated file?)")

    def __iter__(self):
        h_meta = self.h_in[:self.meta_bytes].view(torch.int64).view(self.members, 5)
        for window, raw in self._windows():
            n = len(window)
            meta = h_meta[:n].numpy()
            w = np.array(window, dtype=np.int64)
            meta[:, 0], meta[:, 1], meta[:, 3], meta[:, 4] = w[:, 1], w[:, 2], w[:, 4], w[:, 3]
            meta[:, 2] = np.concatenate([[0], np.cumsum(w[:n - 1, 4])])
            total = int(w[:, 4].sum())
            nbytes = len(raw)
            self.h_in.numpy()[self.meta_bytes:self.meta_bytes + nbytes] = np.frombuffer(raw, dtype=np.uint8)
            status_at = -(-total // 4) * 4
            with torch.cuda.device(self.device), torch.cuda.stream(self.stream):
                used = self.meta_bytes + nbytes
                self.d_in[:used].copy_(self.h_in[:used], non_blocking=True)
                d_meta = self.d_in[:self.meta_bytes].view(torch.int64).view(self.members, 5)[:n]
                status = self.d_out[status_at:status_at + 4 * n].view(torch.int32)
                native.bgzf_decompress(self.d_in[self.meta_bytes:used], d_meta, self.d_out[:total], status,
                                       stream=self.stream)
                got = status_at + 4 * n
                self.h_out[:got].copy_(self.d_out[:got], non_blocking=True)
                self.stream.synchronize()
            st = self.h_out[status_at:got].view(torch.int32).numpy()
            bad = np.flatnonzero(st)
            if bad.size:
                i = int(bad[0])
                why = native.INFLATE_STATUS.get(int(st[i]), f"status {int(st[i])}")
                raise ValueError(f"{self.path}: BGZF member at byte {window[i][0]}: {why}")
            yield self.h_out[:total].numpy().tobytes()


class BamRecordParser:
    """
    BAM records from the uncompressed stream, fed in chunks cut anywhere (a partial record carries over to the next
    chunk).  Checks the magic, `l_text` and `n_ref` and skips the header; then for each record `block_size` >= 32 and
    every field inside the block.  feed() returns the complete records so far as (read name, flag, body, offset of SEQ
    in body, l_seq), body being the record without its block_size; a malformed record is a ValueError with its index.
    """

    def __init__(self):
        self.buf, self.pos, self.in_header, self.count = b"", 0, True, 0

    def _header(self):
        b, p = self.buf, self.pos
        if len(b) - p < 12:
            return False
        if b[p:p + 4] != MAGIC:
            raise ValueError(f"not a BAM stream: magic {bytes(b[p:p + 4])!r}")
        l_text = struct.unpack_from("<i", b, p + 4)[0]
        if l_text < 0:
            raise ValueError(f"BAM header: l_text {l_text}")
        q = p + 8 + l_text
        if len(b) - q < 4:
            return False
        n_ref = struct.unpack_from("<i", b, q)[0]
        if n_ref < 0:
            raise ValueError(f"BAM header: n_ref {n_ref}")
        q += 4
        for i in range(n_ref):
            if len(b) - q < 4:
                return False
            l_name = struct.unpack_from("<i", b, q)[0]
            if l_name < 1:
                raise ValueError(f"BAM header: reference {i} has l_name {l_name}")
            q += 4 + l_name + 4
            if q > len(b):
                return False
        self.pos, self.in_header = q, False
        return True

    def _record(self, body):
        """(name, flag, seq offset, l_seq) of one record body, every field checked."""
        n = len(body)
        _, _, l_name, _, _, n_cigar, flag, l_seq, _, _, _ = struct.unpack_from("<iiBBHHHIiii", body, 0)
        def bad(what):
            return ValueError(f"BAM record {self.count}: {what}")
        if l_name < 1 or 32 + l_name > n or body[32 + l_name - 1] != 0:
            raise bad(f"read name of l_read_name {l_name} is not NUL-terminated inside the block")
        seq_at = 32 + l_name + 4 * n_cigar
        aux = seq_at + (l_seq + 1) // 2 + l_seq
        if l_seq >= 1 << 31 or aux > n:
            raise bad(f"CIGAR ({n_cigar} ops), SEQ and QUAL ({l_seq} bases) overrun block_size {n + 4}")
        p = aux
        while p < n:                                  # aux fields: tag, type, value
            if n - p < 3:
                raise bad("truncated aux field")
            t = body[p + 2]
            p += 3
            if t in _AUX_SIZES:
                p += _AUX_SIZES[t]
            elif t in (0x5a, 0x48):                   # Z, H: NUL-terminated
                end = body.find(b"\0", p)
                if end < 0:
                    raise bad("unterminated Z/H aux field")
                p = end + 1
            elif t == 0x42:                           # B: subtype, count, values
                if n - p < 5 or body[p] not in _AUX_SIZES or body[p] == 0x41:
                    raise bad("malformed B aux field")
                p += 5 + _AUX_SIZES[body[p]] * struct.unpack_from("<I", body, p + 1)[0]
            else:
                raise bad(f"aux field of unknown type {chr(t)!r}")
            if p > n:
                raise bad("aux field overruns the block")
        return body[32:32 + l_name - 1].decode(errors="replace"), flag, seq_at, l_seq

    def feed(self, data):
        self.buf = self.buf[self.pos:] + bytes(data)
        self.pos = 0
        if self.in_header and not self._header():
            return []
        out, b, p = [], self.buf, self.pos
        while len(b) - p >= 4:
            size = struct.unpack_from("<i", b, p)[0]
            if size < 32:
                raise ValueError(f"BAM record {self.count}: block_size {size} < 32")
            if len(b) - p - 4 < size:
                break
            body = b[p + 4:p + 4 + size]
            name, flag, seq_at, l_seq = self._record(body)
            out.append((name, flag, body, seq_at, l_seq))
            self.count += 1
            p += 4 + size
        self.pos = p
        return out

    def close(self):
        if self.in_header:
            raise ValueError("BAM stream ends inside its header")
        if self.pos != len(self.buf):
            raise ValueError(f"BAM record {self.count}: truncated ({len(self.buf) - self.pos} bytes left)")


def record_seq_qual(body, seq_at, l_seq):
    """(SEQ as stored, Q values as uint8 or None for a QUAL of 0xFF bytes); l_seq == 0 gives ("*", None)."""
    if l_seq == 0:
        return "*", None
    packed = np.frombuffer(body, dtype=np.uint8, count=(l_seq + 1) // 2, offset=seq_at)
    codes = np.empty(2 * packed.size, dtype=np.uint8)
    codes[0::2], codes[1::2] = packed >> 4, packed & 15
    seq = _SEQ_CHARS[codes[:l_seq]].tobytes().decode()
    qual = np.frombuffer(body, dtype=np.uint8, count=l_seq, offset=seq_at + (l_seq + 1) // 2)
    return seq, (None if qual[0] == 0xff else qual.copy())


def records_from_chunks(chunks, wanted=None):
    """{read id: (SEQ, Q values or None)} of the first record of each id that is neither secondary (0x100) nor
    supplementary (0x800), restricted to `wanted` ids when given, from uncompressed BAM stream chunks."""
    parser, reads = BamRecordParser(), {}
    for chunk in chunks:
        for name, flag, body, seq_at, l_seq in parser.feed(chunk):
            if flag & 0x900 or name in reads or (wanted is not None and name not in wanted):
                continue
            reads[name] = record_seq_qual(body, seq_at, l_seq)
    parser.close()
    return reads


def read_records(path, wanted=None, device="cuda", members_per_launch=1024):
    """What `duplex` reads from a BAM file, inflated on the GPU: see records_from_chunks."""
    return records_from_chunks(BgzfReader(path, device=device, members_per_launch=members_per_launch), wanted)
