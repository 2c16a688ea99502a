"""
BAM output: the binary encoding of the SAM header and records that bonito_b200.io builds as text, following htslib's
`sam_parse1` (what the reference's `AlignedSegment.fromstring` runs, bonito/io.py:400-503), and a BGZF writer whose
DEFLATE compression runs on the GPU (b200_bgzf_compress).

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
