"""b200_zstd_decompress, b200_bgzf_decompress and b200_bgzf_compress on the hand-built streams of tests/_codec_craft.py:
every valid stream decodes byte for byte (also into a slot of exactly its size), every malformed one gets its
documented status without touching its neighbours, one byte too little room gives OVERFLOW, nothing is written outside
a stream's slot, and the compressor's length-limited codes are complete and no longer than DEFLATE allows."""
import zlib

import numpy as np
import pytest
import torch

from bonito_b200 import native

import _bgzf_corpus as C
import _codec_craft as K

pytestmark = pytest.mark.gpu
CANARY = 0x5A
GAP = 64   # canary bytes between output slots


def _launch_zstd(streams, caps, extra_rows=()):
    """One b200_zstd_decompress launch: (output slots, out_len, status, whether every byte outside the slots kept the
    canary).  extra_rows are meta rows appended as they are (for the BOUNDS status)."""
    rows, blob, at, oat = [], b"", 0, GAP
    for s, cap in zip(streams, caps):
        rows.append([at, len(s), oat, cap])
        blob += s
        at, oat = at + len(s), oat + cap + GAP
    rows += [list(r) for r in extra_rows]
    inp = torch.from_numpy(np.frombuffer(blob + b"\0", np.uint8).copy()).cuda()[:len(blob)]
    out = torch.full((oat,), CANARY, dtype=torch.uint8, device="cuda")
    out_len = torch.full((len(rows),), -1, dtype=torch.int64, device="cuda")
    status = torch.full((len(rows),), -1, dtype=torch.int32, device="cuda")
    native.zstd_decompress(inp, torch.tensor(rows, dtype=torch.int64, device="cuda"), out, out_len, status)
    torch.cuda.synchronize()
    host = out.cpu().numpy()
    outside = np.ones(oat, bool)
    for r in rows[:len(streams)]:
        outside[r[2]:r[2] + r[3]] = False
    lens = out_len.cpu().tolist()
    slots = [host[r[2]:r[2] + max(n, 0)].tobytes() for r, n in zip(rows, lens)]
    return slots, lens, status.cpu().tolist(), bool((host[outside] == CANARY).all())


def test_zstd_crafted_streams_in_one_launch():
    valid, bad = K.zstd_valid(), K.zstd_malformed()
    streams, caps, want = [], [], []
    for i, (name, s, exp, _) in enumerate(valid):   # malformed streams between valid ones
        streams.append(s)
        caps.append(len(exp) + 37)
        want.append((name, K.Z_OK, exp))
        if i < len(bad):
            streams.append(bad[i][1])
            caps.append(bad[i][2])
            want.append((bad[i][0], bad[i][3], None))
    for name, s, cap, st, _ in bad[len(valid):]:
        streams.append(s)
        caps.append(cap)
        want.append((name, st, None))
    slots, lens, status, kept = _launch_zstd(streams, caps, extra_rows=[(0, 10 ** 12, 0, 8)])
    assert status[-1] == K.Z_BOUNDS
    for (name, st, exp), got, n, s in zip(want, slots, lens, status):
        assert s == st, (name, native.ZSTD_STATUS.get(s), native.ZSTD_STATUS.get(st))
        if exp is not None:
            assert n == len(exp) and got == exp, name
    assert kept, "a stream wrote outside its slot"


def test_zstd_exact_capacity_and_one_byte_less():
    valid = K.zstd_valid()
    streams, caps, want = [], [], []
    for name, s, exp, _ in valid:
        streams.append(s)
        caps.append(len(exp))
        want.append((name, K.Z_OK, exp))
        if exp:
            streams.append(s)
            caps.append(len(exp) - 1)
            want.append((name + " (one byte short)", K.Z_OVERFLOW, None))
    slots, lens, status, kept = _launch_zstd(streams, caps)
    for (name, st, exp), got, n, s in zip(want, slots, lens, status):
        assert s == st, (name, native.ZSTD_STATUS.get(s))
        if exp is not None:
            assert got == exp, name
    assert kept, "a stream wrote outside its slot"


def _launch_inflate(members, extra_rows=()):
    """One b200_bgzf_decompress launch over [(BGZF member, ISIZE, CRC32)]: (outputs, status, canary kept)."""
    rows, blob, oat = [], b"", GAP
    for m, isize, crc in members:
        raw_at = len(blob) + 18          # _bgzf_corpus.member: the raw data after the 18-byte header
        rows.append([raw_at, len(m) - 26, oat, isize, crc])
        blob += m
        oat += isize + GAP
    rows += [list(r) for r in extra_rows]
    inp = torch.from_numpy(np.frombuffer(blob + b"\0", np.uint8).copy()).cuda()[:len(blob)]
    out = torch.full((oat,), CANARY, dtype=torch.uint8, device="cuda")
    status = torch.full((len(rows),), -1, dtype=torch.int32, device="cuda")
    native.bgzf_decompress(inp, torch.tensor(rows, dtype=torch.int64, device="cuda"), out, status)
    torch.cuda.synchronize()
    host = out.cpu().numpy()
    outside = np.ones(oat, bool)
    for r in rows[:len(members)]:
        outside[r[2]:r[2] + r[3]] = False
    return ([host[r[2]:r[2] + r[3]].tobytes() for r in rows[:len(members)]], status.cpu().tolist(),
            bool((host[outside] == CANARY).all()))


def test_inflate_crafted_members_in_one_launch():
    valid, bad = K.inflate_valid(), K.inflate_malformed()
    members, want = [], []
    for i in range(max(len(valid), len(bad))):
        if i < len(valid):
            name, raw, exp, _ = valid[i]
            members.append((C.member(raw, exp), len(exp), zlib.crc32(exp)))
            want.append((name, K.I_OK, exp))
        if i < len(bad):
            name, raw, isize, crc, st = bad[i]
            members.append((C.member(raw, b"", isize, crc), isize, crc))
            want.append((name, st, None))
    outs, status, kept = _launch_inflate(members, extra_rows=[(0, 10, 0, 65537, 0)])
    assert status[-1] == K.I_BOUNDS
    for (name, st, exp), got, s in zip(want, outs, status):
        assert s == st, (name, s, st)
        if exp is not None:
            assert got == exp, name
    assert kept, "a member wrote outside its slot"


def test_inflate_one_byte_less_room():
    members, want = [], []
    for name, raw, exp, _ in K.inflate_valid():
        if exp:
            members.append((C.member(raw, exp, len(exp) - 1), len(exp) - 1, zlib.crc32(exp)))
            want.append(name)
    outs, status, kept = _launch_inflate(members)
    assert status == [K.I_OVERFLOW] * len(want), list(zip(want, status))
    assert kept, "a member wrote outside its slot"


def _compress(data):
    from test_gpu_bgzf import compress
    return compress(data)


def _kraft(lens):
    return sum(2.0 ** -l for l in lens if l)


def test_compressor_limits_code_lengths():
    """The optimal literal/length code of these payloads is deeper than 15 bits, so the limiter in bgzf.cu has to cut
    it: the written code reaches exactly 15 bits, no further, and stays complete.  The code-length code is checked the
    same way (complete, at most 7 bits); these payloads do not make its optimal code deeper than 7 (that takes
    code-length frequencies of Fibonacci shape over nine or more lengths, which a byte histogram only loosely steers),
    so its limit is checked but not exercised."""
    payloads = [K.deep_code_payload(seed=s) for s in range(3)]
    for data in payloads:
        packed, off = _compress(data)
        assert len(off) == 2
        assert zlib.decompress(packed, 31) == data     # gzip framing: zlib checks CRC32 and ISIZE too
        raw = packed[18:-8]
        b = K.read_dynamic_block(raw)
        freq = {s: c for s, c in enumerate(b["lit_counts"]) if c}
        assert max(K.huffman_depths(freq).values()) > 15, "the payload does not need the limiter"
        assert max(b["lit_lens"]) == 15 and _kraft(b["lit_lens"]) == 1.0
        assert all(b["lit_lens"][s] for s in freq)
        assert max(b["dist_lens"]) <= 15 and _kraft(b["dist_lens"]) == 1.0
        assert max(b["cl_lens"]) <= 7 and _kraft(b["cl_lens"]) == 1.0
        again, _ = _compress(data)
        assert again == packed


def test_compressor_stores_an_incompressible_member():
    data = np.random.default_rng(4).integers(0, 256, 65280, dtype=np.uint8).tobytes()
    packed, off = _compress(data)
    assert list(off) == [0, 65311] and len(packed) == 65311
    assert packed[18] == 1 and packed[19:23] == bytes([0x00, 0xff, 0xff, 0x00])   # final stored block, LEN 65280
    assert zlib.decompress(packed, 31) == data
    assert _compress(data)[0] == packed
