"""The hand-built zstd and DEFLATE streams of tests/_codec_craft.py are what they claim: libzstd and zlib decode every
valid one to its expected bytes and reject every malformed one (but where the project's decoders are documented to be
stricter), the numpy XXH64 matches libzstd's checksums, and together the lists reach every branch they are there for."""
import struct
import zlib

import numpy as np
import pytest

import _bgzf_corpus as C
import _codec_craft as K
import _pod5_writer as W

needs_libzstd = pytest.mark.skipif(not W.have_libzstd(), reason="needs the system libzstd.so.1")

# the format branches the lists must reach; a change that drops a case fails test_every_branch_has_a_stream
ZSTD_BRANCHES = (
    {("seq", "nseq1"), ("seq", "nseq2"), ("seq", "nseq3"), ("seq", "bits_gt64")}
    | {("ll_code", c) for c in range(25, 36)} | {("ml_code", c) for c in range(43, 53)}
    | {("fse_log", "ll", 9), ("fse_log", "ml", 9), ("fse_log", "of", 8)}
    | {("fse_log", k, lg) for k in ("ll", "ml", "of") for lg in range(5, 9)}
    | {("fse", "below_one"), ("fse", "zero_run_gt3")}
    | {("table_mode", k, m) for k in ("ll", "of", "ml") for m in ("predef", "rle", "fse", "repeat")}
    | {("rle_table_with_extra_bits", "ll"), ("rle_table_with_extra_bits", "ml")}
    | {("repeat", ofv, ll0) for ofv in (1, 2, 3) for ll0 in (False, True)}
    | {("huf_weights", "direct"), ("huf_weights", "fse"), ("huf_weight_count", 255), ("huf_max_bits", 11)}
    | {("lit", "huffman", "1stream", "sf10"), ("lit", "huffman", "4stream", "sf10"),
       ("lit", "huffman", "4stream", "sf14"), ("lit", "huffman", "4stream", "sf18"), ("lit", "4stream_empty_last"),
       ("lit", "treeless")}
    | {("lit", kind, hl) for kind in ("raw", "rle") for hl in (1, 2, 3)}
    | {("fcs", n) for n in (1, 2, 4, 8)} | {("window", "descriptor"), ("window", "single_segment"), "checksum"}
    | {("block", t) for t in ("raw", "rle", "compressed", "compressed_128k")}
    | {("offset", "window"), ("exact_slot", "staged_literals"), ("skippable",)}
)
INFLATE_BRANCHES = (
    {("inflate_lit_len", n) for n in range(1, 16)} | {("inflate_dist_len", n) for n in range(1, 16)}
    | {("inflate_repeat_across", s) for s in (16, 17, 18)}
    | {("inflate", k) for k in ("single_distance_code", "no_distance_codes", "distance_32768", "stored_empty",
                                "stored_after_midbyte", "fixed", "dynamic")}
    | {("inflate_len_sym", 285), ("inflate_dist_sym", 29)}
    | {("hlit", 257), ("hlit", 286), ("hdist", 1), ("hdist", 30), ("hclen", 19)}
)


@pytest.fixture(scope="module")
def zvalid():
    return K.zstd_valid()


@pytest.fixture(scope="module")
def ivalid():
    return K.inflate_valid()


def test_every_branch_has_a_stream(zvalid, ivalid):
    zf = set().union(*(f for *_, f in zvalid))
    inf = set().union(*(f for *_, f in ivalid))
    assert not ZSTD_BRANCHES - zf, sorted(map(str, ZSTD_BRANCHES - zf))
    assert not INFLATE_BRANCHES - inf, sorted(map(str, INFLATE_BRANCHES - inf))
    assert {ofv for (_, ofv, _) in [f for f in zf if f[0] == "repeat"]} == {1, 2, 3}
    # one malformed stream per status code a stream can reach (BOUNDS is a meta row's, built by the GPU test)
    assert {m[3] for m in K.zstd_malformed()} == set(range(1, 13))
    assert {m[4] for m in K.inflate_malformed()} == set(range(1, 11))
    # the header's edges of the 2-byte Frame_Content_Size field, and a fixed size that needs the 4-byte one
    names = {n for n, *_ in zvalid}
    assert {"fcs 256 in 2 bytes", "fcs 65791 in 2 bytes", "fcs 65792 in 4 bytes"} <= names


@needs_libzstd
def test_libzstd_decodes_every_valid_stream(zvalid):
    for name, stream, want, _ in zvalid:
        assert W.zstd_decompress(stream, len(want) + 64) == want, name


@needs_libzstd
def test_libzstd_rejects_every_malformed_stream():
    for name, stream, cap, status, libzstd_rejects in K.zstd_malformed():
        got = W.zstd_decompress(stream, cap)
        if libzstd_rejects:
            assert got is None, name
        else:   # the decoder is documented to be stricter here than libzstd, which decodes the stream
            assert got is not None, name


def test_zlib_inflates_every_valid_stream(ivalid):
    for name, raw, want, _ in ivalid:
        assert zlib.decompress(raw, -15) == want, name


def test_zlib_rejects_every_malformed_member():
    for name, raw, isize, crc, _ in K.inflate_malformed():
        with pytest.raises(zlib.error):
            zlib.decompress(C.member(raw, b"", isize, crc), 31)
        assert name


@needs_libzstd
def test_xxh64_matches_libzstd_checksums(golden_dir):
    c = np.load(f"{golden_dir}/zstd_corpus.npz")
    offs = c["stream_offsets"]
    checked = 0
    for i in range(len(c["labels"])):
        s = c["streams"][offs[i]:offs[i + 1]].tobytes()
        if not s[4] & 4 or s.find(K.MAGIC, 4) >= 0 or b"\x2a\x4d\x18" in s:   # one frame, with a checksum
            continue
        out = W.zstd_decompress(s, int(c["out_lengths"][i]))
        assert struct.unpack("<I", s[-4:])[0] == K.xxh64(out) & 0xffffffff, str(c["labels"][i])
        checked += 1
    assert checked >= 5
    # the published XXH64 test values
    assert K.xxh64(b"") == 0xEF46DB3751D8E999
    assert K.xxh64(b"a") == 0xD24EC4F1A98C6E5B


def test_fse_table_description_round_trip():
    """ncount() against a plain reading of RFC 8878 section 4.1.1, over every accuracy log and zero runs of 0..7."""
    for log in range(5, 10):
        for zeros in range(8):
            counts = {0: 5, zeros + 1: 3, zeros + 2: 40, zeros + 9: 1}
            norm = K.normalize(counts, log, below_one=(zeros + 9,))
            got, used = _read_ncount(K.ncount(norm, log))
            assert got == norm + [0] * (len(got) - len(norm)) and used == len(K.ncount(norm, log))


def _read_ncount(b):
    v, bit = int.from_bytes(b + b"\0" * 8, "little"), 0

    def take(n):
        return (v >> bit) & ((1 << n) - 1)

    log = take(4) + 5
    bit = 4
    remaining, threshold, nb, norm, prev0 = (1 << log) + 1, 1 << log, log + 1, [], False
    while remaining > 1:
        if prev0:
            while True:
                r = take(2)
                bit += 2
                norm += [0] * r
                if r != 3:
                    break
        x = take(nb)
        mx = 2 * threshold - 1 - remaining
        if x & (threshold - 1) < mx:
            c = x & (threshold - 1)
            bit += nb - 1
        else:
            c = x & (2 * threshold - 1)
            if c >= threshold:
                c -= mx
            bit += nb
        c -= 1
        remaining -= abs(c)
        norm.append(c)
        prev0 = c == 0
        while remaining < threshold:
            nb -= 1
            threshold >>= 1
    return norm, (bit + 7) // 8
