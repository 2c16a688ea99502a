"""BAM input on the host: BGZF member headers and their refusals, the BAM record parser on zlib-inflated streams cut
anywhere, and the refusals of `duplex` on unreadable .bam files, which come before any CUDA use."""
import io
import os
import struct
import subprocess
import sys
import zlib

import numpy as np
import pytest

from bonito_b200 import bam

import _bgzf_corpus as C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _member(data=b"hello", extra=b""):
    return C.member(C.deflate(data), data, extra=extra)


def test_member_header_fields_and_an_extra_subfield_before_bc():
    for extra in (b"", b"XY\x03\x00abc"):
        m = _member(b"hello world", extra)
        got, raw, n_raw, crc, isize = bam.next_member(io.BytesIO(m + b"tail"), 0)
        assert got == m and zlib.decompress(m[raw:raw + n_raw], -15) == b"hello world"
        assert (crc, isize) == (zlib.crc32(b"hello world"), 11)
    assert bam.next_member(io.BytesIO(b""), 0) is None
    assert bam.next_member(io.BytesIO(C.EOF_MARKER), 0)[4] == 0


@pytest.mark.parametrize("mutate, what", [
    (lambda m: b"\x1f\x8c" + m[2:], "not a BGZF member header"),
    (lambda m: m[:3] + b"\x05" + m[4:], "not a BGZF member header"),
    (lambda m: m[:12] + b"XY" + m[14:], "no BC subfield"),
    (lambda m: m[:14] + b"\x03\x00" + m[16:], "malformed extra subfield"),
    (lambda m: m[:-4] + struct.pack("<I", 65537), "ISIZE 65537"),
    (lambda m: m[:-3], "truncated member"),
    (lambda m: m[:10], "truncated header"),
])
def test_member_header_refusals_name_the_offset(mutate, what):
    m = mutate(_member())
    with pytest.raises(ValueError, match=f"member at byte 1234: .*{what}"):
        bam.next_member(io.BytesIO(m), 1234)


def test_bgzf_file_check(tmp_path):
    p = tmp_path / "x.bam"
    for content in (b"", b"@HD\tVN:1.6\n", _member()):
        p.write_bytes(content)
        with pytest.raises(ValueError, match="is not a BAM file: empty, or missing the BGZF EOF marker that htslib"):
            bam.check_bgzf_file(str(p))
    p.write_bytes(_member() + C.EOF_MARKER)
    bam.check_bgzf_file(str(p))


# ------------------------------------------------------------------------------------------------ record parser
def _records():
    """(SAM lines, the expected read_records dict) covering every case the reader distinguishes."""
    lines = [
        "r1\t256\t*\t0\t0\t*\t*\t0\t0\tACGT\t!!!!",                       # secondary, then supplementary, first
        "r1\t2048\t*\t0\t0\t*\t*\t0\t0\tACGT\t!!!!",
        "r1\t4\t*\t0\t0\t*\t*\t0\t0\tACGTNACGTT\t+++++,,,,,\tqs:i:20\tmv:B:c,5,1,0,1",
        "r1\t4\t*\t0\t0\t*\t*\t0\t0\tGGGG\t!!!!",                          # a later duplicate primary
        "r2\t16\tctg\t3\t60\t2S5M1I2M\t*\t0\t0\tTTGCAMRWSA\t0123456789\tNM:i:1\tMD:Z:7\tde:f:0.5",
        "r3\t4\t*\t0\t0\t*\t*\t0\t0\t*\t*",
        "r4\t4\t*\t0\t0\t*\t*\t0\t0\tACG\t*",
        "r5\t0\tctg\t1\t0\t3M\t*\t0\t0\tAC=\t$$$\tRG:Z:x",
    ]
    want = {"r1": ("ACGTNACGTT", np.array([10] * 5 + [11] * 5, np.uint8)),
            "r2": ("TTGCAMRWSA", np.arange(15, 25, dtype=np.uint8)),
            "r3": ("*", None), "r4": ("ACG", None), "r5": ("AC=", np.array([3, 3, 3], np.uint8))}
    return lines, want


def _stream(lines):
    ref_ids = {"ctg": 0}
    return bam.encode_header("@HD\tVN:1.6\n@SQ\tSN:ctg\tLN:100\n", [("ctg", 100)]) + \
        b"".join(bam.encode_record(line, ref_ids) for line in lines)


def _same(got, want):
    assert got.keys() == want.keys()
    for k, (seq, q) in want.items():
        assert got[k][0] == seq, k
        assert (got[k][1] is None) == (q is None) and (q is None or np.array_equal(got[k][1], q)), k


def test_records_match_the_sam_reader(tmp_path):
    from bonito_b200.cli import duplex as cli
    lines, want = _records()
    stream = zlib.decompress(zlib.compress(_stream(lines), 6))
    _same(bam.records_from_chunks([stream]), want)
    sam = tmp_path / "r.sam"
    sam.write_text("@HD\tVN:1.6\n" + "\n".join(lines) + "\n")
    _same(cli.read_records(str(sam)), want)
    _same(bam.records_from_chunks([stream], wanted={"r2", "r9"}), {"r2": want["r2"]})


def test_records_cut_at_every_byte_of_the_record_boundaries():
    lines, want = _records()
    stream = _stream(lines)
    header = len(_stream([]))
    bounds, p = [], header
    while p < len(stream):
        bounds.append(p)
        p += 4 + struct.unpack_from("<i", stream, p)[0]
    cuts = sorted({c for b in [0, header] + bounds for c in range(max(0, b - 6), min(len(stream), b + 40))})
    for cut in cuts:
        _same(bam.records_from_chunks([stream[:cut], stream[cut:]]), want)
    for a in range(header - 3, header + 45, 2):          # three chunks, one of them empty
        _same(bam.records_from_chunks([stream[:a], b"", stream[a:a + 7], stream[a + 7:]]), want)


@pytest.mark.parametrize("mutate, what", [
    (lambda b: struct.pack("<i", 31) + b[4:], "block_size 31 < 32"),
    (lambda b: struct.pack("<i", struct.unpack_from("<i", b)[0] - 2) + b[4:-2], "overrun block_size"),
    (lambda b: b[:12] + b"\x00" + b[13:], "not NUL-terminated"),
    (lambda b: b[:-1], "truncated"),
])
def test_malformed_record_names_its_index(mutate, what):
    lines, _ = _records()
    good = b"".join(bam.encode_record(line, {"ctg": 0}) for line in lines[:2])
    last = bam.encode_record("bad\t4\t*\t0\t0\t*\t*\t0\t0\tACGT\t!!!!", {})
    stream = bam.encode_header("", []) + good + mutate(last)
    with pytest.raises(ValueError, match=f"record 2: .*{what}"):
        bam.records_from_chunks([stream])


def test_malformed_header_and_aux():
    with pytest.raises(ValueError, match="not a BAM stream"):
        bam.records_from_chunks([b"BAM\2" + bytes(8)])
    with pytest.raises(ValueError, match="ends inside its header"):
        bam.records_from_chunks([bam.encode_header("@HD\n", [])[:-2]])
    body = bam.encode_record("x\t4\t*\t0\t0\t*\t*\t0\t0\tACGT\t!!!!", {}) + b""
    bad_aux = body + b"XZZabc"                                    # an unterminated Z field
    bad_aux = struct.pack("<i", len(bad_aux) - 4) + bad_aux[4:]
    with pytest.raises(ValueError, match="record 0: unterminated Z/H"):
        bam.records_from_chunks([bam.encode_header("", []) + bad_aux])


# ------------------------------------------------------------------------------------------------ duplex CLI
def _run(args, env):
    return subprocess.run([sys.executable, "-m", "bonito_b200", "duplex", *args], cwd=ROOT, capture_output=True, text=True,
                          env=env)


def test_duplex_refuses_unreadable_bam_before_cuda(tmp_path):
    pairs = tmp_path / "pairs.txt"
    pairs.write_text("a b\n")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    full = _member(b"x" * 100) + C.EOF_MARKER
    for name, content in (("empty.bam", b""), ("cut.bam", full[:-5]), ("text.bam", b"@HD\tVN:1.6\n")):
        (tmp_path / name).write_bytes(content)
        res = _run([str(tmp_path / name), str(pairs)], env)
        assert res.returncode == 1 and len(res.stderr.strip().splitlines()) == 1, res.stderr
        assert "is not a BAM file: empty, or missing the BGZF EOF marker that htslib writes" in res.stderr
    (tmp_path / "ok.bam").write_bytes(full)                       # passes the host check, then needs the GPU
    res = _run([str(tmp_path / "ok.bam"), str(pairs)], env)
    assert res.returncode == 1 and "is not a BAM file" not in res.stderr
    assert res.stderr.strip().splitlines()[-1].startswith("> error:")
    (tmp_path / "r.cram").write_bytes(b"")
    res = _run([str(tmp_path / "r.cram"), str(pairs)], env)
    assert res.returncode == 1 and res.stderr.strip() == \
        "> error: CRAM input needs htslib, which this build does not bundle; convert to .sam or .fastq"
