"""b200_bgzf_decompress and the BAM input of `duplex` on the GPU: zlib-made members inflate byte for byte, the project's
compressor round-trips, each malformed member gets its status without disturbing its neighbours, the reader's output
does not depend on its launch size, and BAM input gives what the same records give as SAM."""
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest
import torch

from bonito_b200 import bam, native

import _bgzf_corpus as C

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def inflate(members, meta_rows=None):
    """(outputs, statuses) of one b200_bgzf_decompress launch over [(raw, isize, crc)]."""
    raws = b"".join(r for r, _, _ in members)
    rows, at, out_at = [], 0, 0
    for raw, isize, crc in members:
        rows.append([at, len(raw), out_at, isize, crc])
        at, out_at = at + len(raw), out_at + isize
    if meta_rows is not None:
        rows = [rows[i] if r is None else r for i, r in enumerate(meta_rows)]
    inp = torch.from_numpy(np.frombuffer(raws + b"\0", dtype=np.uint8).copy()).cuda()[:len(raws)]
    meta = torch.tensor(rows, dtype=torch.int64, device="cuda")
    out = torch.full((max(out_at, 1),), 0xAB, dtype=torch.uint8, device="cuda")[:out_at]
    status = torch.full((len(members),), -1, dtype=torch.int32, device="cuda")
    native.bgzf_decompress(inp, meta, out, status)
    torch.cuda.synchronize()
    out, offs = out.cpu().numpy().tobytes(), [r[2] for r in rows]
    return [out[o:o + m[1]] for o, m in zip(offs, members)], status.cpu().tolist()


def test_inflates_zlib_members_byte_for_byte():
    members = C.valid_members()
    outs, status = inflate([(raw, len(data), zlib.crc32(data)) for _, raw, data in members])
    for (name, raw, data), got, st in zip(members, outs, status):
        assert st == 0 and got == data == zlib.decompress(raw, -15), name


def test_round_trip_through_the_compressor_over_more_than_one_wave():
    from test_gpu_bgzf import _bam_stream, _sam_text, compress
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n_members = 32 * sms                       # more warps than the SMs hold at once
    base = _bam_stream(_sam_text(n_reads=400, seed=9))
    data = (base * -(-n_members * bam.native.BGZF_MEMBER_INPUT // len(base)))[:n_members * native.BGZF_MEMBER_INPUT - 77]
    packed, off = compress(data)
    import io
    fh, members, where = io.BytesIO(packed), [], 0
    while (m := bam.next_member(fh, where)) is not None:
        member, raw, n_raw, crc, isize = m
        members.append((member[raw:raw + n_raw], isize, crc))
        where += len(member)
    assert len(members) == n_members
    outs, status = inflate(members)
    assert status == [0] * n_members and b"".join(outs) == data


def test_malformed_members_between_good_ones():
    good = [(C.deflate(d), len(d), zlib.crc32(d)) for d in (b"A" * 3000 + bytes(range(256)), b"tail " * 999)]
    cases = [(name, (raw, isize, 0), st) for name, raw, isize, st in C.malformed()]
    text = bytes(range(200))
    cases.append(("crc", (C.deflate(text), 200, zlib.crc32(text) ^ 1), C.CRC))
    for name, member, want in cases:
        outs, status = inflate([good[0], member, good[1]])
        assert status == [0, want, 0], name
        assert outs[0] == zlib.decompress(good[0][0], -15) and outs[2] == zlib.decompress(good[1][0], -15), name
    # a meta row reaching past the input, and an ISIZE over 65536
    for row in ([0, 1 << 40, 0, 10, 0], [0, 5, 0, 65537, 0]):
        outs, status = inflate([good[0], (b"", 0, 0), good[1]], [None, row, None])
        assert status == [0, C.BOUNDS, 0] and outs[2] == zlib.decompress(good[1][0], -15)


def test_reader_error_names_the_member_offset(tmp_path):
    first = C.member(C.deflate(b"x" * 5000), b"x" * 5000)
    for name, raw, isize, want in C.malformed():
        bad = C.member(raw, b"", isize=isize, crc=0)
        p = tmp_path / "bad.bam"
        p.write_bytes(first + bad + first + C.EOF_MARKER)
        with pytest.raises(ValueError, match=f"member at byte {len(first)}: {native.INFLATE_STATUS[want]}"):
            list(bam.BgzfReader(str(p), members_per_launch=4))
    p.write_bytes(first * 3)
    with pytest.raises(ValueError, match="does not end with the BGZF EOF marker"):
        list(bam.BgzfReader(str(p)))


# ------------------------------------------------------------------------------------------------ BAM files
def _sam_to_bam(sam_path, bam_path, writer, seed=0):
    lines = sam_path.read_text().splitlines()
    header = "".join(l + "\n" for l in lines if l.startswith("@"))
    contigs = []
    for l in lines:
        if l.startswith("@SQ"):
            f = dict(x.split(":", 1) for x in l.split("\t")[1:])
            contigs.append((f["SN"], int(f["LN"])))
    records = [l for l in lines if l and not l.startswith("@")]
    with open(bam_path, "wb") as fh:
        if writer == "gpu":
            out = bam.BamOutput(fh, header, contigs)
            for l in records:
                out.write_sam(l)
            out.close()
        else:                                  # zlib level 6 with members of random sizes and an empty member
            ids = {n: i for i, (n, _) in enumerate(contigs)}
            stream = bam.encode_header(header, contigs) + b"".join(bam.encode_record(l, ids) for l in records)
            fh.write(C.bgzf_file(stream, np.random.default_rng(seed), max_member=20000, empty_at=1))
    return bam_path


def _same_reads(a, b):
    assert a.keys() == b.keys() and len(a) > 0
    for k in a:
        assert a[k][0] == b[k][0], k
        assert (a[k][1] is None) == (b[k][1] is None) and (a[k][1] is None or np.array_equal(a[k][1], b[k][1])), k


def _golden_sam(tmp_path):
    from test_duplex import _write_inputs, load_golden
    pairs = list(load_golden())
    pfile = tmp_path / "pairs.txt"
    pfile.write_text("temp comp\n" + "".join(f"{p[0]} {p[1]}\n" for p in pairs))
    return _write_inputs(tmp_path, pairs, "sam"), pfile


def test_reader_windows_and_parity_with_the_sam_reader(tmp_path):
    from bonito_b200.cli import duplex as cli
    sam, _ = _golden_sam(tmp_path)
    want = cli.read_records(str(sam))
    for writer in ("gpu", "zlib"):
        path = _sam_to_bam(sam, tmp_path / f"{writer}.bam", writer)
        streams = [b"".join(bam.BgzfReader(str(path), members_per_launch=m)) for m in (1, 3, 1024)]
        assert streams[0] == streams[1] == streams[2]
        for m in (1, 3, 1024):
            _same_reads(bam.read_records(str(path), members_per_launch=m), want)
        _same_reads(cli.read_records(str(path)), want)
        wanted = set(list(want)[:5])
        _same_reads(cli.read_records(str(path), wanted=wanted), cli.read_records(str(sam), wanted=wanted))


def _run_to(cmd, path):
    with open(path, "wb") as fh:
        p = subprocess.run(cmd, cwd=ROOT, stdout=fh, stderr=subprocess.PIPE, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    return p.stderr


def _duplex(reads, pfile, out):
    """`duplex reads pairs > out`, the output with the input path (in the @PG command line) replaced by <reads>."""
    _run_to([sys.executable, "-m", "bonito_b200", "duplex", str(reads), str(pfile)], out)
    return out.read_bytes().replace(str(reads).encode(), b"<reads>")


def test_duplex_from_bam_equals_duplex_from_sam(tmp_path):
    sam, pfile = _golden_sam(tmp_path)
    want = _duplex(sam, pfile, tmp_path / "from_sam.sam")
    assert want.count(b"\n") > 2
    for writer in ("gpu", "zlib"):
        path = _sam_to_bam(sam, tmp_path / f"reads_{writer}.bam", writer)
        assert _duplex(path, pfile, tmp_path / f"from_{writer}.sam") == want


def test_basecaller_then_duplex_through_bam(tmp_path):
    from bonito_b200.cli import duplex as cli
    from test_gpu_bgzf import _model_and_reads
    from _map_helpers import _fasta
    from bonito_b200 import aligner as A
    mdir, rdir = _model_and_reads(tmp_path)
    base = [sys.executable, "-m", "bonito_b200", "basecaller", mdir, str(rdir), "--no-trim"]
    _run_to(base, tmp_path / "calls.bam")
    _run_to(base, tmp_path / "calls.sam")
    ids = sorted(cli.read_records(str(tmp_path / "calls.sam")))
    pfile = tmp_path / "pairs.txt"
    pfile.write_text("temp comp\n" + "".join(f"{a} {b}\n" for a, b in zip(ids[0::2], ids[1::2])))
    assert _duplex(tmp_path / "calls.bam", pfile, tmp_path / "d_bam.sam") == \
        _duplex(tmp_path / "calls.sam", pfile, tmp_path / "d_sam.sam")
    _same_reads(cli.read_records(str(tmp_path / "calls.bam")), cli.read_records(str(tmp_path / "calls.sam")))

    # aligned records (`--reference`): flags, CIGARs and tags, read back as the SAM run's records
    sam = (tmp_path / "calls.sam").read_text().splitlines()
    calls = {f[0]: f[9] for f in (l.split("\t") for l in sam if not l.startswith("@"))}
    _fasta(tmp_path / "ref.fa", [(f"ctg_{rid}", np.frombuffer((A.revcomp(s) if i % 2 else s).encode(), np.uint8))
                               for i, (rid, s) in enumerate(sorted(calls.items()))])
    ref = ["--reference", str(tmp_path / "ref.fa")]
    _run_to(base + ref, tmp_path / "aligned.sam")
    want = cli.read_records(str(tmp_path / "aligned.sam"))
    _same_reads(cli.read_records(str(tmp_path / "aligned.sam")), want)
    for writer in ("gpu", "zlib"):
        path = _sam_to_bam(tmp_path / "aligned.sam", tmp_path / f"aligned_{writer}.bam", writer, seed=3)
        _same_reads(cli.read_records(str(path)), want)
