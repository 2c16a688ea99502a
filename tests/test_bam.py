"""BAM record and header encoding (bonito_b200.bam) against the independent decoder of tests/_oracle_bam.py: the decoded
header and records are the SAM text the text writer produces for the same inputs.  No GPU: the uncompressed stream is
checked here, its BGZF compression in test_gpu_bgzf.py."""
import io
import struct
from types import SimpleNamespace

import numpy as np
import pytest

from bonito_b200 import bam
from bonito_b200.aligner import Mapping
from bonito_b200.io import Writer, read_tags, sam_header, sam_record

from _oracle_bam import decode_bam, decode_record, same_sam_line

CONTIGS = [("chr1", 5000), ("chr2", 80000)]


class FakeRead(SimpleNamespace):
    def tagdata(self):
        return [f"mx:i:{self.mux}", f"ch:i:{self.channel}", f"st:Z:{self.start_time}", f"du:f:{self.duration}",
                f"rn:i:{self.read_number}", f"f5:Z:{self.filename}", f"sm:f:{self.shift}", f"sd:f:{self.scale}",
                f"sv:Z:{self.scaling_strategy}"]


def _read(i, rng, length=200, start_time=""):
    return FakeRead(read_id=f"read_{i:04d}", signal=np.zeros(length * 6, np.float32), run_id="run0", mux=1, channel=100 + i,
                    start_time=start_time, duration=1.23456789 * (i + 1), read_number=i, filename=f"f{i}.pod5",
                    shift=93.7 + i / 7, scale=23.51, scaling_strategy="quantile", trimmed_samples=10 * i, num_samples=length * 6)


def _result(rng, length, mapping=None, qstring=True):
    seq = "".join(rng.choice(list("ACGT"), length))
    res = {"sequence": seq, "qstring": "".join(chr(33 + q) for q in rng.integers(5, 40, length)) if qstring else "*",
           "stride": 6, "moves": (rng.random(length * 3) < 0.3).astype(np.int8)}
    if mapping is not None:
        res["mapping"] = mapping
    return res


def _mapping(ctg, r_st, strand, q_st, q_en, cigar_str):
    return Mapping(ctg=ctg, r_st=r_st, r_en=r_st + 10, q_st=q_st, q_en=q_en, strand=strand, mapq=37, cigar_str=cigar_str, NM=3,
                   MD="5A4")


def _stream(writer_results, contigs):
    """(SAM text from Writer(mode="w"), the BAM stream of the same lines)."""
    text = io.StringIO()
    w = Writer(iter(writer_results), fd=text, mode="w", group_key="model", contigs=contigs)
    w.run()
    assert w.error is None
    sam = text.getvalue()
    header = sam_header([], contigs=contigs)
    ref_ids = {name: i for i, (name, _) in enumerate(contigs or ())}
    raw = bam.encode_header(header, contigs or []) + b"".join(
        bam.encode_record(line, ref_ids) for line in sam.splitlines() if not line.startswith("@"))
    return sam, raw


def test_header_and_records_decode_to_the_sam_text():
    rng = np.random.default_rng(7)
    results = []
    for i in range(8):
        length = int(rng.integers(50, 400))
        mapping = None
        if i % 4 == 1:
            mapping = _mapping("chr1", 100 + i, +1, 5, length - 3, f"{length - 20}M2I3D10M2D5M1X2=")
        elif i % 4 == 2:
            mapping = _mapping("chr2", 70000 + i, -1, 0, length - 9, f"{length - 9}M")
        results.append((_read(i, rng, length, start_time="" if i == 3 else "2024-01-01T00:00:00Z"),
                        _result(rng, length, mapping, qstring=i != 5)))
    sam, raw = _stream(results, CONTIGS)
    text, refs, lines, info = decode_bam(raw)
    assert text == sam_header([], contigs=CONTIGS) and refs == CONTIGS
    want = [line for line in sam.splitlines() if not line.startswith("@")]
    assert len(lines) == len(want) == 8
    for got, exp in zip(lines, want):
        assert same_sam_line(got, exp), (got[:300], exp[:300])
    assert "st:Z:\t" in want[3] and lines[5].split("\t")[10] == "*"
    assert any("\t16\tchr2\t" in line for line in lines) and any("\t0\tchr1\t" in line for line in lines)


def test_unaligned_header_has_no_references():
    rng = np.random.default_rng(1)
    sam, raw = _stream([(_read(0, rng), _result(rng, 33))], None)
    text, refs, lines, _ = decode_bam(raw)
    assert refs == [] and text == sam.split("read_0000")[0] and same_sam_line(lines[0], sam.splitlines()[-1])


@pytest.mark.parametrize("value,typ", [(-2 ** 31, "i"), (-32769, "i"), (-32768, "s"), (-129, "s"), (-128, "c"), (-1, "c"),
                                       (0, "C"), (255, "C"), (256, "S"), (65535, "S"), (65536, "I"), (2 ** 32 - 1, "I")])
def test_integer_tags_take_the_smallest_type(value, typ):
    enc = bam.encode_tag(f"XY:i:{value}")
    assert enc[:3] == b"XY" + typ.encode()
    assert struct.unpack("<" + {"c": "b", "C": "B", "s": "h", "S": "H", "i": "i", "I": "I"}[typ], enc[3:])[0] == value


def test_other_tag_types():
    assert bam.encode_tag("st:Z:") == b"stZ\0"
    assert bam.encode_tag("XA:A:q") == b"XAAq"
    assert bam.encode_tag("du:f:0.1") == b"duf" + struct.pack("<f", 0.1)
    mv = np.array([1, 0, 0, 1, 1, 0], dtype=np.int8)
    assert bam.encode_tag("mv:B:c,12,1,0,0,1,1,0") == b"mvBc" + struct.pack("<i", 7) + bytes([12]) + mv.tobytes()
    assert bam.encode_tag("XB:B:s,-300,7,12") == b"XBBs" + struct.pack("<i3h", 3, -300, 7, 12)
    assert bam.encode_tag("XF:B:f,1.5,-2") == b"XFBf" + struct.pack("<i2f", 2, 1.5, -2.0)


@pytest.mark.parametrize("pos,cigar,want", [(-1, None, 4680), (0, "10M", 4681), (16383, "1M", 4681), (16383, "2M", 585),
                                            (100000, "50M5D50M", 4687), (0, "200000M", 73), (5, "3S", 4681)])
def test_bin(pos, cigar, want):
    """htslib's hts_reg2bin(pos, end, 14, 5); end = pos + 1 without reference bases (4680 for an unmapped record)."""
    if pos < 0:
        line = "\t".join(["r", "4", "*", "0", "0", "*", "*", "0", "0", "ACGT", "*"])
    else:
        line = "\t".join(["r", "0", "chr1", str(pos + 1), "60", cigar, "*", "0", "0", "*", "*"])
    rec = bam.encode_record(line, {"chr1": 0})
    assert struct.unpack_from("<H", rec, 4 + 10)[0] == want


def test_long_cigar_goes_to_a_cg_tag():
    ops = ["1M", "1I", "1M", "1D"] * 17500   # 70 000 ops
    cigar = "".join(ops)
    l_seq = 17500 * 3
    ref_len = 17500 * 3
    seq = "A" * l_seq
    line = "\t".join(["long", "0", "chr1", "11", "60", cigar, "*", "0", "0", seq, "*", "NM:i:35000"])
    rec = bam.encode_record(line, {"chr1": 0})
    _, fields = decode_record(rec[4:], CONTIGS)
    n_cigar = struct.unpack_from("<H", rec, 4 + 12)[0]
    assert n_cigar == 2
    raw = struct.unpack_from("<2I", rec, 4 + 32 + len("long") + 1)
    assert raw == (l_seq << 4 | 4, ref_len << 4 | 3)
    assert fields["bin"] == bam.reg2bin(10, 10 + ref_len)
    got, _ = decode_record(rec[4:], CONTIGS)
    assert got.split("\t")[5] == cigar and got.endswith("\tNM:i:35000")
    assert rec.endswith(b"CGBI" + struct.pack("<i", 70000) + np.array(
        [1 << 4 | 0, 1 << 4 | 1, 1 << 4 | 0, 1 << 4 | 2] * 17500, dtype="<u4").tobytes())


def test_long_read_names_are_refused():
    line = "\t".join(["r" * 255, "4", "*", "0", "0", "*", "*", "0", "0", "ACGT", "*"])
    with pytest.raises(ValueError, match="at most 254"):
        bam.encode_record(line)
    bam.encode_record("\t".join(["r" * 254] + line.split("\t")[1:]))


def test_text_writers_keep_refusing_binary_modes():
    from bonito_b200.io import DuplexWriter
    for cls in (Writer, DuplexWriter):
        with pytest.raises(ValueError, match="htslib"):
            cls(iter(()), mode="wb")


def test_reverse_strand_record_matches_sam_record():
    rng = np.random.default_rng(3)
    read, res = _read(1, rng, 60), _result(rng, 60, _mapping("chr2", 5, -1, 2, 57, "40M2I13M"))
    line = sam_record(read.read_id, res["sequence"], res["qstring"], mapping=res["mapping"], tags=read_tags(read, res, "m"))
    got, _ = decode_record(bam.encode_record(line, {"chr1": 0, "chr2": 1})[4:], CONTIGS)
    assert same_sam_line(got, line)
