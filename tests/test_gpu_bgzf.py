"""b200_bgzf_compress and the BAM output of `basecaller` and `duplex` on the GPU, read back by the independent decoder of
tests/_oracle_bam.py: every member inflates to exactly its slice of the input, the files decode to the records of the
SAM runs, and the output is byte-identical from run to run and whatever the launch size."""
import gzip
import io
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest
import torch

from bonito_b200 import bam, native

import _oracle_bam as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M = native.BGZF_MEMBER_INPUT


def compress(data):
    """(members as bytes, offsets) of one b200_bgzf_compress call."""
    inp = torch.from_numpy(np.frombuffer(bytes(data), dtype=np.uint8).copy()).cuda()
    n = native.bgzf_members(inp.numel())
    out = torch.empty(max(n, 1) * native.BGZF_MEMBER_MAX, dtype=torch.uint8, device="cuda")
    off = torch.full((n + 1,), -1, dtype=torch.int64, device="cuda")
    ws = torch.empty(max(native.bgzf_workspace_bytes(inp.numel()), 1), dtype=torch.uint8, device="cuda")
    native.bgzf_compress(inp, out, off, ws)
    torch.cuda.synchronize()
    off = off.cpu().numpy()
    return out[:int(off[-1])].cpu().numpy().tobytes(), off


def check_members(data, packed, off):
    n = -(-len(data) // M)
    assert len(off) == n + 1 and off[0] == 0 and np.all(np.diff(off) > 0) and off[-1] == len(packed)
    members = O.bgzf_members(packed)
    assert len(members) == n
    for i, (cdata, raw) in enumerate(members):
        assert off[i + 1] - off[i] <= 65536
        assert raw == bytes(data[i * M:(i + 1) * M]) == zlib.decompress(cdata, wbits=-15)
    assert gzip.decompress(packed) == bytes(data)
    return members


def zlib1_size(data):
    """Total size of the same members from zlib level 1 (18 + 8 framing bytes each, as BGZF)."""
    return sum(len(zlib.compress(data[i:i + M], 1)) - 6 + 26 for i in range(0, len(data), M))


def _sam_text(n_reads=300, seed=3):
    rng = np.random.default_rng(seed)
    lines = []
    for i in range(n_reads):
        length = int(rng.integers(200, 3000))
        seq = "".join(rng.choice(list("ACGT"), length))
        qual = "".join(chr(33 + int(q)) for q in np.clip(rng.normal(18, 6, length), 2, 50))
        moves = ",".join(str(int(m)) for m in rng.random(length * 2) < 0.45)
        lines.append(f"read_{i:06d}\t4\t*\t0\t0\t*\t*\t0\t0\t{seq}\t{qual}\tNM:i:0\tRG:Z:run_model\tqs:i:{int(rng.integers(5, 30))}"
                     f"\tns:i:{length * 6}\tts:i:0\tmx:i:1\tch:i:{int(rng.integers(1, 512))}\tst:Z:2024-01-01T00:00:00Z"
                     f"\tdu:f:{rng.random() * 10}\tmv:B:c,6,{moves}")
    return ("\n".join(lines) + "\n").encode()


def _bam_stream(text):
    return bam.encode_header("@HD\tVN:1.5\n") + b"".join(bam.encode_record(l) for l in text.decode().splitlines())


@pytest.mark.parametrize("size", [0, 1, 2, 65279, 65280, 65281])
def test_sizes_at_member_edges(size):
    data = np.random.default_rng(size).integers(0, 4, size, dtype=np.uint8).tobytes()
    packed, off = compress(data)
    if size == 0:
        assert packed == b"" and off.tolist() == [0]
        return
    check_members(data, packed, off)


@pytest.mark.parametrize("name", ["one_byte", "random", "period_32768", "period_32769", "sam", "bam"])
def test_inputs_inflate_and_repeat_exactly(name):
    rng = np.random.default_rng(11)
    if name == "one_byte":
        data = b"\x41" * (1 << 20)
    elif name == "random":
        data = rng.integers(0, 256, 3 * M + 1000, dtype=np.uint8).tobytes()
    elif name.startswith("period"):
        period = int(name.split("_")[1])
        unit = rng.integers(0, 256, period, dtype=np.uint8).tobytes()
        data = (unit * (4 * M // period + 2))[:4 * M + 77]
    elif name == "sam":
        data = _sam_text()
    else:
        data = _bam_stream(_sam_text())
    packed, off = compress(data)
    check_members(data, packed, off)
    assert compress(data)[0] == packed
    if name == "one_byte":
        assert len(packed) < len(data) / 100
    if name == "random":      # stored members
        assert all(off[i + 1] - off[i] == M + 31 for i in range(3))
    if name in ("sam", "bam"):
        assert len(packed) <= 1.02 * zlib1_size(data), (len(packed), zlib1_size(data))


def test_one_launch_over_several_waves():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    data = _bam_stream(_sam_text(n_reads=2000, seed=5))
    reps = -(-4 * sms * M // len(data))
    data = (data * reps)[:4 * sms * M + 12345]
    packed, off = compress(data)
    members = check_members(data, packed, off)
    assert len(members) > 4 * sms
    assert compress(data)[0] == packed


def test_writer_output_does_not_depend_on_launch_size():
    stream = _bam_stream(_sam_text(n_reads=700, seed=0))
    files = []
    for members in (1, 3, 256):
        sink = io.BytesIO()
        w = bam.BgzfWriter(sink, members_per_launch=members)
        for i in range(0, len(stream), 100003):      # writes of any size, not aligned to members
            w.write(stream[i:i + 100003])
        w.close()
        files.append(sink.getvalue())
    assert files[0] == files[1] == files[2]
    assert O.bgzf_decompress(files[0]) == stream


# ------------------------------------------------------------------------------------------------ CLIs
def _model_and_reads(tmp_path):
    from oracle import synth
    spec = synth.model_spec("fast", n_lstm=3)
    weights = synth.make_weights(spec, seed=4)
    mdir = synth.write_model_dir(str(tmp_path / "model"), spec, weights, batchsize=8, chunksize=2000, overlap=120)
    rdir = tmp_path / "reads"
    rdir.mkdir()
    for i in range(6):
        np.save(rdir / f"read{i}.npy", 93.7 + 23.5 * synth.squiggle(1, 24000 + 1000 * i, seed=40 + i)[0, 0].numpy())
    return mdir, rdir


def _run_to(cmd, path):
    with open(path, "wb") as fh:
        p = subprocess.run(cmd, cwd=ROOT, stdout=fh, stderr=subprocess.PIPE, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    return p.stderr


def _assert_bam_equals_sam(bam_path, sam_path, contigs=None):
    text, refs, lines, _ = O.decode_bam(O.bgzf_decompress(bam_path.read_bytes()))
    sam = sam_path.read_text()
    header = "".join(l + "\n" for l in sam.splitlines() if l.startswith("@"))
    records = [l for l in sam.splitlines() if not l.startswith("@")]
    assert text == header
    assert len(lines) == len(records) > 0
    for got, want in zip(lines, records):
        assert O.same_sam_line(got, want), (got[:200], want[:200])
    if contigs is not None:
        assert [name for name, _ in refs] == contigs


def test_cli_basecaller_bam(tmp_path):
    from _map_helpers import _fasta
    from bonito_b200 import aligner as A
    mdir, rdir = _model_and_reads(tmp_path)
    base = [sys.executable, "-m", "bonito_b200", "basecaller", mdir, str(rdir), "--no-trim"]
    err = _run_to(base, tmp_path / "out.bam")
    assert "> outputting unaligned bam" in err
    _run_to(base, tmp_path / "out.sam")
    _assert_bam_equals_sam(tmp_path / "out.bam", tmp_path / "out.sam", [])

    sam = (tmp_path / "out.sam").read_text().splitlines()
    calls = {f[0]: f[9] for f in (l.split("\t") for l in sam if not l.startswith("@"))}
    _fasta(tmp_path / "ref.fa", [(f"ctg_{rid}", np.frombuffer((A.revcomp(s) if i % 2 else s).encode(), np.uint8))
                               for i, (rid, s) in enumerate(sorted(calls.items()))])
    ref = ["--reference", str(tmp_path / "ref.fa")]
    err = _run_to(base + ref, tmp_path / "aligned.bam")
    assert "> loading reference" in err and "> outputting aligned bam" in err
    _run_to(base + ref, tmp_path / "aligned.sam")
    _assert_bam_equals_sam(tmp_path / "aligned.bam", tmp_path / "aligned.sam", [f"ctg_{r}" for r in sorted(calls)])
    lines = O.decode_bam(O.bgzf_decompress((tmp_path / "aligned.bam").read_bytes()))[2]
    assert sum(l.split("\t")[1] == "16" for l in lines) == 3

    with open(tmp_path / "out.cram", "wb") as fh:
        p = subprocess.run(base, cwd=ROOT, stdout=fh, stderr=subprocess.PIPE, text=True, timeout=600)
    assert p.returncode == 1 and "htslib" in p.stderr


def test_cli_duplex_bam(tmp_path):
    from test_duplex import _write_inputs, load_golden
    pairs = list(load_golden())
    reads = _write_inputs(tmp_path, pairs, "sam")
    pfile = tmp_path / "pairs.txt"
    pfile.write_text("temp comp\n" + "".join(f"{p[0]} {p[1]}\n" for p in pairs))
    base = [sys.executable, "-m", "bonito_b200", "duplex", str(reads), str(pfile)]
    err = _run_to(base, tmp_path / "out.bam")
    assert "> outputting unaligned bam" in err
    _run_to(base, tmp_path / "out.sam")
    _assert_bam_equals_sam(tmp_path / "out.bam", tmp_path / "out.sam", [])
