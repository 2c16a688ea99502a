"""b200_zstd_decompress, b200_svb16_decode and POD5 input on the GPU: the libzstd corpus decodes to what libzstd gives
(its length and SHA-256), each malformed stream gets its status between intact neighbours, svb16 rows match the numpy
oracle, the reader's output does not depend on its window size, POD5 reads give the writer's samples, and `basecaller`
on POD5 matches `.npy` input."""
import hashlib
import os
import shutil
import struct
import subprocess
import sys

import numpy as np
import pytest
import torch

from bonito_b200 import native
from bonito_b200.pod5 import Pod5File

import _pod5_writer as W

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
MAGIC = struct.pack("<I", 0xFD2FB528)


def _corpus():
    """(label, stream, output length, SHA-256 of the output) per libzstd stream of the corpus."""
    c = np.load(os.path.join(GOLDEN, "zstd_corpus.npz"))
    st = c["stream_offsets"]
    return [(str(label), c["streams"][st[i]:st[i + 1]].tobytes(), int(c["out_lengths"][i]), c["sha256"][i].tobytes())
            for i, label in enumerate(c["labels"])]


def decompress(streams, caps, meta_rows=None):
    """(outputs, out_len, statuses) of one b200_zstd_decompress launch."""
    blob = b"".join(streams)
    rows, at, oat = [], 0, 0
    for s, cap in zip(streams, caps):
        rows.append([at, len(s), oat, cap])
        at, oat = at + len(s), oat + cap
    if meta_rows is not None:
        rows = [rows[i] if r is None else r for i, r in enumerate(meta_rows)]
    inp = torch.from_numpy(np.frombuffer(blob + b"\0", dtype=np.uint8).copy()).cuda()[:len(blob)]
    meta = torch.tensor(rows, dtype=torch.int64, device="cuda")
    out = torch.full((max(oat, 1),), 0xAB, dtype=torch.uint8, device="cuda")[:oat]
    out_len = torch.full((len(streams),), -1, dtype=torch.int64, device="cuda")
    status = torch.full((len(streams),), -1, dtype=torch.int32, device="cuda")
    native.zstd_decompress(inp, meta, out, out_len, status)
    torch.cuda.synchronize()
    host, lens = out.cpu().numpy().tobytes(), out_len.cpu().tolist()
    return [host[r[2]:r[2] + n] for r, n in zip(rows, lens)], lens, status.cpu().tolist()


def test_corpus_decodes_byte_for_byte():
    corpus = _corpus()
    outs, lens, st = decompress([c[1] for c in corpus], [c[2] + 64 for c in corpus])
    for (label, _, want_len, want_sha), got, n, s in zip(corpus, outs, lens, st):
        assert s == 0, (label, native.ZSTD_STATUS.get(s))
        assert n == want_len == len(got) and hashlib.sha256(got).digest() == want_sha, label


def _frame(fhd, *parts):
    return MAGIC + bytes([fhd]) + b"".join(parts)


def _block(last, btype, content, size=None):
    size = len(content) if size is None else size
    return struct.pack("<I", int(last) | btype << 1 | size << 3)[:3] + content


def _seq_block(ofcode, bits, modes=0x54):
    """A compressed block of no literals and one sequence whose LL / OF / ML tables are RLE (LL 0, OF `ofcode`, ML 3);
    `bits` is the bit stream, the end marker included."""
    return bytes([0x00, 0x01, modes, 0, ofcode, 0]) + bytes(bits)


MALFORMED = {
    1: (b"\x00\x01\x02\x03\x04\x05", 16),
    2: (_frame(0x28, b"\x05", _block(1, 0, b"abcde")), 16),                            # reserved bit
    3: (_frame(0x20, b"\x05", _block(1, 3, b"abcde")), 16),                            # block type 3
    4: (_frame(0x20, b"\x05", _block(1, 2, bytes([0x03 | 5 << 4, 1 << 6, 0]) + b"\x00\x00")), 16),  # Treeless, no table
    5: (_frame(0x20, b"\x05", _block(1, 2, bytes([0x02 | 5 << 4, 2 << 6, 0]) + bytes([129, 0x00]) + b"\x00")), 16),
    6: (_frame(0x20, b"\x05", _block(1, 2, bytes([0x00, 0x01, 0x80, 0x0f, 0x00]))), 16),  # accuracy log 20
    7: (_frame(0x20, b"\x05", _block(1, 2, bytes([0x00, 0x01, 0x55, 0, 5, 0, 0x20]))), 16),  # reserved mode bits
    8: (_frame(0x20, b"\x05", _block(1, 2, _seq_block(5, [0x20]))), 16),              # offset 29 before any output
    9: (_frame(0x00, b"\x00", _block(1, 0, b"0123456789")), 5),                        # 10 bytes into 5
    10: (_frame(0x20, b"\x0b", _block(1, 0, b"0123456789")), 16),                      # content size 11, 10 written
    11: (_frame(0x20, b"\x0a", _block(1, 0, b"01234", size=10)), 16),                 # raw block cut short
    12: (_frame(0x24, b"\x0a", _block(1, 0, b"0123456789"), b"\x00\x00\x00\x00"), 16),  # wrong checksum
}


def test_malformed_streams_between_good_ones():
    good = _corpus()[:3]
    streams, caps, codes = [], [], []
    for code, (blob, cap) in MALFORMED.items():
        g = good[code % 3]
        streams += [g[1], blob]
        caps += [g[2], cap]
        codes += [0, code]
    g = good[0]
    streams += [g[1], g[1], g[1]]
    caps += [g[2]] * 3
    codes += [0, 13, 0]
    meta_rows = [None] * (len(streams) - 2) + [[0, 10 ** 12, 0, 8], None]   # a row reaching past the input
    outs, lens, st = decompress(streams, caps, meta_rows)
    assert st == codes, [(native.ZSTD_STATUS.get(a), native.ZSTD_STATUS.get(b)) for a, b in zip(st, codes) if a != b]
    for s, c, o, cap in zip(streams, codes, outs, caps):
        if c == 0:
            assert hashlib.sha256(o).digest() == next(g[3] for g in good if g[1] == s)


def _literal_block(bits):
    """8 raw literals, then one sequence of RLE tables: LL 8, offset code 0 (repeat offset 1), ML 3."""
    return _block(1, 2, bytes([8 << 3]) + b"abcdefgh" + bytes([0x01, 0x54, 8, 0, 0]) + bytes(bits))


def test_repeat_offsets_and_an_exactly_consumed_bit_stream():
    outs, lens, st = decompress([_frame(0x20, b"\x0b", _literal_block([0x01]))], [16])
    assert st == [0] and outs == [b"abcdefghhhh"]
    outs, lens, st = decompress([_frame(0x20, b"\x0b", _literal_block([0x03]))], [16])  # one bit left unread
    assert st == [7]
    # with no literals the first repeat offset is Rep2 = 4, before the frame's first byte
    assert decompress([_frame(0x20, b"\x00", _block(1, 2, _seq_block(0, [0x01])))], [16])[2] == [8]


def _svb(rows, meta_rows=None):
    blob = b"".join(r for r, _ in rows)
    meta, at, oat = [], 0, 0
    for r, n in rows:
        meta.append([at, len(r), n, oat])
        at, oat = at + len(r), oat + n
    if meta_rows is not None:
        meta = [meta[i] if m is None else m for i, m in enumerate(meta_rows)]
    inp = torch.from_numpy(np.frombuffer(blob + b"\0", dtype=np.uint8).copy()).cuda()[:len(blob)]
    out = torch.full((max(oat, 1),), 0x5555, dtype=torch.int16, device="cuda")[:oat]
    status = torch.full((len(rows),), -1, dtype=torch.int32, device="cuda")
    native.svb16_decode(inp, torch.tensor(meta, dtype=torch.int64, device="cuda").reshape(-1, 4), out, status)
    torch.cuda.synchronize()
    host = out.cpu().numpy()
    return [host[m[3]:m[3] + n] for m, (_, n) in zip(meta, rows)], status.cpu().tolist()


def test_svb16_edges_against_the_oracle():
    rng = np.random.default_rng(3)
    sigs = [np.empty(0, np.int16), np.array([5], np.int16), rng.integers(-300, 300, 7).astype(np.int16),
            rng.integers(-300, 300, 8).astype(np.int16), rng.integers(-300, 300, 9).astype(np.int16),
            np.array([32767, -32768, 32767, 0, -1, -32768], np.int16), np.arange(256, dtype=np.int16),
            rng.integers(-32768, 32767, 1000).astype(np.int16), rng.integers(-100, 100, 257).astype(np.int16),
            rng.integers(-2000, 2000, 102400).astype(np.int16)]
    rows = [(W.svb16_encode(s), len(s)) for s in sigs]
    outs, st = _svb(rows + [(rows[7][0] + b"\x00", 1000), (rows[7][0][:-1], 1000), (b"", 9), rows[3]],
                    meta_rows=[None] * (len(rows) + 3) + [[0, 10 ** 12, 8, 0]])
    assert st == [0] * len(rows) + [1, 1, 1, 2]
    for s, (enc, n), o in zip(sigs, rows, outs):
        assert np.array_equal(o, s) and np.array_equal(W.svb16_decode(enc, n), s)


def test_svb16_over_more_rows_than_one_wave():
    reads = W.synthetic_reads(20000, seed=9, min_len=1, max_len=700)
    rows = [(W.svb16_encode(r["signal"]), len(r["signal"])) for r in reads]
    outs, st = _svb(rows)
    assert st == [0] * len(rows)
    assert all(np.array_equal(o, r["signal"]) for o, r in zip(outs, reads))


def _expected():
    e = np.load(os.path.join(GOLDEN, "pod5_expected.npz"))
    ids, sig, offs = e["read_ids"], e["signals"], e["offsets"]
    return [(str(ids[i]), sig[offs[i]:offs[i + 1]]) for i in range(len(ids))]


def test_pod5_reads_give_the_writers_samples():
    want = _expected()
    for name in ("pod5_vbz.pod5", "pod5_raw.pod5"):
        got = list(Pod5File(os.path.join(GOLDEN, name)).signals())
        assert [g[0] for g in got] == [w[0] for w in want]
        for g, (_, sig) in zip(got, want):
            assert g[1].dtype == np.int16 and np.array_equal(g[1], sig), name


def test_output_does_not_depend_on_the_window_size():
    f = Pod5File(os.path.join(GOLDEN, "pod5_vbz.pod5"))
    ref = [(g[0], g[1].tobytes()) for g in f.signals()]
    for rows, nbytes in ((1, 1 << 30), (3, 1 << 30), (4096, 1), (4096, 5000)):
        assert [(g[0], g[1].tobytes()) for g in f.signals(window_rows=rows, window_bytes=nbytes)] == ref


def test_a_bad_row_names_the_file_row_and_status(tmp_path):
    reads = W.synthetic_reads(3, seed=2, min_len=3000, max_len=4000)
    W.write_pod5(tmp_path / "x.pod5", reads, vbz=True, checksum=True)
    data = bytearray((tmp_path / "x.pod5").read_bytes())
    blob = W.vbz_compress(reads[1]["signal"], level=1, checksum=True)
    at = bytes(data).find(blob)
    assert at > 0
    data[at + len(blob) - 1] ^= 0xff   # the checksum's last byte
    (tmp_path / "x.pod5").write_bytes(bytes(data))
    with pytest.raises(ValueError, match=r"x.pod5: signal row 1 .*checksum mismatch"):
        list(Pod5File(str(tmp_path / "x.pod5")).signals())


def _run_to(cmd, path):
    with open(path, "wb") as fh:
        p = subprocess.run(cmd, cwd=ROOT, stdout=fh, stderr=subprocess.PIPE, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]


def test_basecaller_on_pod5_matches_npy(tmp_path):
    from oracle import synth
    spec = synth.model_spec("fast", n_lstm=3)
    mdir = synth.write_model_dir(str(tmp_path / "model"), spec, synth.make_weights(spec, seed=4), batchsize=8,
                                 chunksize=2000, overlap=120)
    pod, npy = tmp_path / "pod5", tmp_path / "npy"
    pod.mkdir()
    npy.mkdir()
    shutil.copy(os.path.join(GOLDEN, "pod5_vbz.pod5"), pod)
    for rid, raw, off, scale, meta in Pod5File(str(pod / "pod5_vbz.pod5")).signals():
        np.save(npy / f"{rid}.npy", np.float32(scale) * (raw.astype(np.float32) + np.float32(off)))
    out = {}
    for src in ("pod5", "npy"):
        for ext in ("fastq", "sam"):
            path = tmp_path / f"{src}.{ext}"
            _run_to([sys.executable, "-m", "bonito_b200", "basecaller", mdir, str(tmp_path / src)], path)
            out[src, ext] = path.read_text().replace(str(tmp_path / src), "<reads>")  # the @PG command line
    # the same records; POD5 reads come in reads-table order, .npy files in file name order
    fastq = {}
    for src in ("pod5", "npy"):
        lines = out[src, "fastq"].splitlines()
        fastq[src] = sorted("\n".join(lines[i:i + 4]) for i in range(0, len(lines), 4))
    assert fastq["pod5"] == fastq["npy"] and len(fastq["pod5"]) == 8

    meta_tags = ("RG", "mx", "ch", "st", "du", "rn", "f5")

    def split(text):
        head = [l for l in text.splitlines() if l.startswith("@")]
        recs = {}
        for l in text.splitlines():
            if not l.startswith("@"):
                f = l.split("\t")
                recs[f[0]] = (f[:11], [t for t in f[11:] if t[:2] not in meta_tags], {t[:2]: t for t in f[11:]})
        return head, recs

    ph, pr = split(out["pod5", "sam"])
    nh, nr = split(out["npy", "sam"])
    assert [h for h in ph if not h.startswith("@RG")] == [h for h in nh if not h.startswith("@RG")]
    info = W.RUN_INFO
    rg = [h for h in ph if h.startswith("@RG")]
    group = f"{info['tracking_id']['run_id']}_model"
    assert len(rg) == 1 and rg[0].startswith(f"@RG\tID:{group}\tPL:ONT\t") and f"PU:{info['flow_cell_id']}" in rg[0]
    assert not [h for h in nh if h.startswith("@RG")]
    assert sorted(pr) == sorted(nr) and len(pr) == 8
    f = Pod5File(str(pod / "pod5_vbz.pod5"))
    metas = {g[0]: g[4] for g in f.signals()}
    for rid in pr:
        assert pr[rid][:2] == nr[rid][:2]
        tags, m = pr[rid][2], metas[rid]
        assert tags["RG"] == f"RG:Z:{group}" and tags["f5"] == "f5:Z:pod5_vbz.pod5"
        assert tags["ch"] == f"ch:i:{m['channel']}" and tags["mx"] == f"mx:i:{m['mux']}"
        assert tags["rn"] == f"rn:i:{m['read_number']}" and tags["st"] == f"st:Z:{m['start_time']}"
