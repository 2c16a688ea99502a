"""POD5 input on the host: the test writer's svb16 encoder against hand-worked vectors, the container's refusals, the
uncompressed-signal path end to end, the reads' metadata against the reference's formulas (bonito/pod5.py:18-67),
read-id selection and the @RG lines.  Nothing here touches CUDA: uncompressed rows are decoded on the host."""
import os
import shutil
import struct
from datetime import timedelta, timezone

import numpy as np
import pyarrow as pa
import pytest

from bonito_b200.pod5 import Pod5File
from bonito_b200.reader import Read, Reader

import _pod5_writer as W

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
EXPECTED = np.load(os.path.join(GOLDEN, "pod5_expected.npz"))


def _expected():
    ids, sig, offs = EXPECTED["read_ids"], EXPECTED["signals"], EXPECTED["offsets"]
    return [(str(ids[i]), sig[offs[i]:offs[i + 1]]) for i in range(len(ids))]


# ----------------------------------------------------------------------------------------------------------------- svb16
def test_svb16_one_byte_values():
    v = np.arange(256)
    assert W.svb16_encode_values(v) == bytes(32) + bytes(range(256))


def test_svb16_two_byte_values():
    assert W.svb16_encode_values([256, 0x1234, 0xffff]) == bytes([0b111, 0x00, 0x01, 0x34, 0x12, 0xff, 0xff])
    assert W.svb16_encode_values([1, 0x100, 2]) == bytes([0b010, 0x01, 0x00, 0x01, 0x02])


@pytest.mark.parametrize("n, want", [
    (0, b""),
    (1, bytes([0, 5])),
    (7, bytes([0b1000000]) + bytes([1, 2, 3, 4, 5, 6, 0x2c, 0x01])),
    (8, bytes([0b10000000]) + bytes([1, 2, 3, 4, 5, 6, 7, 0x2c, 0x01])),
    (9, bytes([0b10000000, 0b1]) + bytes([1, 2, 3, 4, 5, 6, 7, 0x2c, 0x01, 0x00, 0x10])),
])
def test_svb16_counts(n, want):
    values = {0: [], 1: [5], 7: [1, 2, 3, 4, 5, 6, 300], 8: [1, 2, 3, 4, 5, 6, 7, 300],
              9: [1, 2, 3, 4, 5, 6, 7, 300, 0x1000]}[n]
    assert W.svb16_encode_values(values) == want
    assert np.array_equal(W.svb16_decode(want, n).view(np.uint16), np.cumsum(
        [(z >> 1) ^ -(z & 1) for z in values], dtype=np.int64).astype(np.uint16) if n else np.empty(0, np.uint16))


def test_vbz_deltas_wrap_across_the_int16_range():
    # deltas 32767, +1 (mod 2^16), -1: zigzag 0xfffe, 2, 1
    assert W.svb16_encode([32767, -32768, 32767]) == bytes([0b001, 0xfe, 0xff, 0x02, 0x01])
    assert W.svb16_encode([-32768, 32767]) == bytes([0b01, 0xff, 0xff, 0x01])
    for s in ([32767, -32768, 32767], [-32768, 32767, 0, -1, -32768]):
        assert np.array_equal(W.svb16_decode(W.svb16_encode(s), len(s)), np.array(s, np.int16))


# ------------------------------------------------------------------------------------------------------------- container
def _raw(tmp_path):
    path = tmp_path / "ok.pod5"
    shutil.copy(os.path.join(GOLDEN, "pod5_raw.pod5"), path)
    return path


def _footer(data):
    flen = struct.unpack_from("<q", data, len(data) - 32)[0]
    return len(data) - 32 - flen, flen


def _patched(tmp_path, edit, name="bad.pod5"):
    data = bytearray(_raw(tmp_path).read_bytes())
    edit(data)
    path = tmp_path / name
    path.write_bytes(bytes(data))
    return path


def _table_offsets(data):
    """(offset, position of the int64 offset in the file, position of content_type) per footer entry of our writer."""
    fstart, flen = _footer(data)
    foot = bytes(data[fstart:fstart + flen])
    out = []
    for ct in (W.SIGNAL_TABLE, W.RUN_INFO_TABLE, W.READS_TABLE):
        for p in range(0, flen - 20, 8):
            off, length, fmt, c = struct.unpack_from("<qqhh", foot, p)
            if 24 <= off < fstart and 0 < length and fmt == 0 and c == ct and data[off:off + 6] == b"ARROW1":
                out.append((off, fstart + p, fstart + p + 18))
                break
    return out


def test_the_golden_files_open():
    assert Pod5File(os.path.join(GOLDEN, "pod5_raw.pod5")).vbz is False
    assert Pod5File(os.path.join(GOLDEN, "pod5_vbz.pod5")).vbz is True


@pytest.mark.parametrize("edit, message", [
    (lambda d: d.__delitem__(slice(len(d) // 2, None)), "bad signature"),
    (lambda d: d.__setitem__(slice(0, 8), b"\x89PNG\r\n\x1a\n"), "bad signature"),
    (lambda d: d.__setitem__(slice(len(d) - 32, len(d) - 24), struct.pack("<q", len(d))), "reaches outside the file"),
])
def test_container_refusals(tmp_path, edit, message):
    with pytest.raises(ValueError, match=message) as err:
        Pod5File(str(_patched(tmp_path, edit)))
    assert "bad.pod5" in str(err.value)


def test_truncated_file_is_refused(tmp_path):
    path = _patched(tmp_path, lambda d: d.__delitem__(slice(40, None)))
    with pytest.raises(ValueError, match="too short"):
        Pod5File(str(path))


def test_embedded_range_out_of_bounds(tmp_path):
    data = bytearray(_raw(tmp_path).read_bytes())
    _, pos, _ = _table_offsets(data)[0]
    struct.pack_into("<q", data, pos, len(data) - 100)
    (tmp_path / "bad.pod5").write_bytes(bytes(data))
    with pytest.raises(ValueError, match="outside the file's body"):
        Pod5File(str(tmp_path / "bad.pod5"))


def test_embedded_table_without_arrow_magic(tmp_path):
    data = bytearray(_raw(tmp_path).read_bytes())
    off, _, _ = _table_offsets(data)[1]
    data[off:off + 6] = b"ARROWX"
    (tmp_path / "bad.pod5").write_bytes(bytes(data))
    with pytest.raises(ValueError, match="ARROW1"):
        Pod5File(str(tmp_path / "bad.pod5"))


def test_missing_table(tmp_path):
    data = bytearray(_raw(tmp_path).read_bytes())
    _, _, ct = _table_offsets(data)[1]   # the run info table becomes "OtherIndex"
    struct.pack_into("<h", data, ct, 3)
    (tmp_path / "bad.pod5").write_bytes(bytes(data))
    with pytest.raises(ValueError, match="no run info table"):
        Pod5File(str(tmp_path / "bad.pod5"))


def test_missing_and_mistyped_columns(tmp_path):
    reads = W.synthetic_reads(2, seed=1, min_len=500, max_len=600)
    W.write_pod5(tmp_path / "a.pod5", reads, vbz=False, drop_columns=("calibration_scale",))
    with pytest.raises(ValueError, match="a.pod5.*no column 'calibration_scale'"):
        Pod5File(str(tmp_path / "a.pod5"))
    W.write_pod5(tmp_path / "b.pod5", reads, vbz=False, retype={"channel": pa.uint32()})
    with pytest.raises(ValueError, match="b.pod5.*'channel' has type uint32"):
        Pod5File(str(tmp_path / "b.pod5"))
    c = tmp_path / "c"
    c.mkdir()
    W.write_pod5(c / "c.pod5", reads, vbz=False, drop_columns=("num_samples",))
    with pytest.raises(ValueError, match="c.pod5"):  # the Reader refuses a directory holding such a file
        Reader(str(c))


# ------------------------------------------------------------------------------------------------------- reads, metadata
def test_uncompressed_pod5_end_to_end_matches_npy(tmp_path):
    """Reads of the uncompressed file give the writer's int16 input, and Read.signal equals that of an .npy file holding
    the same pA array, bit for bit."""
    want = _expected()
    got = list(Pod5File(os.path.join(GOLDEN, "pod5_raw.pod5")).signals())
    assert [g[0] for g in got] == [w[0] for w in want]
    for (rid, raw, off, scale, meta), (_, sig) in zip(got, want):
        assert raw.dtype == np.int16 and np.array_equal(raw, sig)
    pod = tmp_path / "pod5"
    pod.mkdir()
    shutil.copy(os.path.join(GOLDEN, "pod5_raw.pod5"), pod)
    npy = tmp_path / "npy"
    npy.mkdir()
    for rid, raw, off, scale, meta in got:
        np.save(npy / f"{rid}.npy", np.float32(scale) * (raw.astype(np.float32) + np.float32(off)))
    a = {r.read_id: r for r in Reader(str(pod)).get_reads(str(pod))}
    b = {r.read_id: r for r in Reader(str(npy)).get_reads(str(npy))}
    assert sorted(a) == sorted(b) and len(a) == 8
    for rid in a:
        assert a[rid].signal.tobytes() == b[rid].signal.tobytes()
        assert (a[rid].shift, a[rid].scale, a[rid].trimmed_samples) == (b[rid].shift, b[rid].scale, b[rid].trimmed_samples)


def test_read_metadata_follows_the_reference_formulas():
    info = W.RUN_INFO
    f = Pod5File(os.path.join(GOLDEN, "pod5_raw.pod5"))
    t0 = W.utc_ms(info["acquisition_start_time_ms"])
    for i, (rid, raw, off, scale, meta) in enumerate(f.signals()):
        rate = int(info["context_tags"]["sample_frequency"])
        start = (5000 * i + 17) / rate
        read = Read(rid, scale * (raw.astype(np.float32) + off), filename="pod5_raw.pod5", meta=meta)
        assert read.run_id == info["acquisition_id"]
        assert (read.sample_id, read.flow_cell_id, read.device_id) == (info["sample_id"], info["flow_cell_id"],
                                                                       info["sequencer_position"])
        assert read.exp_start_time == t0.isoformat().replace("Z", "") == "2023-11-14T22:13:20.123000+00:00"
        assert (read.channel, read.mux, read.read_number) == (1 + i % 512, 1 + i % 4, 100 + i)
        assert read.sample_rate == rate and read.start == start and read.duration == len(raw) / rate
        assert read.start_time == (t0 + timedelta(seconds=start)).astimezone(timezone.utc).isoformat(timespec="milliseconds")
        assert read.template_start == start + read.trimmed_samples / rate
        assert read.template_duration == len(raw) / rate - read.trimmed_samples / rate
        assert (off, scale) == (float(np.float32(-243.0 + i)), float(np.float32(0.1462 + 0.0001 * i)))
        tags = read.tagdata()
        assert "f5:Z:pod5_raw.pod5" in tags and f"ch:i:{1 + i % 512}" in tags and f"st:Z:{read.start_time}" in tags


def test_read_id_selection_and_skip(tmp_path):
    shutil.copy(os.path.join(GOLDEN, "pod5_raw.pod5"), tmp_path)
    ids = [w[0] for w in _expected()]
    r = Reader(str(tmp_path))
    keep = {ids[1], ids[5], "not-a-read"}
    assert [x.read_id for x in r.get_reads(str(tmp_path), read_ids=keep)] == [ids[1], ids[5]]
    assert [x.read_id for x in r.get_reads(str(tmp_path), read_ids=keep, skip=True)] == [i for i in ids if i not in keep]
    assert [x.read_id for x in r.get_reads(str(tmp_path))] == ids


def test_read_groups(tmp_path):
    shutil.copy(os.path.join(GOLDEN, "pod5_raw.pod5"), tmp_path)
    info = W.RUN_INFO
    run_id = info["tracking_id"]["run_id"]
    assert Reader(str(tmp_path)).get_read_groups(str(tmp_path), "dna_model") == [
        f"@RG\tID:{run_id}_dna_model\tPL:ONT\tDT:{info['tracking_id']['exp_start_time']}\tPU:{info['flow_cell_id']}\t"
        f"PM:{info['system_name']}\tLB:{info['sample_id']}\tSM:{info['sample_id']}\t"
        f"DS:run_id={run_id} basecall_model=dna_model"]
    # the records' RG:Z tag names the same group
    read = next(Reader(str(tmp_path)).get_reads(str(tmp_path)))
    assert f"{read.run_id}_dna_model" == f"{run_id}_dna_model"
    npy = tmp_path / "npy"
    npy.mkdir()
    np.save(npy / "r.npy", np.zeros(100, np.float32))
    assert Reader(str(npy)).get_read_groups(str(npy), "dna_model") == []
