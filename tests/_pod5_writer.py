"""
A POD5 writer for the tests, written from the published POD5 layout and the VBZ definition, independent of the reader in
bonito_b200/pod5.py:

  * svb16 (StreamVByte-16) with numpy: ceil(n / 8) key bytes, LSB first (a set bit: the value takes 2 bytes, little-endian),
    then the data bytes; VBZ codes the int16 samples as zigzag(delta from 0) in 16-bit arithmetic before packing;
  * zstd through the system libzstd.so.1 (ctypes, ZSTD_compress2), with settable level, checksum, content-size flag and
    target block size; `have_libzstd()` says whether it is present;
  * the Arrow tables with pyarrow, the extension types named in the field metadata as MinKNOW names them;
  * the container: signature, section markers, the embedded tables, FOOTER, a flatbuffer footer and its length.
"""
import ctypes
import ctypes.util
import struct
import uuid
from datetime import datetime, timezone

import numpy as np
import pyarrow as pa

SIGNATURE = b"\x8bPOD\r\n\x1a\n"
MARKER = uuid.UUID("f5a3a2c1-1b4e-4c8a-9b2d-3e7f6a5b4c3d").bytes
READS_TABLE, SIGNAL_TABLE, RUN_INFO_TABLE = 0, 1, 4
ROW_SAMPLES = 102400  # pod5's signal row size

# --------------------------------------------------------------------------------------------------------------- svb16


def zigzag_delta(samples):
    s = np.asarray(samples, dtype=np.int16).astype(np.uint16)
    d = np.diff(s, prepend=np.uint16(0)).astype(np.uint16)
    return ((d << np.uint16(1)) ^ (d.view(np.int16) >> np.int16(15)).view(np.uint16)).astype(np.uint16)


def svb16_encode_values(values):
    """svb16 of uint16 values: keys, then data."""
    v = np.asarray(values, dtype=np.uint16)
    two = v > 255
    keys = np.packbits(two, bitorder="little")
    lo = (v & 0xff).astype(np.uint8)
    hi = (v >> 8).astype(np.uint8)
    data = np.stack([lo, hi], 1).reshape(-1)[np.stack([np.ones_like(two), two], 1).reshape(-1)]
    return keys.tobytes() + data.tobytes()


def svb16_encode(samples):
    """The svb16 stage of VBZ: zigzag-delta int16 samples, packed."""
    return svb16_encode_values(zigzag_delta(samples))


def svb16_decode(buf, count):
    """numpy inverse of svb16_encode (the oracle of the GPU decoder); None when the length is not keys + data."""
    b = np.frombuffer(buf, dtype=np.uint8)
    nkeys = (count + 7) // 8
    if len(b) < nkeys:
        return None
    two = np.unpackbits(b[:nkeys], bitorder="little")[:count].astype(bool)
    if len(b) != nkeys + count + int(two.sum()):
        return None
    if count == 0:
        return np.empty(0, np.int16)
    pos = np.concatenate([[0], np.cumsum(1 + two)[:-1]]).astype(np.int64) + nkeys
    z = b[pos].astype(np.uint16)
    z[two] |= b[pos[two] + 1].astype(np.uint16) << 8
    d = (z >> 1) ^ (0 - (z & 1)).astype(np.uint16)
    return np.cumsum(d, dtype=np.uint16).view(np.int16)


# ---------------------------------------------------------------------------------------------------------------- zstd
_ZSTD = None


def _zstd():
    global _ZSTD
    if _ZSTD is None:
        lib = ctypes.CDLL(ctypes.util.find_library("zstd") or "libzstd.so.1")
        lib.ZSTD_createCCtx.restype = ctypes.c_void_p
        lib.ZSTD_freeCCtx.argtypes = [ctypes.c_void_p]
        lib.ZSTD_CCtx_setParameter.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
        lib.ZSTD_CCtx_setParameter.restype = ctypes.c_size_t
        lib.ZSTD_compressBound.argtypes = [ctypes.c_size_t]
        lib.ZSTD_compressBound.restype = ctypes.c_size_t
        lib.ZSTD_compress2.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_size_t, ctypes.c_char_p, ctypes.c_size_t]
        lib.ZSTD_compress2.restype = ctypes.c_size_t
        lib.ZSTD_decompress.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_char_p, ctypes.c_size_t]
        lib.ZSTD_decompress.restype = ctypes.c_size_t
        lib.ZSTD_isError.argtypes = [ctypes.c_size_t]
        lib.ZSTD_versionNumber.restype = ctypes.c_uint
        _ZSTD = lib
    return _ZSTD


def have_libzstd():
    try:
        _zstd()
        return True
    except OSError:
        return False


# ZSTD_cParameter values (zstd.h): compressionLevel, windowLog, contentSizeFlag, checksumFlag, targetCBlockSize
_LEVEL, _WINDOW_LOG, _CONTENT_SIZE, _CHECKSUM, _TARGET_BLOCK = 100, 101, 200, 201, 1005


def zstd_compress(data, level=1, checksum=False, content_size=True, target_block=0, window_log=0):
    """One zstd frame of `data` from libzstd's ZSTD_compress2."""
    lib = _zstd()
    cctx = lib.ZSTD_createCCtx()
    try:
        params = [(_LEVEL, level), (_CHECKSUM, int(checksum)), (_CONTENT_SIZE, int(content_size))]
        params += [(_TARGET_BLOCK, target_block)] if target_block else []
        params += [(_WINDOW_LOG, window_log)] if window_log else []
        for k, v in params:
            if lib.ZSTD_isError(lib.ZSTD_CCtx_setParameter(cctx, k, v)):
                raise ValueError(f"libzstd refuses parameter {k} = {v}")
        cap = lib.ZSTD_compressBound(len(data))
        out = ctypes.create_string_buffer(cap)
        n = lib.ZSTD_compress2(cctx, out, cap, bytes(data), len(data))
        if lib.ZSTD_isError(n):
            raise ValueError("ZSTD_compress2 failed")
        return out.raw[:n]
    finally:
        lib.ZSTD_freeCCtx(cctx)


def zstd_decompress(blob, capacity):
    """libzstd's ZSTD_decompress: the output bytes, or None for an error."""
    lib = _zstd()
    out = ctypes.create_string_buffer(max(capacity, 1))
    n = lib.ZSTD_decompress(out, capacity, bytes(blob), len(blob))
    return None if lib.ZSTD_isError(n) else out.raw[:n]


def vbz_compress(samples, level=1, **kw):
    return zstd_compress(svb16_encode(samples), level=level, **kw)


# ------------------------------------------------------------------------------------------------------------ footer


class _Flat:
    """A forward flatbuffer builder: every referenced object is written after its referrer (uoffsets are unsigned)."""

    def __init__(self):
        self.b = bytearray()

    def align(self, n):
        self.b += b"\0" * (-len(self.b) % n)

    def u32_at(self, pos, target):
        struct.pack_into("<I", self.b, pos, target - pos)


def footer_bytes(contents, software="bonito_b200 test writer", version="0.3.10"):
    """The Footer flatbuffer: file_identifier, software, pod5_version, contents [EmbeddedFile]."""
    f = _Flat()
    f.b += b"\0" * 4                                        # root uoffset
    vt = len(f.b)
    f.b += struct.pack("<6H", 12, 20, 4, 8, 12, 16)         # vtable: 4 uoffset fields
    f.align(4)
    table = len(f.b)
    f.b += struct.pack("<i", table - vt) + b"\0" * 16
    f.u32_at(0, table)
    for i, text in enumerate(["5b2e2f9e-5a7c-4b1e-9d3f-0c6a8e4b2d10", software, version]):
        f.align(4)
        f.u32_at(table + 4 + 4 * i, len(f.b))
        raw = text.encode()
        f.b += struct.pack("<I", len(raw)) + raw + b"\0"
    f.align(4)
    vec = len(f.b)
    f.u32_at(table + 16, vec)
    f.b += struct.pack("<I", len(contents)) + b"\0" * 4 * len(contents)
    for i, (offset, length, content_type) in enumerate(contents):
        f.align(4)
        evt = len(f.b)
        f.b += struct.pack("<6H", 12, 28, 8, 16, 24, 26)
        f.align(8)
        et = len(f.b)
        f.b += struct.pack("<iIqqhh", et - evt, 0, offset, length, 0, content_type) + b"\0" * 4
        f.u32_at(vec + 4 + 4 * i, et)
    f.align(8)
    return bytes(f.b)


# ------------------------------------------------------------------------------------------------------------- tables


def _ext(name, typ, ext):
    return pa.field(name, typ, metadata={b"ARROW:extension:name": ext.encode(), b"ARROW:extension:metadata": b""})


def _ipc(table):
    sink = pa.BufferOutputStream()
    with pa.ipc.new_file(sink, table.schema) as w:
        w.write_table(table, max_chunksize=1000)
    return sink.getvalue().to_pybytes()


RUN_INFO = dict(acquisition_id="a5e1c3d2b4f60718293a4b5c6d7e8f9012345678", acquisition_start_time_ms=1700000000123,
                adc_max=2047, adc_min=-2048, experiment_name="exp", flow_cell_id="FAX12345", flow_cell_product_code="FLO-MIN114",
                protocol_name="sequencing/sequencing_MIN114_DNA", protocol_run_id="c0ffee00-1111-2222-3333-444455556666",
                protocol_start_time_ms=1699999990000, sample_id="sample_7", sample_rate=5000, sequencing_kit="sqk-lsk114",
                sequencer_position="MN12345", sequencer_position_type="MinION Mk1B", software="MinKNOW 23.07",
                system_name="host-7", system_type="Linux", context_tags={"sample_frequency": "5000", "experiment_type": "genomic_dna"},
                tracking_id={"run_id": "a5e1c3d2b4f60718293a4b5c6d7e8f9012345678", "exp_start_time": "2023-11-14T22:13:20Z",
                             "flow_cell_id": "FAX12345"})


def run_info_table(infos):
    ts = pa.timestamp("ms", tz="UTC")
    smap = pa.map_(pa.string(), pa.string())
    cols = {
        "acquisition_id": pa.array([r["acquisition_id"] for r in infos], pa.string()),
        "acquisition_start_time": pa.array([r["acquisition_start_time_ms"] for r in infos], ts),
        "adc_max": pa.array([r["adc_max"] for r in infos], pa.int16()),
        "adc_min": pa.array([r["adc_min"] for r in infos], pa.int16()),
        "context_tags": pa.array([list(r["context_tags"].items()) for r in infos], smap),
        "experiment_name": pa.array([r["experiment_name"] for r in infos], pa.string()),
        "flow_cell_id": pa.array([r["flow_cell_id"] for r in infos], pa.string()),
        "flow_cell_product_code": pa.array([r["flow_cell_product_code"] for r in infos], pa.string()),
        "protocol_name": pa.array([r["protocol_name"] for r in infos], pa.string()),
        "protocol_run_id": pa.array([r["protocol_run_id"] for r in infos], pa.string()),
        "protocol_start_time": pa.array([r["protocol_start_time_ms"] for r in infos], ts),
        "sample_id": pa.array([r["sample_id"] for r in infos], pa.string()),
        "sample_rate": pa.array([r["sample_rate"] for r in infos], pa.uint16()),
        "sequencing_kit": pa.array([r["sequencing_kit"] for r in infos], pa.string()),
        "sequencer_position": pa.array([r["sequencer_position"] for r in infos], pa.string()),
        "sequencer_position_type": pa.array([r["sequencer_position_type"] for r in infos], pa.string()),
        "software": pa.array([r["software"] for r in infos], pa.string()),
        "system_name": pa.array([r["system_name"] for r in infos], pa.string()),
        "system_type": pa.array([r["system_type"] for r in infos], pa.string()),
        "tracking_id": pa.array([list(r["tracking_id"].items()) for r in infos], smap),
    }
    return pa.table(cols)


def _dictionary(values, pool):
    return pa.DictionaryArray.from_arrays(pa.array([pool.index(v) for v in values], pa.int16()), pa.array(pool, pa.string()))


def write_pod5(path, reads, vbz=True, row_samples=ROW_SAMPLES, level=1, run_infos=None, drop_columns=(), retype=None,
               **zstd_kw):
    """Write `reads` (dicts: read_id (uuid.UUID), signal (int16), and optional channel, well, read_number, start,
    calibration_offset, calibration_scale, run_info (an acquisition id)) as a POD5 file.  Returns the reads' signal rows."""
    run_infos = run_infos or [RUN_INFO]
    rows, row_ids, row_bytes, row_counts, read_rows = [], [], [], [], []
    for r in reads:
        sig = np.asarray(r["signal"], dtype=np.int16)
        idx = []
        for a in range(0, max(len(sig), 1), row_samples):
            part = sig[a:a + row_samples]
            idx.append(len(rows))
            rows.append(part)
            row_ids.append(r["read_id"].bytes)
            row_counts.append(len(part))
            if vbz:
                row_bytes.append(vbz_compress(part, level=level, **zstd_kw))
        read_rows.append(idx)
    uuid_t = pa.binary(16)
    if vbz:
        sig_field = _ext("signal", pa.large_binary(), "minknow.vbz")
        sig_col = pa.array(row_bytes, pa.large_binary())
    else:
        sig_field = pa.field("signal", pa.large_list(pa.int16()))
        sig_col = pa.array([p.tolist() for p in rows], pa.large_list(pa.int16()))
    signal = pa.Table.from_arrays([pa.array(row_ids, uuid_t), sig_col, pa.array(row_counts, pa.uint32())],
                                  schema=pa.schema([_ext("read_id", uuid_t, "minknow.uuid"), sig_field,
                                                    pa.field("samples", pa.uint32())]))
    acq = [ri["acquisition_id"] for ri in run_infos]
    n = len(reads)
    get = lambda k, d: [r.get(k, d(i)) for i, r in enumerate(reads)]  # noqa: E731
    cols = [
        (_ext("read_id", uuid_t, "minknow.uuid"), pa.array([r["read_id"].bytes for r in reads], uuid_t)),
        (pa.field("signal", pa.list_(pa.uint64())), pa.array(read_rows, pa.list_(pa.uint64()))),
        (pa.field("read_number", pa.uint32()), pa.array(get("read_number", lambda i: 100 + i), pa.uint32())),
        (pa.field("start", pa.uint64()), pa.array(get("start", lambda i: 5000 * i + 17), pa.uint64())),
        (pa.field("median_before", pa.float32()), pa.array([200.0] * n, pa.float32())),
        (pa.field("num_minknow_events", pa.uint64()), pa.array([0] * n, pa.uint64())),
        (pa.field("tracked_scaling_scale", pa.float32()), pa.array([1.0] * n, pa.float32())),
        (pa.field("tracked_scaling_shift", pa.float32()), pa.array([0.0] * n, pa.float32())),
        (pa.field("predicted_scaling_scale", pa.float32()), pa.array([1.0] * n, pa.float32())),
        (pa.field("predicted_scaling_shift", pa.float32()), pa.array([0.0] * n, pa.float32())),
        (pa.field("num_reads_since_mux_change", pa.uint32()), pa.array([0] * n, pa.uint32())),
        (pa.field("time_since_mux_change", pa.float32()), pa.array([0.0] * n, pa.float32())),
        (pa.field("num_samples", pa.uint64()), pa.array([len(r["signal"]) for r in reads], pa.uint64())),
        (pa.field("channel", pa.uint16()), pa.array(get("channel", lambda i: 1 + i % 512), pa.uint16())),
        (pa.field("well", pa.uint8()), pa.array(get("well", lambda i: 1 + i % 4), pa.uint8())),
        (pa.field("pore_type", pa.dictionary(pa.int16(), pa.string())), _dictionary(["not_set"] * n, ["not_set"])),
        (pa.field("calibration_offset", pa.float32()), pa.array(get("calibration_offset", lambda i: -243.0 + i), pa.float32())),
        (pa.field("calibration_scale", pa.float32()), pa.array(get("calibration_scale", lambda i: 0.1462 + 0.0001 * i),
                                                               pa.float32())),
        (pa.field("end_reason", pa.dictionary(pa.int16(), pa.string())), _dictionary(["signal_positive"] * n, ["unknown", "signal_positive"])),
        (pa.field("end_reason_forced", pa.bool_()), pa.array([False] * n, pa.bool_())),
        (pa.field("run_info", pa.dictionary(pa.int16(), pa.string())), _dictionary(get("run_info", lambda i: acq[i % len(acq)]), acq)),
    ]
    cols = [(f, a) for f, a in cols if f.name not in drop_columns]
    if retype:
        cols = [(pa.field(f.name, retype[f.name]), a.cast(retype[f.name])) if f.name in retype else (f, a) for f, a in cols]
    reads_t = pa.Table.from_arrays([a for _, a in cols], schema=pa.schema([f for f, _ in cols]))
    tables = [(SIGNAL_TABLE, _ipc(signal)), (RUN_INFO_TABLE, _ipc(run_info_table(run_infos))), (READS_TABLE, _ipc(reads_t))]
    out = bytearray(SIGNATURE + MARKER)
    contents = []
    for content_type, blob in tables:
        contents.append((len(out), len(blob), content_type))
        out += blob + b"\0" * (-len(blob) % 8) + MARKER
    out += b"FOOTER\0\0"
    foot = footer_bytes(contents)
    out += foot + struct.pack("<q", len(foot)) + MARKER + SIGNATURE
    with open(path, "wb") as fh:
        fh.write(out)
    return rows


def synthetic_reads(n, seed=0, min_len=3000, max_len=30000):
    """Reads of squiggle-like int16 signals (level steps plus noise, with rare large jumps), random UUIDs."""
    rng = np.random.default_rng(seed)
    reads = []
    for i in range(n):
        length = int(rng.integers(min_len, max_len))
        levels = rng.normal(500, 120, length // 10 + 1).repeat(10)[:length]
        sig = levels + rng.normal(0, 12, length)
        jumps = rng.random(length) < 0.002
        sig[jumps] += rng.choice([-20000, 20000], jumps.sum())
        reads.append(dict(read_id=uuid.UUID(bytes=rng.bytes(16), version=4), signal=np.clip(sig, -32768, 32767).astype(np.int16)))
    return reads


def expected_pa(read, index):
    """The pA signal the reference computes for a read this writer wrote (bonito/pod5.py:57)."""
    off = np.float32(read.get("calibration_offset", -243.0 + index))
    scale = np.float32(read.get("calibration_scale", 0.1462 + 0.0001 * index))
    return float(scale) * (np.asarray(read["signal"], np.int16).astype(np.float32) + float(off))


def utc_ms(ms):
    return datetime.fromtimestamp(ms // 1000, tz=timezone.utc).replace(microsecond=(ms % 1000) * 1000)
