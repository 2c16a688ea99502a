"""
POD5 input without the pod5 package: the container is parsed on the host, the VBZ signal rows are decompressed on the GPU.

A POD5 file is the 8-byte signature and a 16-byte section marker, the embedded Arrow IPC files (signal, run-info and reads
tables, each followed by the marker), then `FOOTER\\0\\0`, a flatbuffer footer that lists the embedded files, the footer's
length (int64 LE), the marker and the signature.  The file is memory-mapped; pyarrow opens each table on its mapped
slice.  A malformed container is refused with a ValueError naming the file, before any CUDA use.

A VBZ signal row (`large_binary`, extension `minknow.vbz`) is one zstd frame of svb16-packed, zigzag-delta-coded int16
samples.  Rows go to the GPU in windows of a bounded number of rows and bytes: one host-to-device copy, the zstd and svb16
launches (bonito_b200.native.zstd_decompress / svb16_decode) on the reader's own stream, and one device-to-host copy of
the samples.  Uncompressed rows (`large_list<int16>`) are taken on the host.  The metadata follows the reference's
bonito/pod5.py:18-67 and the read groups its get_read_groups (bonito/pod5.py:84-110).
"""
import os
import struct
import uuid
from collections import OrderedDict
from datetime import datetime, timedelta, timezone

import numpy as np
import pyarrow as pa
import pyarrow.ipc

SIGNATURE = b"\x8bPOD\r\n\x1a\n"
FOOTER_MAGIC = b"FOOTER\0\0"
READS_TABLE, SIGNAL_TABLE, RUN_INFO_TABLE = 0, 1, 4
WINDOW_ROWS = 4096            # signal rows per GPU window
WINDOW_BYTES = 64 << 20       # compressed bytes per GPU window (a window holds at least one read)
_EPOCH = datetime(1970, 1, 1, tzinfo=timezone.utc)


def _is_str(t):
    return pa.types.is_string(t) or pa.types.is_large_string(t)


def _is_dict_str(t):
    return pa.types.is_dictionary(t) and _is_str(t.value_type)


def _is_str_map(t):
    return pa.types.is_map(t) and _is_str(t.key_type) and _is_str(t.item_type)


_UUID = lambda t: pa.types.is_fixed_size_binary(t) and t.byte_width == 16  # noqa: E731
_SIGNAL_COLUMNS = {"read_id": _UUID, "samples": pa.types.is_uint32,
                   "signal": lambda t: pa.types.is_large_binary(t) or (pa.types.is_large_list(t) and t.value_type == pa.int16())}
_READS_COLUMNS = {"read_id": _UUID, "signal": lambda t: pa.types.is_list(t) and t.value_type == pa.uint64(),
                  "read_number": pa.types.is_uint32, "start": pa.types.is_uint64, "num_samples": pa.types.is_uint64,
                  "channel": pa.types.is_uint16, "well": pa.types.is_uint8, "calibration_offset": pa.types.is_float32,
                  "calibration_scale": pa.types.is_float32, "run_info": _is_dict_str}
_RUN_INFO_COLUMNS = {"acquisition_id": _is_str, "acquisition_start_time": pa.types.is_timestamp,
                     "context_tags": _is_str_map, "tracking_id": _is_str_map, "flow_cell_id": _is_str, "sample_id": _is_str,
                     "sequencer_position": _is_str, "system_name": _is_str}


def _footer_contents(buf, name):
    """(offset, length, content_type) of every EmbeddedFile in the Footer flatbuffer `buf`."""
    def get(fmt, p):
        if p < 0 or p + struct.calcsize(fmt) > len(buf):
            raise ValueError(f"{name}: the POD5 footer is malformed (offset {p} outside its {len(buf)} bytes)")
        return struct.unpack_from(fmt, buf, p)[0]

    def field(table, i):  # position of field i of the table at `table`, or None when absent
        vt = table - get("<i", table)
        if 4 + 2 * i >= get("<H", vt):
            return None
        off = get("<H", vt + 4 + 2 * i)
        return table + off if off else None

    root = get("<I", 0)
    p = field(root, 3)  # contents
    if p is None:
        raise ValueError(f"{name}: the POD5 footer lists no embedded tables")
    vec = p + get("<I", p)
    out = []
    for k in range(get("<I", vec)):
        e = vec + 4 + 4 * k
        t = e + get("<I", e)
        vals = [field(t, i) for i in range(4)]
        offset = get("<q", vals[0]) if vals[0] is not None else 0
        length = get("<q", vals[1]) if vals[1] is not None else 0
        content_type = get("<h", vals[3]) if vals[3] is not None else 0
        out.append((offset, length, content_type))
    return out


def _check_columns(table, schema, columns, name):
    for col, ok in columns.items():
        i = schema.get_field_index(col)
        if i < 0:
            raise ValueError(f"{name}: the POD5 {table} table has no column '{col}' (a file older than POD5 v3?)")
        if not ok(schema.field(i).type):
            raise ValueError(f"{name}: the POD5 {table} table's column '{col}' has type {schema.field(i).type}")


class Pod5File:
    """One POD5 file: its three tables, opened on the memory-mapped file."""

    def __init__(self, path):
        self.path, self.name = path, os.path.basename(path)
        size = os.path.getsize(path)
        tail = len(FOOTER_MAGIC) + 8 + 16 + len(SIGNATURE)
        if size < len(SIGNATURE) + 16 + tail:
            raise ValueError(f"{path}: too short for a POD5 file ({size} bytes)")
        self._map = pa.memory_map(path, "r")
        self._buf = self._map.read_buffer()
        mv = memoryview(self._buf)
        if bytes(mv[:8]) != SIGNATURE or bytes(mv[-8:]) != SIGNATURE:
            raise ValueError(f"{path}: not a POD5 file (bad signature)")
        if bytes(mv[8:24]) != bytes(mv[-24:-8]):
            raise ValueError(f"{path}: the POD5 section markers differ")
        flen = struct.unpack_from("<q", mv, size - 32)[0]
        fstart = size - 32 - flen
        if flen <= 0 or fstart - len(FOOTER_MAGIC) < 24:
            raise ValueError(f"{path}: the POD5 footer length {flen} reaches outside the file")
        if bytes(mv[fstart - 8:fstart]) != FOOTER_MAGIC:
            raise ValueError(f"{path}: no FOOTER magic before the POD5 footer")
        tables = {}
        for offset, length, content_type in _footer_contents(bytes(mv[fstart:fstart + flen]), path):
            if offset < 24 or length < 12 or offset + length > fstart - 8:
                raise ValueError(f"{path}: an embedded table [{offset}, {offset + length}) lies outside the file's body")
            if bytes(mv[offset:offset + 6]) != b"ARROW1" or bytes(mv[offset + length - 6:offset + length]) != b"ARROW1":
                raise ValueError(f"{path}: the embedded table at {offset} is not an Arrow IPC file (no ARROW1)")
            tables.setdefault(content_type, (offset, length))
        opened = {}
        for ct, what, columns in ((SIGNAL_TABLE, "signal", _SIGNAL_COLUMNS), (READS_TABLE, "reads", _READS_COLUMNS),
                                  (RUN_INFO_TABLE, "run info", _RUN_INFO_COLUMNS)):
            if ct not in tables:
                raise ValueError(f"{path}: the POD5 file has no {what} table")
            offset, length = tables[ct]
            try:
                reader = pa.ipc.open_file(self._buf.slice(offset, length))
            except pa.ArrowInvalid as err:
                raise ValueError(f"{path}: the POD5 {what} table does not open: {err}") from err
            _check_columns(what, reader.schema, columns, path)
            opened[ct] = reader
        sig = opened[SIGNAL_TABLE]
        field = sig.schema.field("signal")
        self.vbz = pa.types.is_large_binary(field.type)
        if self.vbz and (field.metadata or {}).get(b"ARROW:extension:name") != b"minknow.vbz":
            raise ValueError(f"{path}: the POD5 signal column is binary but not minknow.vbz")
        self._signal_index = sig.schema.get_field_index("signal")
        self._batches = [sig.get_batch(i) for i in range(sig.num_record_batches)]
        self._batch_start = np.cumsum([0] + [b.num_rows for b in self._batches])
        self.reads = opened[READS_TABLE].read_all()
        self.run_info = opened[RUN_INFO_TABLE].read_all()

    # ------------------------------------------------------------------------------------------------------ metadata
    def run_infos(self):
        """acquisition_id -> dict of the run-info row."""
        t = self.run_info
        start_ms = t.column("acquisition_start_time").cast(pa.timestamp("ms")).cast(pa.int64()).to_pylist()
        out = {}
        for i, acq in enumerate(t.column("acquisition_id").to_pylist()):
            out[acq] = dict(
                acquisition_id=acq, acquisition_start_time=_EPOCH + timedelta(milliseconds=start_ms[i]),
                context_tags=dict(t.column("context_tags")[i].as_py()), tracking_id=dict(t.column("tracking_id")[i].as_py()),
                flow_cell_id=t.column("flow_cell_id")[i].as_py(), sample_id=t.column("sample_id")[i].as_py(),
                sequencer_position=t.column("sequencer_position")[i].as_py(), system_name=t.column("system_name")[i].as_py())
        return out

    def read_groups(self, model):
        """The reference's @RG lines of the run-info table (bonito/pod5.py:95-109)."""
        groups = set()
        for info in self.run_infos().values():
            tracking = info["tracking_id"]
            fields = OrderedDict([
                ("ID", f"{tracking.get('run_id')}_{model}"), ("PL", "ONT"), ("DT", f"{tracking.get('exp_start_time')}"),
                ("PU", f"{info['flow_cell_id']}"), ("PM", f"{info['system_name']}"), ("LB", f"{info['sample_id']}"),
                ("SM", f"{info['sample_id']}"), ("DS", f"run_id={tracking.get('run_id')} basecall_model={model}")])
            groups.add("\t".join(["@RG", *[f"{k}:{v}" for k, v in fields.items()]]))
        return groups

    def read_ids(self):
        return [str(uuid.UUID(bytes=b)) for b in self.reads.column("read_id").to_pylist()]

    def _metadata(self):
        """Per read of the reads table: (read id, signal rows, num_samples, calibration offset and scale, meta dict)."""
        t = self.reads
        infos = self.run_infos()
        run_info = t.column("run_info").combine_chunks()
        acq = run_info.dictionary.to_pylist()
        acq_index = run_info.indices.to_numpy(zero_copy_only=False)
        cols = {k: t.column(k).to_numpy() for k in ("read_number", "start", "num_samples", "channel", "well",
                                                      "calibration_offset", "calibration_scale")}
        rows = t.column("signal").to_pylist()
        for i, rid in enumerate(self.read_ids()):
            a = acq[acq_index[i]]
            if a not in infos:
                raise ValueError(f"{self.path}: read {rid} names run info '{a}', which the run info table lacks")
            info = infos[a]
            try:
                rate = int(info["context_tags"]["sample_frequency"])
            except (KeyError, ValueError) as err:
                raise ValueError(f"{self.path}: run info '{a}' has no sample_frequency context tag") from err
            start = int(cols["start"][i]) / rate
            n = int(cols["num_samples"][i])
            t0 = info["acquisition_start_time"]
            meta = dict(run_id=a, sample_id=info["sample_id"], flow_cell_id=info["flow_cell_id"],
                        device_id=info["sequencer_position"], exp_start_time=t0.isoformat().replace("Z", ""),
                        channel=int(cols["channel"][i]), mux=int(cols["well"][i]), read_number=int(cols["read_number"][i]),
                        sample_rate=rate, start=start, duration=n / rate,
                        start_time=(t0 + timedelta(seconds=start)).astimezone(timezone.utc).isoformat(timespec="milliseconds"))
            yield rid, rows[i], n, float(cols["calibration_offset"][i]), float(cols["calibration_scale"][i]), meta

    # -------------------------------------------------------------------------------------------------------- signal
    def _row(self, r):
        """The signal column of row r: (batch column, index in the batch)."""
        if not 0 <= r < self._batch_start[-1]:
            raise ValueError(f"{self.path}: a read names signal row {r}, the signal table has {self._batch_start[-1]}")
        b = int(np.searchsorted(self._batch_start, r, side="right")) - 1
        return self._batches[b], r - int(self._batch_start[b])

    def _row_samples(self, r):
        batch, i = self._row(r)
        return int(batch.column("samples")[i].as_py())

    def _vbz_bytes(self, r):
        batch, i = self._row(r)
        col = batch.column(self._signal_index)
        offs = np.frombuffer(col.buffers()[1], dtype=np.int64, count=len(col) + 1 + col.offset)[col.offset:]
        return np.frombuffer(col.buffers()[2], dtype=np.uint8, count=int(offs[i + 1]), offset=0)[int(offs[i]):]

    def _decode_rows(self, rows, device, stream):
        """int16 samples of the signal rows `rows` (a list), VBZ rows through one GPU window."""
        if not self.vbz:
            out = []
            for r in rows:
                batch, i = self._row(r)
                v = batch.column(self._signal_index)[i].values.to_numpy(zero_copy_only=False).astype(np.int16)
                if len(v) != self._row_samples(r):
                    raise ValueError(f"{self.path}: signal row {r} holds {len(v)} samples, its samples field says "
                                     f"{self._row_samples(r)}")
                out.append(v)
            return out
        import torch
        from bonito_b200 import native
        blobs = [self._vbz_bytes(r) for r in rows]
        counts = np.array([self._row_samples(r) for r in rows], dtype=np.int64)
        lens = np.array([len(b) for b in blobs], dtype=np.int64)
        caps = (counts + 7) // 8 + 2 * counts
        n = len(rows)
        zmeta = np.empty((n, 4), dtype=np.int64)
        zmeta[:, 0] = np.concatenate([[0], np.cumsum(lens)[:-1]])
        zmeta[:, 1] = lens
        zmeta[:, 2] = np.concatenate([[0], np.cumsum(caps)[:-1]])
        zmeta[:, 3] = caps
        smeta = np.empty((n, 4), dtype=np.int64)
        smeta[:, 0] = zmeta[:, 2]
        smeta[:, 1] = 0
        smeta[:, 2] = counts
        smeta[:, 3] = np.concatenate([[0], np.cumsum(counts)[:-1]])
        host = np.concatenate(blobs) if n else np.empty(0, np.uint8)
        with torch.cuda.stream(stream):
            inp = torch.from_numpy(host).to(device, non_blocking=False)
            meta = torch.from_numpy(np.concatenate([zmeta, smeta])).to(device)
            zm, sm = meta[:n], meta[n:]
            out = torch.empty(int(caps.sum()), dtype=torch.uint8, device=device)
            samples = torch.empty(int(counts.sum()), dtype=torch.int16, device=device)
            out_len = torch.empty(n, dtype=torch.int64, device=device)
            status = torch.empty(2 * n, dtype=torch.int32, device=device)
            native.zstd_decompress(inp, zm, out, out_len, status[:n], stream=stream)
            sm[:, 1] = out_len
            native.svb16_decode(out, sm, samples, status[n:], stream=stream)
            st = status.cpu().numpy()
            host_samples = samples.cpu().numpy()
        for k in range(n):
            if st[k]:
                raise ValueError(f"{self.path}: signal row {rows[k]} does not decompress: zstd status {st[k]} "
                                 f"({native.ZSTD_STATUS.get(int(st[k]), 'unknown')})")
            if st[n + k]:
                raise ValueError(f"{self.path}: signal row {rows[k]} does not decode: svb16 status {st[n + k]} "
                                 f"({native.SVB16_STATUS.get(int(st[n + k]), 'unknown')})")
        return np.split(host_samples, smeta[1:, 3]) if n else []

    def signals(self, read_ids=None, skip=False, device=None, window_rows=WINDOW_ROWS, window_bytes=WINDOW_BYTES):
        """(read id, int16 raw signal, calibration offset, calibration scale, meta) per selected read, in reads-table
        order.  read_ids: a set of UUID strings to keep (or, with skip, to drop)."""
        stream = None
        if self.vbz:
            import torch
            device = torch.device(device if device is not None else "cuda")
            if device.index is None:
                device = torch.device("cuda", torch.cuda.current_device())
            stream = torch.cuda.Stream(device=device)
        pending, nrows, nbytes = [], 0, 0

        def flush():
            rows = [r for p in pending for r in p[1]]
            decoded = self._decode_rows(rows, device, stream)
            k = 0
            for rid, rws, n, off, scale, meta in pending:
                parts = decoded[k:k + len(rws)]
                k += len(rws)
                raw = np.concatenate(parts) if parts else np.empty(0, np.int16)
                if len(raw) != n:
                    raise ValueError(f"{self.path}: read {rid} has {len(raw)} samples in its signal rows, num_samples "
                                     f"says {n}")
                yield rid, raw, off, scale, meta

        for item in self._metadata():
            rid, rows = item[0], item[1]
            if read_ids is not None and ((rid in read_ids) == bool(skip)):
                continue
            pending.append(item)
            nrows += len(rows)
            nbytes += sum(len(self._vbz_bytes(r)) for r in rows) if self.vbz else 0
            if nrows >= window_rows or nbytes >= window_bytes:
                yield from flush()
                pending, nrows, nbytes = [], 0, 0
        if pending:
            yield from flush()


def pa_signal(raw, offset, scale):
    """The reference's pA signal: scale * (raw + offset) in float32 (bonito/pod5.py:57)."""
    return scale * (raw.astype(np.float32) + offset)
