"""
Read ingestion for `bonito_b200 basecaller`.

The reference picks a pod5 or fast5 reader by globbing the reads directory (`bonito/reader.py:23-48`).  Supported
inputs:
  * `*.pod5`  read by bonito_b200.pod5 without the pod5 package: the container parsed on the host, the VBZ signal rows
              decompressed on the GPU, signal in pA = scale * (raw + offset), the reference's metadata and @RG lines;
              reads in reads-table order, `read_ids` / `skip` matched against the read UUID strings;
  * `*.npy`   one read per file: a 1-D array of picoampere samples, read id = file stem (what the tests and the
              synthetic benchmarks use); no metadata and no read groups.
fast5 input is not supported.
Trimming and normalisation follow `bonito/reader.py:122-166` (trim of the leading stall, pA standardisation or
quantile scaling).
"""

import os
from glob import glob

import numpy as np

__default_norm_params__ = {"quantile_a": 0.2, "quantile_b": 0.9, "shift_multiplier": 0.51, "scale_multiplier": 0.53}


def trim(signal, window_size=40, threshold=2.4, min_trim=10, min_elements=3, max_samples=8000, max_trim=0.3):
    """Number of leading samples to drop: end of the first run of windows with > min_elements samples above threshold."""
    limit = min(max_samples, len(signal))
    seen_peak = False
    for pos in range(limit // window_size):
        start = pos * window_size + min_trim
        end = start + window_size
        window = signal[start:end]
        if seen_peak or np.count_nonzero(window > threshold) > min_elements:
            seen_peak = True
            if window[-1] > threshold:
                continue
            if end >= limit or end / len(signal) > max_trim:
                return min_trim
            return end
    return min_trim


def normalisation(sig, scaling_strategy=None, norm_params=None):
    """(shift, scale) for `(sig - shift) / scale`: pA standardisation from the config, else quantile scaling."""
    strategy = scaling_strategy.get("strategy") if scaling_strategy else None
    if strategy == "pa":
        if norm_params and norm_params.get("standardise") == 1:
            return norm_params.get("mean"), norm_params.get("stdev")
        if norm_params and norm_params.get("standardise") == 0:
            return 0.0, 1.0
        raise ValueError("Picoampere scaling requested, but standardisation flag not provided")
    if strategy in (None, "quantile"):
        p = norm_params or __default_norm_params__
        qa, qb = np.quantile(sig, [p["quantile_a"], p["quantile_b"]])
        return max(10, p["shift_multiplier"] * (qa + qb)), max(1.0, p["scale_multiplier"] * (qb - qa))
    raise ValueError(f"Scaling strategy {strategy} not supported; choose quantile or pa.")


class Read:
    """What `basecall()` needs (`read_id`, float32 `signal`) plus the bookkeeping the writers use."""

    def __init__(self, read_id, pa_signal, filename="", do_trim=True, scaling_strategy=None, norm_params=None, meta=None):
        meta = meta or {}
        self.read_id, self.filename = str(read_id), filename
        pa = np.asarray(pa_signal, dtype=np.float32)
        self.num_samples = len(pa)
        self.shift, self.scale = normalisation(pa, scaling_strategy, norm_params)
        self.trimmed_samples = trim(pa, threshold=self.scale * 2.4 + self.shift) if do_trim else 0
        self.template_start = self.trimmed_samples
        if "sample_rate" in meta:  # POD5: positions in seconds (bonito/pod5.py:44-65)
            self.sample_rate, self.start = meta["sample_rate"], meta["start"]
            self.template_start = self.start + self.trimmed_samples / self.sample_rate
            self.template_duration = meta["duration"] - self.trimmed_samples / self.sample_rate
        self.signal = ((pa[self.trimmed_samples:] - self.shift) / self.scale).astype(np.float32)
        self.scaling_strategy = (scaling_strategy or {}).get("strategy") or "quantile"
        # acquisition metadata the SAM tags carry (bonito/reader.py:59-87); .npy reads have none
        self.run_id, self.mux, self.channel, self.read_number = meta.get("run_id", "unknown"), meta.get("mux", 0), \
            meta.get("channel", 0), meta.get("read_number", 0)
        self.start_time, self.duration = meta.get("start_time", ""), meta.get("duration", self.num_samples / 5000.0)
        self.flow_cell_id, self.device_id, self.sample_id, self.exp_start_time = (
            meta.get(k, "") for k in ("flow_cell_id", "device_id", "sample_id", "exp_start_time"))

    def readgroup(self, model):
        """@RG header line (reference: bonito/reader.py:59-73)."""
        fields = [("ID", f"{self.run_id}_{model}"), ("PL", "ONT"), ("DT", self.exp_start_time), ("PU", self.flow_cell_id),
                  ("PM", self.device_id), ("LB", self.sample_id), ("SM", self.sample_id),
                  ("DS", f"run_id={self.run_id} basecall_model={model}")]
        return "\t".join(["@RG", *[f"{k}:{v}" for k, v in fields]])

    def tagdata(self):
        """Per-read SAM tags (reference: bonito/reader.py:75-86)."""
        return [f"mx:i:{self.mux}", f"ch:i:{self.channel}", f"st:Z:{self.start_time}", f"du:f:{self.duration}",
                f"rn:i:{self.read_number}", f"f5:Z:{self.filename}", f"sm:f:{self.shift}", f"sd:f:{self.scale}",
                f"sv:Z:{self.scaling_strategy}"]


class ReadChunk:
    """One fixed-size window of a read, basecalled as a read of its own for `basecaller --save-ctc` (reference:
    bonito/reader.py:89-104): named `<read_id>:<i>:<n>`, with the parent's metadata and `template_start` /
    `template_duration` set to the parent's start time and duration."""

    def __init__(self, read, chunk, i, n):
        self.read_id = f"{read.read_id}:{i}:{n}"
        self.filename, self.run_id, self.mux, self.channel = read.filename, read.run_id, read.mux, read.channel
        self.read_number, self.shift, self.scale = read.read_number, read.shift, read.scale
        self.scaling_strategy = read.scaling_strategy
        self.start, self.duration = read.start_time, read.duration
        self.template_start, self.template_duration = self.start, self.duration
        self.signal = chunk

    def __repr__(self):
        return f"ReadChunk('{self.read_id}')"


def read_chunks(read, chunksize=4000, overlap=400):
    """
    The read's (already trimmed and normalised) signal cut into `chunksize` windows `chunksize - overlap` apart, as
    ReadChunks (reference: bonito/reader.py:107-119).  A read shorter than a chunk gives none; otherwise the first
    `(len - chunksize) % (chunksize - overlap)` samples are dropped, so the last window ends at the read's end.
    """
    length = len(read.signal)
    if length < chunksize:
        return
    step = chunksize - overlap
    offset = (length - chunksize) % step
    n = (length - offset - chunksize) // step + 1
    for i in range(n):
        start = offset + i * step
        yield ReadChunk(read, read.signal[start:start + chunksize], i + 1, n)


class Reader:
    """The reads of a directory: `*.pod5` files if there are any, else `*.npy` files.  Every POD5 file's container is
    checked here, so a malformed one is refused (ValueError naming it) before any CUDA use."""

    def __init__(self, directory, recursive=False):
        self.fmt = None
        for fmt in ("pod5", "npy"):
            pattern = f"**/*.{fmt}" if recursive else f"*.{fmt}"
            if glob(os.path.join(directory, pattern), recursive=True):
                self.fmt = fmt
                break
        if self.fmt is None:
            raise FileNotFoundError(directory)
        if self.fmt == "pod5":
            from bonito_b200.pod5 import Pod5File
            for path in self._paths(directory, recursive):
                Pod5File(path)

    def _paths(self, directory, recursive):
        pattern = f"**/*.{self.fmt}" if recursive else f"*.{self.fmt}"
        return sorted(glob(os.path.join(directory, pattern), recursive=True))

    def get_reads(self, directory, recursive=False, read_ids=None, skip=False, do_trim=True, scaling_strategy=None,
                  norm_params=None, device=None, **_ignored):
        for path in self._paths(directory, recursive):
            if self.fmt == "npy":
                read_id = os.path.splitext(os.path.basename(path))[0]
                if read_ids is not None and ((read_id in read_ids) == bool(skip)):
                    continue
                yield Read(read_id, np.load(path), filename=os.path.basename(path), do_trim=do_trim,
                           scaling_strategy=scaling_strategy, norm_params=norm_params)
                continue
            from bonito_b200.pod5 import Pod5File, pa_signal
            for read_id, raw, offset, scale, meta in Pod5File(path).signals(read_ids, skip, device=device):
                yield Read(read_id, pa_signal(raw, offset, scale), filename=os.path.basename(path), do_trim=do_trim,
                           scaling_strategy=scaling_strategy, norm_params=norm_params, meta=meta)

    def get_read_groups(self, directory, model, recursive=False, **_ignored):
        """The reference's @RG header lines of every POD5 file's run info (bonito/pod5.py:84-110), sorted; none for
        `.npy` input."""
        if self.fmt != "pod5":
            return []
        from bonito_b200.pod5 import Pod5File
        groups = set()
        for path in self._paths(directory, recursive):
            groups |= Pod5File(path).read_groups(model)
        return sorted(groups)
