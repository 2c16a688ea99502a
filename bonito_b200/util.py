"""
Host-side helpers of the chunked basecalling path: chunk / stitch / batchify /
unbatchify and the model loader.  Semantics follow the reference bit for bit
(`bonito/util.py:142-311`); the tests in `tests/test_host_logic.py`
replay the known answers recorded in SURVEY.md Appendix A and the golden
fixtures generated from the reference's own functions.
"""

import os
import re
import random
from glob import glob
from itertools import groupby
from importlib import import_module
from collections import OrderedDict
from pathlib import Path

import numpy as np
import torch

try:
    import toml as _toml

    def _load_toml(path):
        return _toml.load(path)
except ImportError:  # pragma: no cover - python >= 3.11 always has tomllib
    import tomllib

    def _load_toml(path):
        with open(path, "rb") as fh:
            return tomllib.load(fh)

__dir__ = Path(__file__).parent
__models_dir__ = __dir__ / "models"

# model packages named in reference configs resolve to their native counterparts
_PACKAGE_ALIASES = {
    "bonito.crf": "bonito_b200.crf",
    "bonito.transformer": "bonito_b200.transformer",
    "bonito.ctc": "bonito_b200.ctc",
}


def init(seed, device, deterministic=True):
    """Seed python / numpy / torch (reference: bonito/util.py:40-53)."""
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    if str(device) == "cpu":
        return
    assert torch.cuda.is_available()


# ---------------------------------------------------------------------------
# type-agnostic container helpers (reference: bonito/util.py:66-102)
# ---------------------------------------------------------------------------

def concat(xs, dim=0):
    head = xs[0]
    if isinstance(head, torch.Tensor):
        return torch.cat(xs, dim=dim)
    if isinstance(head, np.ndarray):
        return np.concatenate(xs, axis=dim)
    if isinstance(head, list):
        return [item for x in xs for item in x]
    if isinstance(head, str):
        return "".join(xs)
    if isinstance(head, dict):
        return {k: concat([x[k] for x in xs], dim) for k in head}
    raise TypeError(type(head))


def select_range(x, start, end, dim=0):
    if isinstance(x, dict):
        return {k: select_range(v, start, end, dim) for k, v in x.items()}
    if dim == 0 or isinstance(x, list):
        return x[start:end]
    return x[(slice(None),) * dim + (slice(start, end),)]


def size(x, dim=0):
    if hasattr(x, "shape"):
        return x.shape[dim]
    if dim == 0:
        return len(x)
    raise TypeError(type(x))


def phred(prob, scale=1.0, bias=0.0):
    """ASCII phred char for `prob` (reference: bonito/util.py:105-112)."""
    err = max(1 - prob, 1e-4)
    q = -10 * np.log10(err) * scale + bias
    return chr(int(np.round(q) + 33))


def mean_qscore_from_qstring(qstring):
    if len(qstring) == 0:
        return 0.0
    qs = np.frombuffer(qstring.encode(), dtype=np.uint8).astype(np.float64) - 33
    mean_err = np.exp(qs * (-np.log(10) / 10.0)).mean()
    return -10 * np.log10(max(mean_err, 1e-4))


# ---------------------------------------------------------------------------
# chunk / stitch (reference: bonito/util.py:142-183)
# ---------------------------------------------------------------------------

def chunk(signal, chunksize, overlap):
    """
    Cut one read into overlapping windows -> [n_chunks, 1, chunksize].

    Reads shorter than a chunk are tiled up to `chunksize`; when the windows do
    not tile the read exactly a leading chunk over signal[:chunksize] is added.
    """
    if signal.is_cuda and chunksize > 0 and signal.numel() == signal.shape[-1] and signal.dtype in (torch.float16, torch.float32):
        # a read that is already on the device: one native gather (+ fp16 conversion) instead of unfold / cat / half()
        from bonito_b200 import native
        return native.chunk_signal(signal.contiguous(), chunksize, overlap)
    if signal.ndim == 1:
        signal = signal.unsqueeze(0)
    length = signal.shape[-1]
    if chunksize == 0:
        return signal[None, :]
    if length < chunksize:
        reps, rest = divmod(chunksize, length)
        tiled = torch.cat([signal.repeat(1, reps), signal[..., :rest]], dim=-1)
        return tiled[None, :]
    step = chunksize - overlap
    stub = (length - overlap) % step
    windows = signal[..., stub:].unfold(-1, chunksize, step).movedim(-2, 0)
    if stub > 0:
        windows = torch.cat([signal[None, ..., :chunksize], windows], dim=0)
    return windows


def stitch(chunks, chunksize, overlap, length, stride, reverse=False):
    """Drop half of each overlap at chunk joins and concatenate along time."""
    if chunks.shape[0] == 1:
        return chunks.squeeze(0)
    half = overlap // 2
    lo, hi = half // stride, (chunksize - half) // stride
    stub = (length - overlap) % (chunksize - overlap)
    first_hi = (stub + half) // stride if stub > 0 else hi
    if reverse:
        parts = list(chunks)
        return concat([parts[-1][:-lo], *(x[-hi:-lo] for x in reversed(parts[1:-1])), parts[0][-first_hi:]])
    return concat([chunks[0, :first_hi], *chunks[1:-1, lo:hi], chunks[-1, lo:]])


# ---------------------------------------------------------------------------
# batchify / unbatchify (reference: bonito/util.py:186-220)
# ---------------------------------------------------------------------------

def batchify(items, batchsize, dim=0):
    """
    Regroup (key, value) items into batches of exactly `batchsize` rows (the
    final batch may be short).  Yields (keys, batch) where every key is
    (item_key, (row_start, row_end)) locating that item's rows in the batch.
    """
    pending, fill = [], 0
    for key, value in items:
        total = size(value, dim)
        cuts = list(range(batchsize - fill, total, batchsize))
        for lo, hi in zip([0] + cuts, cuts + [total]):
            rows = hi - lo
            pending.append(((key, (fill, fill + rows)), select_range(value, lo, hi, dim)))
            fill += rows
            if fill == batchsize:
                keys, vals = zip(*pending)
                yield keys, concat(vals, dim)
                pending, fill = [], 0
    if pending:
        keys, vals = zip(*pending)
        yield keys, concat(vals, dim)


def unbatchify(batches, dim=0):
    """Inverse of `batchify`: regroup batch rows by consecutive equal key."""
    pieces = (
        (key, select_range(value, lo, hi, dim))
        for keys, value in batches
        for key, (lo, hi) in keys
    )
    return (
        (key, concat([v for _, v in group], dim))
        for key, group in groupby(pieces, key=lambda kv: kv[0])
    )


# ---------------------------------------------------------------------------
# model loading (reference: bonito/util.py:223-311)
# ---------------------------------------------------------------------------

def _resolve_model_dir(name):
    if not os.path.isdir(name) and os.path.isdir(os.path.join(__models_dir__, name)):
        return os.path.join(__models_dir__, name)
    return name


def load_symbol(config, symbol):
    """Import `config['model']['package']` and return its attribute `symbol`."""
    if not isinstance(config, dict):
        config = _load_toml(os.path.join(_resolve_model_dir(config), "config.toml"))
    package = config["model"]["package"]
    module = import_module(_PACKAGE_ALIASES.get(package, package))
    return getattr(module, symbol)


def match_names(state_dict, model):
    """Map checkpoint keys to model keys by sorted (shape, position)."""
    def ordered(sd):
        triples = sorted((tuple(v.shape), i, k) for i, (k, v) in enumerate(sd.items()))
        return [k for _, _, k in triples], [s for s, _, _ in triples]

    ckpt_keys, ckpt_shapes = ordered(state_dict)
    model_keys, model_shapes = ordered(model.state_dict())
    assert ckpt_shapes == model_shapes
    remap = dict(zip(ckpt_keys, model_keys))
    return OrderedDict((k, remap[k]) for k in state_dict.keys())


def get_last_checkpoint(dirname):
    found = glob(os.path.join(dirname, "weights_*.tar"))
    if not found:
        raise FileNotFoundError("no model weights found in '%s'" % dirname)
    newest = max(int(re.sub(r".*_([0-9]+).tar", r"\1", w)) for w in found)
    return os.path.join(dirname, "weights_%s.tar" % newest)


def set_config_defaults(config, chunksize=None, batchsize=None, overlap=None, quantize=False):
    """CLI value > [basecaller] table > 4000/500/64 (reference: bonito/util.py:259-268)."""
    params = config.get("basecaller", {})
    params["chunksize"] = chunksize or params.get("chunksize", 4000)
    params["overlap"] = overlap if overlap is not None else params.get("overlap", 500)
    params["batchsize"] = batchsize or params.get("batchsize", 64)
    params["quantize"] = params.get("quantize") if quantize is None else quantize
    config["basecaller"] = params
    return config


def load_model(dirname, device, weights=None, half=True, chunksize=None, batchsize=None,
               overlap=None, quantize=False, use_koi=False):
    """Load `config.toml` + `weights_N.tar` from a model directory."""
    dirname = _resolve_model_dir(dirname)
    weights = get_last_checkpoint(dirname) if weights is None else os.path.join(dirname, "weights_%s.tar" % weights)
    config = set_config_defaults(_load_toml(os.path.join(dirname, "config.toml")),
                                 chunksize, batchsize, overlap, quantize)
    return _load_model(weights, config, device, half, use_koi)


def _load_model(model_file, config, device, half=True, use_koi=False):
    device = torch.device(device)
    model = load_symbol(config, "Model")(config)

    if use_koi:
        params = config["basecaller"]
        params["chunksize"] -= params["chunksize"] % model.stride
        # overlap must be an even multiple of the stride for stitching to line up
        params["overlap"] -= params["overlap"] % (model.stride * 2)
        model.use_koi(batchsize=params["batchsize"], chunksize=params["chunksize"], quantize=params["quantize"])

    state = torch.load(model_file, map_location=device)
    state = {new: state[old] for old, new in match_names(state, model).items()}
    model.load_state_dict(OrderedDict((k.replace("module.", ""), v) for k, v in state.items()))

    if half:
        model = model.half()
    model.eval()
    model.to(device)
    return model
