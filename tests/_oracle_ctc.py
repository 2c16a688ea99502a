"""
ORACLE -- TEST INFRASTRUCTURE ONLY.  A functional CPU restatement of the QuartzNet CTC models (bonito/ctc/model.py) and of
the greedy CTC decode, independent of the module classes of `bonito_b200.ctc`:

  * `forward(state, config, x)` -- float64 conv1d / BatchNorm / residual / activation from the config and a state dict;
    `rounding=True` rounds to fp16 where the reference's half model does: every conv output, BatchNorm output, residual
    sum, activation, the logits and the log-probs;
  * `greedy(logp, ...)` -- per-frame argmax (highest index on ties) and the collapse, written as a plain loop;
  * `load_ctc()` -- the reference's own `bonito.ctc.model` module tree, imported through oracle/reference_shim.py with a
    `fast_ctc_decode` stand-in whose functions raise (only the module tree is used).
"""
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F


def _r(x, rounding):
    return x.half().double() if rounding else x


def _act(x, name, rounding):
    if name == "relu":
        return torch.clamp(x, min=0.0)
    return _r(x * torch.sigmoid(x), rounding)


def _bn(x, state, prefix, rounding, eps=1e-3):
    g, b = state[prefix + "weight"].double(), state[prefix + "bias"].double()
    m, v = state[prefix + "running_mean"].double(), state[prefix + "running_var"].double()
    return _r((x - m[None, :, None]) / torch.sqrt(v[None, :, None] + eps) * g[None, :, None] + b[None, :, None], rounding)


def _tcs(x, state, prefix, k, stride, separable, rounding):
    if separable:
        wd = state[prefix + "depthwise.weight"].double()
        x = _r(F.conv1d(x, wd, stride=stride, padding=k // 2, groups=wd.shape[0]), rounding)
        return _r(F.conv1d(x, state[prefix + "pointwise.weight"].double()), rounding)
    return _r(F.conv1d(x, state[prefix + "conv.weight"].double(), stride=stride, padding=k // 2), rounding)


def forward(state, config, x, rounding=False, eps=1e-3, return_blocks=False):
    """x [N, 1, L] -> log-probs [N, T, 5] float64 (batch-first); `return_blocks`: also the per-block outputs."""
    act = config["encoder"]["activation"]
    h = _r(x.double(), rounding)
    outs = []
    for i, blk in enumerate(config["block"]):
        pre = f"encoder.encoder.{i}."
        k, s, sep, R = blk["kernel"][0], blk["stride"][0], blk["separable"], blk["repeat"]
        y = h
        for r in range(R):
            y = _tcs(y, state, f"{pre}conv.{4 * r}.", k, s, sep, rounding)
            y = _bn(y, state, f"{pre}conv.{4 * r + 1}.", rounding, eps)
            if r < R - 1:
                y = _act(y, act, rounding)
        if blk["residual"]:
            res = _r(F.conv1d(h, state[pre + "residual.0.conv.weight"].double()), rounding)
            y = _r(y + _bn(res, state, pre + "residual.1.", rounding, eps), rounding)
        h = _act(y, act, rounding)
        outs.append(h)
    logits = _r(F.conv1d(h, state["decoder.layers.0.weight"].double(), state["decoder.layers.0.bias"].double()), rounding)
    logp = _r(torch.log_softmax(logits, dim=1), rounding).permute(0, 2, 1)
    return (logp, outs) if return_blocks else logp


def greedy(logp, alphabet="NACGT", qscale=1.0, qbias=0.0):
    """[T, 5] log-probs of one read -> (sequence str, qstring str, moves uint8 [T]), by a frame-by-frame loop."""
    logp = np.asarray(logp, dtype=np.float32)
    seq, qual, moves = [], [], np.zeros(len(logp), dtype=np.uint8)
    prev, run = 0, None
    for t, row in enumerate(logp):
        lab = max(i for i in range(len(row)) if row[i] == row.max())
        p = float(np.exp(np.float32(row[lab])))
        if lab != 0 and lab != prev:
            if run is not None:
                qual.append(run)
            seq.append(alphabet[lab])
            moves[t] = 1
            run = [p]
        elif lab != 0 and run is not None:
            run.append(p)
        prev = lab
    if run is not None:
        qual.append(run)

    def phred(ps):
        q = np.rint(-10 * np.log10(max(1 - float(np.mean(np.asarray(ps, dtype=np.float64))), 1e-4)) * qscale + qbias) + 33
        return chr(int(np.clip(q, 33, 126)))
    return "".join(seq), "".join(phred(r) for r in qual), moves


def load_ctc():
    """The reference's bonito.ctc.model module (module tree only; its decoders are stubs that raise)."""
    from oracle import reference_shim
    reference_shim.load()

    def _absent(*args, **kwargs):
        raise RuntimeError("fast_ctc_decode is not available; only the reference module tree is used")
    if "fast_ctc_decode" not in sys.modules:
        mod = types.ModuleType("fast_ctc_decode")
        mod.beam_search, mod.viterbi_search = _absent, _absent
        sys.modules["fast_ctc_decode"] = mod
    import importlib
    return importlib.import_module("bonito.ctc.model")
