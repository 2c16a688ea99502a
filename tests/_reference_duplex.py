"""
The reference's own `bonito/cli/duplex.py`, importable on a CPU box without its aligners: `load_duplex()` installs
stand-ins for the absent third-party modules and returns the module, whose `call_basespace_duplex` then runs unchanged.

  pysam     only the CIGAR op constants (C* = 0..8, the htslib codes)
  mappy     revcomp
  edlib     align(query, target, task="path") -> {"editDistance", "cigar"}: the GLOBAL_EDIT oracle's ops as an extended
            CIGAR string (=, X, I, D)
  parasail  sg_trace_scan_32(query, target, 10, 2, dnafull).cigar.decode -> bytes: the SEMIGLOBAL_AFFINE oracle's ops,
            covering both sequences (leading / trailing gaps included)

Only usable where the reference checkout exists (`available()`); nothing on the GPU path imports this.
"""

import importlib
import sys
import types

import _oracle_duplex as O
from oracle import reference_shim

available = reference_shim.available


def cigar(ops):
    out, prev, n = [], None, 0
    for op in ops:
        if op == prev:
            n += 1
            continue
        if prev is not None:
            out.append(f"{n}{prev}")
        prev, n = op, 1
    if prev is not None:
        out.append(f"{n}{prev}")
    return "".join(out)


def _edlib_align(query, target, task="path", **kw):
    dist, ops = O.global_edit(query, target)
    return {"editDistance": dist, "cigar": cigar(ops)}


def _sg_trace_scan_32(query, target, open_, extend, matrix):
    assert (open_, extend) == (10, 2)
    score, ops = O.semiglobal_affine(query, target)
    return types.SimpleNamespace(score=score, cigar=types.SimpleNamespace(decode=cigar(ops).encode()))


def _revcomp(seq):
    return seq.translate(str.maketrans("ACGTacgt", "TGCAtgca"))[::-1]


def _module(name, **attrs):
    mod = sys.modules.get(name) or types.ModuleType(name)
    mod.__dict__.update(attrs)
    sys.modules[name] = mod
    return mod


def load_duplex():
    if "bonito.cli.duplex" in sys.modules:
        return sys.modules["bonito.cli.duplex"]
    reference_shim.load()
    ops = dict(CMATCH=0, CINS=1, CDEL=2, CREF_SKIP=3, CSOFT_CLIP=4, CHARD_CLIP=5, CPAD=6, CEQUAL=7, CDIFF=8)
    _module("pysam", **ops)
    _module("mappy", revcomp=_revcomp)
    _module("edlib", align=_edlib_align)
    _module("parasail", dnafull=object(), sg_trace_scan_32=_sg_trace_scan_32)
    # the command's I/O and minimap2 plumbing is not exercised: stand-ins for the names it imports
    _module("bonito.io", DuplexWriter=None, biofmt=None)
    _module("bonito.aligner", align_map=None, Aligner=None)
    _module("bonito.multiprocessing", ProcessMap=None)
    if not hasattr(sys.modules["bonito.util"], "tqdm_environ"):
        sys.modules["bonito.util"].tqdm_environ = dict
    return importlib.import_module("bonito.cli.duplex")
