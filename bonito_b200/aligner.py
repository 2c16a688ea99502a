"""
Read-to-reference mapping on the GPU for `basecaller --reference` (the reference maps with minimap2 through mappy,
bonito/aligner.py).  minimap2's heuristics are not reproducible here, so the rules are this project's, stated in
bonito_b200/csrc/map.cu and restated by the CPU oracle tests/_oracle_map.py:

- minimizers of canonical k-mers (minimap2's hash64), the smallest hash of each window of w k-mers, ties to the leftmost;
- an index of the reference minimizers sorted by hash, where a hash seen more than MAX_OCC times is never a seed;
- anchors, a chaining DP over the 50 previous anchors of the same strand and contig, a greedy chain extraction;
- a local affine alignment (match +2, mismatch -4, N -1, a gap of g bases 4 + 2 g) in a band around the primary chain.

`Aligner(fasta, preset)` builds the index once on the device; `map_batch(sequences)` maps many reads in one pass of
launches and returns one `Mapping` (mappy's attribute names) or None per read.  Only the primary alignment is reported.
"""

import gzip
import math
import queue
from dataclasses import dataclass
from threading import Thread

import numpy as np
import torch

from bonito_b200 import native
from bonito_b200.align import _budget_groups

PRESETS = {"lr:hq": (19, 19), "map-ont": (15, 10)}   # preset -> (k, w)
MAX_OCC = 500                    # a hash with more reference entries than this is never a seed
MAX_BAND = 2048                  # band half-width cap: 64 + the largest diagonal change between chain anchors
MIN_ANCHORS, MIN_SCORE = 3, 40   # a primary chain below either is reported unmapped
MAX_READ = 500_000               # the alignment's end-cell key holds the score in 20 bits: longer reads are not mapped
MAX_WINDOW = (1 << 22) - 1       # ... and the target column in 22 bits
TRACE_BUDGET = 2 << 30           # traceback bytes per alignment launch (a read of MAX_READ bases at MAX_BAND needs 1.1 GB)
BATCH_READS, BATCH_BASES = 2048, 16 << 20   # align_map batches

_ACGT = np.zeros(256, dtype=bool)
_ACGT[np.frombuffer(b"ACGT", dtype=np.uint8)] = True
_COMP = np.arange(256, dtype=np.uint8)
_COMP[np.frombuffer(b"ACGT", dtype=np.uint8)] = np.frombuffer(b"TGCA", dtype=np.uint8)


class IndexBuildError(ValueError):
    """The reference cannot be read as FASTA (or FASTA.gz) with at least one base."""


@dataclass(frozen=True)
class Mapping:
    """The primary alignment of a read, with mappy's attribute names.  r_st / r_en are 0-based contig coordinates; q_st /
    q_en are in the read's own orientation; strand is +1 or -1; cigar_str has M / I / D only (clips are the caller's)."""
    ctg: str
    r_st: int
    r_en: int
    q_st: int
    q_en: int
    strand: int
    mapq: int
    cigar_str: str
    NM: int
    MD: str


def read_fasta(path):
    """[(name, upper-case bytes)] of a FASTA or gzipped FASTA file; a contig's name is the first word of its header and
    every byte other than A C G T becomes N.  Records without bases are dropped."""
    if str(path).endswith(".mmi"):
        raise IndexBuildError(f"{path}: .mmi indexes are not supported, give the FASTA")
    try:
        with open(path, "rb") as fh:
            data = fh.read()
        if data[:2] == b"\x1f\x8b":
            data = gzip.decompress(data)
    except (OSError, EOFError) as err:
        raise IndexBuildError(f"{path}: {err}") from err
    if not data.lstrip().startswith(b">"):
        raise IndexBuildError(f"{path}: not FASTA")
    contigs = []
    for record in data.split(b"\n>"):
        header, _, body = record.lstrip(b">").partition(b"\n")
        words = header.split()
        seq = np.frombuffer(b"".join(body.split()).upper(), dtype=np.uint8).copy()
        if not words or not seq.size:
            continue
        seq[~_ACGT[seq]] = ord("N")
        contigs.append((words[0].decode(errors="replace"), seq))
    if not contigs:
        raise IndexBuildError(f"{path}: no sequence")
    if sum(s.size for _, s in contigs) >= 1 << 32:
        raise IndexBuildError(f"{path}: the reference must have fewer than 2^32 bases")
    return contigs


def revcomp(seq):
    """Reverse complement of a str (A C G T complemented, any other byte kept)."""
    return _COMP[np.frombuffer(seq.encode(), dtype=np.uint8)[::-1]].tobytes().decode()


def mapq(f1, f2, n):
    """minimap2's formula on the integer chain scores, in float64."""
    if f2 >= f1:
        return 0
    return min(60, int(math.floor(40 * (1 - f2 / f1) * min(1.0, n / 10) * math.log(f1))))


def cigar_nm_md(ops, ref):
    """(CIGAR with M / I / D, NM, MD) of an op string (uint8 '=' 'X' 'I' 'D') against the reference bases it covers.  numpy
    per op; Python only per CIGAR run and per MD mismatch / deletion run."""
    ops = np.asarray(ops, dtype=np.uint8)
    if not ops.size:
        return "", 0, "0"
    code = np.where(ops == ord("I"), 1, np.where(ops == ord("D"), 2, 0))
    starts = np.concatenate(([0], np.flatnonzero(np.diff(code)) + 1))
    runs = np.diff(np.concatenate((starts, [ops.size])))
    cigar = "".join(f"{n}{'MID'[c]}" for n, c in zip(runs.tolist(), code[starts].tolist()))
    nm = int(np.count_nonzero(ops != ord("=")))
    o = ops[ops != ord("I")]                         # each of these consumes ref[index]
    isd = o == ord("D")
    prev_d = np.concatenate(([False], isd[:-1]))
    ev = np.flatnonzero((o == ord("X")) | (isd & ~prev_d))
    eq = np.concatenate(([0], np.cumsum(o == ord("="))))
    d_end = np.flatnonzero(isd & ~np.concatenate((isd[1:], [False]))) + 1
    counts = np.diff(np.concatenate(([0], eq[ev]))).tolist()
    ref = np.asarray(ref, dtype=np.uint8)
    parts, di = [], 0
    for c, p in zip(counts, ev.tolist()):
        if isd[p]:
            parts.append(f"{c}^{ref[p:d_end[di]].tobytes().decode()}")
            di += 1
        else:
            parts.append(f"{c}{chr(ref[p])}")
    parts.append(str(int(eq[-1] - (eq[ev[-1]] if ev.size else 0))))
    return cigar, nm, "".join(parts)


def _to_device(array, device):
    return torch.from_numpy(np.require(array, requirements=["C", "W"])).pin_memory().to(device, non_blocking=True)


class Aligner:
    """The index of one reference on one device; `seq_names`, `seq(name)`, `map_batch(sequences)`."""

    def __init__(self, fasta, preset="lr:hq", device="cuda"):
        if preset not in PRESETS:
            raise ValueError(f"unknown preset {preset!r}: choose one of {', '.join(PRESETS)}")
        self.k, self.w = PRESETS[preset]
        contigs = read_fasta(fasta)
        self.seq_names = [name for name, _ in contigs]
        self.lengths = [int(s.size) for _, s in contigs]
        self._host = np.concatenate([s for _, s in contigs])
        self._ctg_off = np.concatenate(([0], np.cumsum(self.lengths))).astype(np.int64)
        self._by_name = {name: c for c, name in enumerate(self.seq_names)}
        self.device = torch.device(device)
        native.require()
        with torch.cuda.device(self.device):
            self.ref = _to_device(self._host, self.device)
            self.ctg_off = _to_device(self._ctg_off, self.device)
            mm = self._minimizers(self.ref, self.ctg_off)
            pos = torch.nonzero(mm >= 0).squeeze(1)
            keys = mm[pos]
            hashes, order = torch.sort(keys >> 1, stable=True)     # (hash, position): pos is ascending
            self.idx_val = ((pos << 1) | (keys & 1))[order].contiguous()
            self.idx_hash, counts = torch.unique_consecutive(hashes, return_counts=True)
            self.idx_start = torch.zeros(self.idx_hash.numel() + 1, dtype=torch.int64, device=self.device)
            torch.cumsum(counts, 0, out=self.idx_start[1:])
            del mm, pos, keys, hashes, order, counts
            torch.cuda.current_stream().synchronize()

    @property
    def contigs(self):
        return list(zip(self.seq_names, self.lengths))

    def seq(self, name, start=0, end=None):
        c = self._by_name.get(name)
        if c is None:
            return None
        return self._host[self._ctg_off[c]:self._ctg_off[c + 1]][start:end].tobytes().decode()

    def _minimizers(self, seq, seq_off):
        kmer = torch.empty(seq.numel(), dtype=torch.int64, device=seq.device)
        mm = torch.empty_like(kmer)
        native.map_minimizers(seq, seq_off, self.k, self.w, kmer, mm)
        return mm

    def chains(self, sequences):
        """Device stages up to chain extraction -> (per-read int64 [n, 9] of n, f1, f2, strand, W, q0, r0, q1, r1 (global r),
        device chain pairs, device read anchor offsets, host read lengths); also kept for the tests."""
        raw = [s.encode() if isinstance(s, str) else bytes(s) for s in sequences]
        lens = np.array([len(s) if len(s) <= MAX_READ else 0 for s in raw], dtype=np.int64)
        n = len(raw)
        off = np.zeros(n + 1, dtype=np.int64)
        np.cumsum(lens, out=off[1:])
        data = np.frombuffer(b"".join(s.upper() for s, m in zip(raw, lens) if m), dtype=np.uint8)
        empty = np.zeros((n, 9), dtype=np.int64), None, None, lens
        if not data.size:
            return empty
        dev = self.device
        seq, seq_off = _to_device(data, dev), _to_device(off, dev)
        mm = self._minimizers(seq, seq_off)
        count = torch.empty(mm.numel(), dtype=torch.int32, device=dev)
        native.map_anchors(mm, seq_off, self.k, self.idx_hash, self.idx_start, self.idx_val, MAX_OCC, count=count)
        csum = torch.zeros(mm.numel() + 1, dtype=torch.int64, device=dev)
        torch.cumsum(count, 0, out=csum[1:])
        read_aoff = csum[seq_off].contiguous()
        n_anchors = int(csum[-1])
        if not n_anchors:
            return empty
        akey = torch.empty(n_anchors, dtype=torch.int64, device=dev)
        aq = torch.empty(n_anchors, dtype=torch.int32, device=dev)
        native.map_anchors(mm, seq_off, self.k, self.idx_hash, self.idx_start, self.idx_val, MAX_OCC, aoff=csum[:-1],
                           akey=akey, aq=aq)
        akey, perm = torch.sort(akey, stable=True)
        aq = aq[perm].contiguous()
        f = torch.empty(n_anchors, dtype=torch.int32, device=dev)
        pred = torch.empty_like(f)
        native.map_chain(akey, aq, read_aoff, self.ctg_off, self.k, f, pred)
        _, order = torch.sort(((akey >> 33) << 32) | (0x7FFFFFFF - f.long()), stable=True)
        taken = torch.zeros(n_anchors, dtype=torch.uint8, device=dev)
        chain = torch.empty(n_anchors, 2, dtype=torch.int64, device=dev)
        out = torch.empty(n, 9, dtype=torch.int64, device=dev)
        native.map_extract(akey, aq, f, pred, order, read_aoff, seq_off, self.k, MAX_BAND, taken, chain, out)
        return out.cpu().numpy(), chain, read_aoff.cpu().numpy(), lens

    def plan(self, res, lens):
        """Host plan of the alignments: per mapped read (index, strand, contig, window start, window length, W)."""
        idx = np.flatnonzero((res[:, 0] >= MIN_ANCHORS) & (res[:, 1] >= MIN_SCORE))
        W, q0, r0, q1, r1 = (res[idx, c] for c in (4, 5, 6, 7, 8))
        ctg = np.searchsorted(self._ctg_off, r0, side="right") - 1
        cs, ce = self._ctg_off[ctg], self._ctg_off[ctg + 1]
        ts = np.maximum(cs, r0 - q0 - W)
        te = np.minimum(ce, r1 + (lens[idx] - q1) + W)
        keep = te - ts <= MAX_WINDOW
        return idx[keep], res[idx[keep], 3], ctg[keep], ts[keep], (te - ts)[keep], W[keep]

    def map_batch(self, sequences):
        """One Mapping (or None) per sequence (str or bytes), in order."""
        sequences = list(sequences)
        with torch.cuda.device(self.device):
            res, chain, read_aoff, lens = self.chains(sequences)
            mapped = [None] * len(sequences)
            if chain is None:
                return mapped
            idx, strand, ctg, ts, tn, W = self.plan(res, lens)
            if not idx.size:
                return mapped
            queries = []
            for r, s in zip(idx.tolist(), strand.tolist()):
                q = np.frombuffer((sequences[r].encode() if isinstance(sequences[r], str) else bytes(sequences[r])).upper(),
                                  dtype=np.uint8)
                queries.append(_COMP[q[::-1]] if s else q)
            m = lens[idx]
            q_off = np.concatenate(([0], np.cumsum(m)[:-1])).astype(np.int64)
            query = _to_device(np.concatenate(queries), self.device)
            sizes = [native.map_align_trace_bytes(a, b) for a, b in zip(m.tolist(), W.tolist())]
            for group in _budget_groups(sizes, TRACE_BUDGET):
                g = np.asarray(group)
                slot = m[g] + tn[g]
                meta = np.stack([q_off[g], m[g], ts[g], tn[g], read_aoff[idx[g]], res[idx[g], 0], W[g],
                                 np.concatenate(([0], np.cumsum(np.asarray(sizes)[g])[:-1])),
                                 np.concatenate(([0], np.cumsum(slot)[:-1]))], axis=1).astype(np.int64)
                cen = torch.empty(max(int(m.sum()), 1), dtype=torch.int32, device=self.device)
                trace = torch.empty(max(int(np.asarray(sizes)[g].sum()), 1), dtype=torch.uint8, device=self.device)
                ops = torch.empty(max(int(slot.sum()), 1), dtype=torch.uint8, device=self.device)
                out = torch.empty(len(g), 6, dtype=torch.int32, device=self.device)
                native.map_align(query, self.ref, chain, _to_device(meta, self.device), int(W[g].max()), cen, trace, ops,
                                 out)
                o, ops_h = out.cpu().numpy(), ops.cpu().numpy()
                for t, p in enumerate(group):
                    score, qs, qe, t_st, t_en, n_ops = o[t].tolist()
                    if score <= 0:
                        continue
                    r, c = int(idx[p]), int(ctg[p])
                    end = int(meta[t, 8] + slot[t])
                    cigar, nm, md = cigar_nm_md(ops_h[end - n_ops:end], self._host[ts[p] + t_st:ts[p] + t_en])
                    if strand[p]:
                        qs, qe = int(lens[r]) - qe, int(lens[r]) - qs
                    base = int(ts[p] - self._ctg_off[c])
                    mapped[r] = Mapping(self.seq_names[c], base + t_st, base + t_en, qs, qe, -1 if strand[p] else 1,
                                        mapq(int(res[r, 1]), int(res[r, 2]), int(res[r, 0])), cigar, nm, md)
        return mapped


def align_map(aligner, results, n_thread=None, batch_reads=BATCH_READS, batch_bases=BATCH_BASES):
    """Adds `mapping` (a Mapping or None) to every (read, result) of `results`, in order (the shape of the reference's
    bonito/aligner.py align_map).  Consecutive reads are mapped in batches of at most `batch_reads` reads or `batch_bases`
    bases on a CUDA stream of their own, on a background thread.  `n_thread` is accepted for the reference's signature and
    has no effect."""
    done = queue.Queue(maxsize=2)
    sentinel = object()

    def work():
        try:
            stream = torch.cuda.Stream(aligner.device)
            batch, bases = [], 0
            for item in results:
                batch.append(item)
                bases += len(item[1]["sequence"])
                if len(batch) >= batch_reads or bases >= batch_bases:
                    done.put(_mapped(aligner, batch, stream))
                    batch, bases = [], 0
            if batch:
                done.put(_mapped(aligner, batch, stream))
            done.put(sentinel)
        except BaseException as err:       # raised again in the consumer
            done.put(err)

    Thread(target=work, daemon=True).start()
    while True:
        item = done.get()
        if item is sentinel:
            return
        if isinstance(item, BaseException):
            raise item
        yield from item


def _mapped(aligner, batch, stream):
    with torch.cuda.stream(stream):
        mappings = aligner.map_batch([res["sequence"] for _, res in batch])
    return [(read, {**res, "mapping": m}) for (read, res), m in zip(batch, mappings)]
