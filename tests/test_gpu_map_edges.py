"""The mapping kernels of bonito_b200/csrc/map.cu at their edges, byte for byte against the CPU oracle tests/_oracle_map.py:
alignment bands from W = 0 to the kernel's limit of 4096 and warps that align a wide pair and then a narrow one, index
hashes at MAX_OCC, the chaining limits (gap 10000, 50 predecessors, two lane passes, contig boundaries), extraction ties,
indels wide enough to reach MAX_BAND, grid-stride loops past 2^24 bases and a read of MAX_READ bases.

Every comparison is exact.  Each test prints what its cases reached (run with -s to see it)."""
import numpy as np
import pytest
import torch

import _oracle_map as O
from _map_helpers import _fasta, _mutate, _rand, _rc
from bonito_b200 import aligner as A
from bonito_b200 import native

pytestmark = pytest.mark.gpu
CANARY = 0xA5                    # not one of the op bytes = X I D
GRID_BASES = 65536 * 256         # the grid-stride kernels' threads per pass


def _cuda(a, dtype=None):
    return torch.from_numpy(np.ascontiguousarray(a if dtype is None else np.asarray(a, dtype=dtype))).cuda()


def _b(s):
    return np.frombuffer(bytes(s), dtype=np.uint8)


# ------------------------------------------------------------------------------------------------ map_align directly
def _launch_align(pairs, max_band):
    """pairs: [(query, target, chain [(q, r)] with r relative to the target, W)] in one b200_map_align launch ->
    [(score, i, ei, j, ej, cnt, ops)].  Every byte of an ops slot before its op string must still hold the canary."""
    qs, ts, chain, meta = [], [], [], []
    qoff = toff = coff = troff = soff = 0
    for q, t, ch, W in pairs:
        m, n = len(q), len(t)
        qs.append(_b(q))
        ts.append(_b(t))
        chain += [(cq, cr + toff) for cq, cr in ch]
        meta.append((qoff, m, toff, n, coff, len(ch), W, troff, soff))
        qoff, toff, coff = qoff + m, toff + n, coff + len(ch)
        troff += native.map_align_trace_bytes(m, W)
        soff += m + n
    meta = np.array(meta, dtype=np.int64).reshape(-1, 9)
    cen = torch.empty(max(qoff, 1), dtype=torch.int32, device="cuda")
    trace = torch.empty(max(troff, 1), dtype=torch.uint8, device="cuda")
    ops = torch.full((max(soff, 1),), CANARY, dtype=torch.uint8, device="cuda")
    out = torch.full((len(pairs), 6), -7, dtype=torch.int32, device="cuda")
    native.map_align(_cuda(np.concatenate(qs)), _cuda(np.concatenate(ts)), _cuda(np.array(chain, dtype=np.int64)),
                     _cuda(meta), max_band, cen, trace, ops, out)
    o, ops_h = out.cpu().numpy(), ops.cpu().numpy()
    res = []
    for p, row in enumerate(meta):
        slot = ops_h[row[8]:row[8] + row[1] + row[3]]
        cnt = int(o[p, 5])
        assert 0 <= cnt <= len(slot), (p, cnt)
        assert (slot[:len(slot) - cnt] == CANARY).all(), p
        res.append((*o[p].tolist(), slot[len(slot) - cnt:].tobytes()))
    return res


def _oracle_align(pair):
    q, t, ch, W = pair
    score, i, ei, j, ej, ops = O.band_align(bytes(q), bytes(t), ch, W)
    return (score, i, ei, j, ej, len(ops), ops)


def _cells(W):
    return native.map_align_trace_bytes(1, W) // 16      # band_cells(W)


def _width_pair(rng, W):
    """A query whose alignment runs about W - W/8 columns right of a straight chain, with a small deletion and insertion:
    the path uses the band's far side, and its traceback words past the first when W >= 256."""
    D = W - W // 8
    core = _rand(rng, 220)
    q = np.concatenate((_mutate(rng, core[:100], 0.03, 0, 0), core[106:180], _rand(rng, 4), core[180:]))
    t = np.concatenate((_rand(rng, D), core, _rand(rng, 20)))
    return q.tobytes(), t.tobytes(), [(0, 0), (len(q) - 1, len(q) - 1)], W


WIDTHS = [0, 1, 15, 16, 127, 128, 255, 256, 1023, 1024, 2047, 2048, 4095, 4096]


def test_align_band_widths():
    """W on both sides of every band_cells step up to the kernel's limit: each alone at max_band = W, then all in one
    launch at max_band = 4096 (a shared-memory pitch wider than every pair's)."""
    rng = np.random.default_rng(10)
    pairs = [_width_pair(rng, W) for W in WIDTHS]
    want = [_oracle_align(p) for p in pairs]
    for p, w in zip(pairs, want):
        assert _launch_align([p], p[3]) == [w], p[3]
        assert w[0] > 100, p[3]                        # the core aligns at every width
    assert _launch_align(pairs, 4096) == want
    print(f"reached: W up to {max(WIDTHS)} against the oracle; band_cells values {sorted({_cells(W) for W in WIDTHS})}")


def _geometry_pairs(rng):
    t = _rand(rng, 600)
    pairs = []
    # first rows: the band reaches column 0, starts at column 1 (W = 0 too), starts at column 2
    q = _mutate(rng, t[:300], 0.03, 0.01, 0.01).tobytes()
    for W in (0, 8, 40):
        pairs.append((q, t[:320].tobytes(), [(0, 0), (len(q) - 1, 299)], W))
        pairs.append((t[W:W + 200].tobytes(), t[:400].tobytes(), [(0, W), (199, W + 199)], W))        # lo == 1
        pairs.append((t[W + 1:W + 201].tobytes(), t[:400].tobytes(), [(0, W + 1), (199, W + 200)], W))  # lo == 2
    # last rows whose band runs past n
    pairs.append((t[300:500].tobytes(), t[:500].tobytes(), [(0, 300), (199, 499)], 30))
    # query overhangs: whole rows outside the target at both ends
    q = np.concatenate((_rand(rng, 60), t[:200], _rand(rng, 60))).tobytes()
    pairs.append((q, t[:200].tobytes(), [(60, 0), (259, 199)], 16))
    # a steep segment (a deletion of 299): the centre moves by more than 2W + 1 between two rows
    q = np.concatenate((t[:101], t[400:500])).tobytes()
    pairs.append((q, t[:500].tobytes(), [(0, 0), (100, 100), (101, 400), (200, 499)], 16))
    # a flat segment (an insertion of 300): the centre stays put for 300 rows
    q = np.concatenate((t[:100], _rand(rng, 300), t[100:200])).tobytes()
    pairs.append((q, t[:200].tobytes(), [(0, 0), (99, 99), (400, 100), (499, 199)], 16))
    pairs.append((q, t[:200].tobytes(), [(0, 0), (99, 99), (400, 100), (499, 199)], 300))
    return pairs


def _content_pairs(rng):
    unit = b"ACGGT"
    hom = b"GATTACA" + b"A" * 30 + b"C" * 20 + unit * 12 + b"TTTTTTGGGG" + b"AC" * 15
    hom_q = b"GATTACA" + b"A" * 27 + b"C" * 22 + unit * 10 + b"TTTTTGGGG" + b"AC" * 17
    t = _rand(rng, 300)
    qn = _mutate(rng, t[:250], 0.02, 0.01, 0.01).copy()
    qn[100:110] = ord("N")
    tn = t.copy()
    tn[40:45] = ord("N")
    rnd = _rand(rng, 250).tobytes()
    diag = lambda q, t, W: (q, t, [(0, 0), (len(q) - 1, len(q) - 1)], W)
    return [
        diag(_mutate(rng, t, 0.05, 0.03, 0.03).tobytes(), t.tobytes(), 24),       # random with errors
        diag(hom_q, hom, 24),                                                     # homopolymers and a tandem repeat
        diag(hom, hom, 24),
        diag(unit * 20, unit * 23, 40),
        diag(b"A" * 50, b"A" * 64, 20),
        diag(qn.tobytes(), tn.tobytes(), 24),                                     # N runs in both
        diag(b"N" * 30, t[:40].tobytes(), 8),                                     # only N: no positive cell
        diag(rnd, rnd, 16),                                                       # identical
        diag(b"A" * 20, b"C" * 30, 16),                                           # no positive cell
        diag(b"A", b"A", 0), diag(b"A", b"C", 3), diag(b"G", b"N", 1),            # m = n = 1
        (b"A", t[:50].tobytes(), [(0, 25)], 30),                                  # m = 1
        (t[:50].tobytes(), t[20:21].tobytes(), [(20, 0)], 30),                    # n = 1
    ]


def test_align_band_geometry_and_content():
    rng = np.random.default_rng(11)
    pairs = _geometry_pairs(rng) + _content_pairs(rng)
    want = [_oracle_align(p) for p in pairs]
    assert _launch_align(pairs, max(p[3] for p in pairs)) == want
    assert [_launch_align([p], p[3])[0] for p in pairs] == want
    assert _launch_align(pairs, 4096) == want
    zero = sum(w[0] == 0 for w in want)
    assert zero >= 4 and all(w[5] == 0 for w in want if w[0] == 0)
    print(f"reached: {len(pairs)} geometry / content pairs, {zero} without a positive cell")


def _small_pair(rng, W, m):
    t = _rand(rng, m + 10)
    q = _mutate(rng, t[3:m + 3], 0.04, 0.02, 0.02)
    return q.tobytes(), t.tobytes(), [(0, 3), (len(q) - 1, min(len(q) + 2, m + 9))], W


def _wide_pair(rng, W):
    D = W - 100 + int(rng.integers(0, 60))
    core = _rand(rng, 60)
    t = np.concatenate((_rand(rng, D), core, _rand(rng, 5)))
    return _mutate(rng, core, 0.03, 0.02, 0.02).tobytes(), t.tobytes(), [(0, 0), (59, 59)], W


def test_align_warp_reuse():
    """4096 + 77 pairs: the grid has 4096 warps, so pair p and pair p + 4096 share one.  Wide pairs (W near 1024) then
    narrow ones (W = 64) on the same warps, then the other way round; every pair equals itself launched alone."""
    rng = np.random.default_rng(12)
    extra = 77
    wide = [_wide_pair(rng, 1024 - int(rng.integers(0, 24))) for _ in range(extra)]
    narrow = [_small_pair(rng, 64, 60) for _ in range(extra)]
    middle = [_small_pair(rng, 16, 30) for _ in range(4096 - extra)]
    solo = {}
    for p in wide + narrow:
        solo[id(p)] = _launch_align([p], p[3])[0]
    rest = _launch_align(middle, 16)
    oracle = {id(p): _oracle_align(p) for p in wide + narrow}
    assert all(solo[id(p)] == oracle[id(p)] for p in wide + narrow)
    sample = list(range(0, len(middle), 101))
    assert [rest[t] for t in sample] == [_oracle_align(middle[t]) for t in sample]
    for first, second in ((wide, narrow), (narrow, wide)):
        pairs = first + middle + second
        got = _launch_align(pairs, 1024)
        assert got[:extra] == [solo[id(p)] for p in first]
        assert got[4096:] == [solo[id(p)] for p in second]
        assert got[extra:4096] == rest
    print(f"reached: {2 * 2 * extra} pairs on reused warps ({2 * extra} distinct) against the oracle")


def test_align_refusals():
    rng = np.random.default_rng(13)
    q, t, ch, _ = _small_pair(rng, 16, 40)
    meta = _cuda(np.array([[0, len(q), 0, len(t), 0, 2, 16, 0, 0]], dtype=np.int64))
    out = torch.full((1, 6), -7, dtype=torch.int32, device="cuda")
    ops = torch.full((len(q) + len(t),), CANARY, dtype=torch.uint8, device="cuda")
    cen = torch.zeros(len(q), dtype=torch.int32, device="cuda")
    trace = torch.zeros(native.map_align_trace_bytes(len(q), 16), dtype=torch.uint8, device="cuda")
    args = (_cuda(_b(q)), _cuda(_b(t)), _cuda(np.array(ch, dtype=np.int64)))
    with pytest.raises(native.NativeError, match="bad sizes"):
        native.map_align(*args, meta, 4097, cen, trace, ops, out)
    torch.cuda.synchronize()
    assert (out.cpu() == -7).all() and (ops.cpu() == CANARY).all()
    native.map_align(*args, meta[:0], 4096, cen, trace, ops, out[:0])
    torch.cuda.synchronize()
    assert (out.cpu() == -7).all() and (ops.cpu() == CANARY).all() and not cen.any() and not trace.any()


# ------------------------------------------------------------------------------------------------ anchors at MAX_OCC
def _anchors_by_rule(mm, off, k, table, max_occ):
    """count per position and the anchors (akey, aq) in write order, from the header rules."""
    count = np.zeros(len(mm), dtype=np.int32)
    akey, aq = [], []
    for s in range(len(off) - 1):
        L = int(off[s + 1] - off[s])
        for x in range(L):
            key = int(mm[off[s] + x])
            hits = table.get(key >> 1, []) if key >= 0 else []
            if not hits or len(hits) > max_occ:
                continue
            count[off[s] + x] = len(hits)
            for v in hits:
                rel = (key ^ v) & 1
                akey.append(s << 33 | rel << 32 | v >> 1)
                aq.append(L - x - k if rel else x)
    return count, np.array(akey, dtype=np.int64), np.array(aq, dtype=np.int32)


def test_anchor_kernel_at_max_occ():
    """Hand-built index tables with 1, 2, 499, 500 and 501 entries per hash, entries of both strands and positions up to
    2^32 - 1; read keys absent from the table, below its smallest and above its largest hash."""
    rng = np.random.default_rng(20)
    k = 15
    sizes = {1000: 1, 2000: 499, 3000: 500, 4000: 501, 5000: 2}
    table = {}
    for h, n in sizes.items():
        pos = np.sort(rng.integers(0, 1 << 32, n, dtype=np.int64))
        if h == 5000:
            pos[-1] = (1 << 32) - 1
        table[h] = ((pos << 1) | rng.integers(0, 2, n)).tolist()
    uniq = np.array(sorted(table), dtype=np.int64)
    start = np.concatenate(([0], np.cumsum([len(table[h]) for h in uniq]))).astype(np.int64)
    val = np.concatenate([table[h] for h in uniq]).astype(np.int64)
    lens = [60, 0, 40, 15, 80]
    off = np.concatenate(([0], np.cumsum(lens))).astype(np.int64)
    mm = np.full(off[-1], -1, dtype=np.int64)
    hashes = [1000, 2000, 3000, 4000, 5000, 7, 2500, 9999]       # 7 and 9999 lie outside the table, 2500 between
    for s, L in enumerate(lens):
        for x in range(0, L - k + 1, 3):
            mm[off[s] + x] = hashes[(s + x) % len(hashes)] << 1 | int(rng.integers(0, 2))
    dropped = 0
    for max_occ in (500, 499, 0, 1 << 20):
        want_count, want_key, want_q = _anchors_by_rule(mm, off, k, table, max_occ)
        count = torch.full((len(mm),), -7, dtype=torch.int32, device="cuda")
        args = (_cuda(mm), _cuda(off), k, _cuda(uniq), _cuda(start), _cuda(val), max_occ)
        native.map_anchors(*args, count=count)
        assert np.array_equal(count.cpu().numpy(), want_count), max_occ
        aoff = np.concatenate(([0], np.cumsum(want_count)[:-1])).astype(np.int64)
        n = len(want_key)
        akey = torch.full((max(n, 1),), -7, dtype=torch.int64, device="cuda")
        aq = torch.full((max(n, 1),), -7, dtype=torch.int32, device="cuda")
        native.map_anchors(*args, aoff=_cuda(aoff), akey=akey, aq=aq)
        if n:
            assert np.array_equal(akey.cpu().numpy(), want_key) and np.array_equal(aq.cpu().numpy(), want_q), max_occ
        else:
            assert int(akey[0]) == -7 and int(aq[0]) == -7
        if max_occ == 500:
            dropped = int(sum(len(table[int(m >> 1)]) for m in mm if m >= 0 and len(table.get(int(m >> 1), [])) > 500))
            assert dropped > 0 and (want_count == 500).any() and ((want_key >> 32) & 1).any()
    print(f"reached: {dropped} anchors dropped by max_occ = 500 on the hand-built table")


def _oracle_chains_and_maps(al, index, reads):
    """Aligner.chains and map_batch against the oracle, read by read; -> (the per-read chain rows, the mappings)."""
    res, _, _, _ = al.chains(reads)
    got = al.map_batch(reads)
    for t, read in enumerate(reads):
        anc = O.anchors(index, read, index.k)
        f, pred = O.chain_dp(anc, index.off, index.k)
        ch = O.extract(anc, f, pred, len(read), index.k)
        if ch is None:
            assert res[t, 0] == 0, t
        else:
            assert res[t].tolist() == [ch["n"], ch["f1"], ch["f2"], ch["strand"], ch["W"], *ch["chain"][0],
                                       *ch["chain"][-1]], t
        assert (None if got[t] is None else tuple(vars(got[t]).values())) == O.map_read(index, read), t
    return res, got


@pytest.fixture(scope="module")
def repeat_genome(tmp_path_factory):
    """A 200-base unit in exactly 500 copies and another in 501, each copy between random spacers."""
    rng = np.random.default_rng(21)
    ua, ub = _rand(rng, 200), _rand(rng, 200)
    parts, starts = [], []
    pos = 0
    for c in range(1001):
        sp = _rand(rng, 120)
        parts += [sp, ua if c < 500 else ub]
        starts.append(pos + 120)
        pos += 320
    parts.append(_rand(rng, 120))
    seq = np.concatenate(parts)
    path = tmp_path_factory.mktemp("rep") / "ref.fa"
    _fasta(path, [("rep", seq)])
    return str(path), seq, starts


@pytest.mark.parametrize("preset", ["lr:hq", "map-ont"])
def test_map_at_max_occ(repeat_genome, preset):
    path, seq, starts = repeat_genome
    rng = np.random.default_rng(22)
    al = A.Aligner(path, preset=preset)
    index = O.Index([("rep", seq.tobytes())], *A.PRESETS[preset])
    occ = [len(v) for v in index.table.values()]
    assert occ.count(500) >= 3 and occ.count(501) >= 3 and max(occ) == 501
    reads = []
    for c in (3, 250, 499, 500, 501, 1000):                        # copies of either unit, and the two on the border
        st = starts[c]
        r = _mutate(rng, seq[st - 100:st + 300], 0.01, 0, 0)
        reads.append((r if c % 2 else _rc(r)).tobytes())
    reads.append(seq[starts[10] + 20:starts[10] + 180].tobytes())   # inside one copy: only 500-hit seeds
    res, got = _oracle_chains_and_maps(al, index, reads)
    assert sum(g is not None for g in got) >= 5
    dropped = sum(len(index.table[key >> 1]) for read in reads for _, key in O.minimizers(read, index.k, index.w)
                  if len(index.table.get(key >> 1, [])) > A.MAX_OCC)
    assert dropped > 0
    print(f"reached: {preset}: {dropped} anchors dropped by MAX_OCC over {len(reads)} reads; "
          f"{occ.count(500)} hashes at 500 entries, {occ.count(501)} at 501")


# ------------------------------------------------------------------------------------------------ map_chain directly
TIES = [(35, 1), (45, 34), (20, 5)]


def _chain_templates():
    """Reads as [(strand, r, q)] in the host's order (strand, then r), each at one chaining edge."""
    T = []
    T.append([(0, 6000, 0), (0, 16000, 10000)])                  # dr = dq = 10000: linked
    T.append([(0, 6000, 0), (0, 16001, 10001)])                  # 10001: not
    T.append([(0, 6000, 0), (0, 16000, 10001)])                  # dq = 10001
    T.append([(0, 6000, 0), (0, 16001, 10000)])                  # dr = 10001
    T.append([(0, 6000, 0), (0, 15990, 10000)])                  # dq = 10000, dr = 9990
    T.append([(0, 500, 0), (0, 500, 30), (0, 530, 60)])          # dr = 0
    T.append([(0, 100, 50), (0, 130, 20), (0, 160, 80), (0, 190, 110)])   # a negative dq
    for back in (33, 40, 49, 50, 51):
        # a short colinear chain, its best anchor `back` before the last one, unlinkable anchors in between
        head = [(0, 10 * u, 10 * u) for u in range(6)]
        fill = [(0, 100 + 10 * t, 5000 - t) for t in range(back - 1)]
        T.append(head + fill + [(0, 1000, 1000)])
    for a, b in TIES:
        # equal-score predecessors a and b anchors back (one or both in the second lane pass): ties go to the largest j
        fill = [(0, 100, 5000 + t) for t in range(a - b - 1)]
        T.append([(0, 100, 0)] + fill + [(0, 100, 0)] + [(0, 100, 6000 + t) for t in range(b - 1)] + [(0, 140, 40)])
    T.append([(0, 100, 0), (0, 130, 30), (1, 160, 60), (1, 190, 90)])     # a strand change
    T.append([(0, 4970, 0), (0, 4990, 20), (0, 5001, 31), (0, 5002, 32), (0, 5010, 40), (0, 5030, 60)])  # contigs 3 bases apart
    T.append([(0, 7 * u + (u % 5), 7 * u) for u in range(150)])           # more than 64 anchors: the ring wraps
    T.append([(0, 200 + 11 * u, 9 * u) for u in range(70)])
    T.append([(1, (1 << 32) - 400 + 20 * u, 20 * u) for u in range(19)])  # r near 2^32
    T.append([])
    T.append([(1, 777, 5)])
    return T


CHAIN_CTG = np.array([0, 5000, 5003, 1 << 32], dtype=np.int64)


def _launch_chain(templates, want, reads, k):
    """Reads (template indices) in one b200_map_chain launch; f and pred must equal the oracle's `want` per template."""
    n_t = np.array([len(templates[tp]) for tp in reads], dtype=np.int64)
    aoff = np.concatenate(([0], np.cumsum(n_t)))
    cat = lambda rows, dtype: np.concatenate([np.asarray(rows[tp], dtype=dtype).reshape(-1) for tp in reads])
    anc = cat([np.array(tp, dtype=np.int64).reshape(-1, 3) for tp in templates], np.int64).reshape(-1, 3)
    rd = np.repeat(np.arange(len(reads), dtype=np.int64), n_t)
    akey = rd << 33 | anc[:, 0] << 32 | anc[:, 1]
    assert np.array_equal(np.argsort(akey, kind="stable"), np.arange(len(akey)))      # the host's order
    want_f = cat([wf for wf, _ in want], np.int64)
    local = cat([wp for _, wp in want], np.int64)
    want_pred = np.where(local >= 0, local + np.repeat(aoff[:-1], n_t), -1)
    f = torch.full((len(akey),), -7, dtype=torch.int32, device="cuda")
    pred = torch.full_like(f, -7)
    native.map_chain(_cuda(akey), _cuda(anc[:, 2], np.int32), _cuda(aoff), _cuda(CHAIN_CTG), k, f, pred)
    assert np.array_equal(f.cpu().numpy(), want_f) and np.array_equal(pred.cpu().numpy(), want_pred), len(reads)


def test_chain_kernel_limits():
    """Every template alone, then all of them cycled over 4 * 65536 + 1000 reads in one launch (the grid's warps take a
    second read each)."""
    k = 15
    T = _chain_templates()
    want = [O.chain_dp(tp, CHAIN_CTG, k) for tp in T]
    # the edges the templates are built for
    assert want[0][1][1] == 0 and want[1][1][1] == want[2][1][1] == want[3][1][1] == -1 and want[4][1][1] == 0
    assert [want[7 + t][1][-1] for t in range(5)] == [5, 5, 5, 5, -1]      # the chain head's last anchor, 51 back: none
    assert [want[12 + t][1][-1] for t in range(3)] == [len(T[12 + t]) - 1 - b for t, (_, b) in enumerate(TIES)]
    n_reads = 4 * 65536 + 1000
    _launch_chain(T, want, list(range(len(T))), k)
    _launch_chain(T, want, [rd % len(T) for rd in range(n_reads)], k)
    print(f"reached: {len(T)} chain templates, {n_reads} reads in one launch")


# ------------------------------------------------------------------------------------------------ map_extract directly
def _extract_reads(k):
    """[(anchors, read length)]: equal-f chains, secondaries overlapping the primary by half the shorter span and by one
    base less (on both strands), and diagonal jumps that put W at MAX_BAND - 1, MAX_BAND and past it."""
    col = lambda s, r, q0, n, step=10: [(s, r + step * u, q0 + step * u) for u in range(n)]
    reads = []
    reads.append((col(0, 1000, 0, 10) + col(0, 30000, 0, 10), 200))           # equal f: the lower index is primary
    # primary [0, 105); a secondary [60, 150) overlaps it by 45 = half of 90; [61, 150) by 44 < 89 / 2
    for q0 in (60, 61):
        sec = [(0, 40000 + q - q0, q) for q in (q0, 75, 90, 105, 120, 135)]
        reads.append((col(0, 1000, 0, 10) + sec, 300))
        reads.append(([(1, r, q) for _, r, q in col(0, 1000, 0, 10) + sec], 300))
    for jump in (1983, 1984, 1985, 2500):
        reads.append((col(0, 1000, 0, 40) + col(0, 1400 + jump, 400, 40), 900))   # d jumps by `jump` mid-chain
    reads.append((col(0, 1000, 0, 5) + col(1, 1000, 0, 5, 11), 100))           # two strands, the second one longer
    reads.append(([], 50))
    return reads


def test_extract_kernel_ties_overlap_and_cap():
    k = 15
    cases = _extract_reads(k)
    akey, aq, f, pred, aoff, soff, want = [], [], [], [], [0], [0], []
    for rd, (anc, L) in enumerate(cases):
        anc = sorted(anc, key=lambda a: (a[0], a[1]))
        wf, wp = O.chain_dp(anc, CHAIN_CTG, k)
        base = len(akey)
        akey += [rd << 33 | s << 32 | r for s, r, _ in anc]
        aq += [q for _, _, q in anc]
        f += wf
        pred += [base + p if p >= 0 else -1 for p in wp]
        aoff.append(len(akey))
        soff.append(soff[-1] + L)
        want.append(O.extract(anc, wf, wp, L, k, A.MAX_BAND))
    akey, f = np.array(akey, dtype=np.int64), np.array(f, dtype=np.int64)
    order = np.argsort(((akey >> 33) << 32) | (0x7FFFFFFF - f), kind="stable")
    n = len(akey)
    taken = torch.zeros(n, dtype=torch.uint8, device="cuda")
    chain = torch.full((n, 2), -7, dtype=torch.int64, device="cuda")
    out = torch.full((len(cases), 9), -7, dtype=torch.int64, device="cuda")
    native.map_extract(_cuda(akey), _cuda(aq, np.int32), _cuda(f, np.int32), _cuda(pred, np.int32), _cuda(order),
                       _cuda(np.array(aoff, dtype=np.int64)), _cuda(np.array(soff, dtype=np.int64)), k, A.MAX_BAND,
                       taken, chain, out)
    o, ch = out.cpu().numpy(), chain.cpu().numpy()
    for rd, w in enumerate(want):
        if w is None:
            assert o[rd, 0] == 0, rd
            continue
        assert o[rd].tolist() == [w["n"], w["f1"], w["f2"], w["strand"], w["W"], *w["chain"][0], *w["chain"][-1]], rd
        assert [tuple(x) for x in ch[aoff[rd]:aoff[rd] + w["n"]].tolist()] == w["chain"], rd
    f2 = [w["f2"] for w in want[1:5]]
    assert f2[0] > 0 and f2[1] > 0 and f2[2] == 0 and f2[3] == 0          # half overlap counts, one base less does not
    assert want[0]["chain"][0] == (0, 1000)
    assert [w["W"] for w in want[5:9]] == [2047, 2048, 2048, 2048]


# ------------------------------------------------------------------------------------------------ indels and contig edges
@pytest.fixture(scope="module")
def indel_genome(tmp_path_factory):
    rng = np.random.default_rng(30)
    contigs = [("chrA", _rand(rng, 60000)), ("chrB", _rand(rng, 20000)), ("chrC", _rand(rng, 5000))]
    path = tmp_path_factory.mktemp("indel") / "ref.fa"
    _fasta(path, contigs)
    return str(path), contigs


INDELS = [150, 700, 1500, 1990, 2100]     # the last two reach MAX_BAND (a diagonal change above 1984)


@pytest.mark.parametrize("preset", ["lr:hq", "map-ont"])
def test_map_planted_indels_reach_max_band(indel_genome, preset):
    path, contigs = indel_genome
    rng = np.random.default_rng(31 if preset == "lr:hq" else 32)
    al = A.Aligner(path, preset=preset)
    index = O.Index([(n, s.tobytes()) for n, s in contigs], *A.PRESETS[preset])
    a = contigs[0][1]
    reads = []
    for t, D in enumerate(INDELS):
        st = 1000 + 11000 * t
        dele = np.concatenate((a[st:st + 600], a[st + 600 + D:st + 1200 + D]))
        ins = np.concatenate((a[st + 5000:st + 5600], _rand(rng, D), a[st + 5600:st + 6200]))
        reads += [(_rc(dele) if t % 2 else dele).tobytes(), (ins if t % 2 else _rc(ins)).tobytes()]
    res, got = _oracle_chains_and_maps(al, index, reads)
    W = res[:, 4].tolist()
    assert all(128 <= w <= A.MAX_BAND for w in W), W
    assert W[-4:] == [A.MAX_BAND] * 4, W
    assert all(g is not None for g in got)
    assert {op for g in got for op in "ID" if op in g.cigar_str} == {"I", "D"}
    print(f"reached: {preset}: W {sorted(W)} through map_batch against the oracle")


@pytest.mark.parametrize("preset", ["lr:hq", "map-ont"])
def test_map_contig_edges(indel_genome, preset):
    """Reads overhanging a contig's start or end with random bases, and reads joining one contig's end to the next's
    start."""
    path, contigs = indel_genome
    rng = np.random.default_rng(33 if preset == "lr:hq" else 34)
    al = A.Aligner(path, preset=preset)
    index = O.Index([(n, s.tobytes()) for n, s in contigs], *A.PRESETS[preset])
    a, b, c = (s for _, s in contigs)
    reads = [np.concatenate((_rand(rng, 200), b[:800])), np.concatenate((b[-800:], _rand(rng, 150))),
             np.concatenate((a[-600:], b[:600])), np.concatenate((b[-300:], c[:900])),
             np.concatenate((_rand(rng, 40), c[:400], _rand(rng, 40))), _mutate(rng, np.concatenate((a[-500:], b[:200])),
                                                                                  0.02, 0.01, 0.01)]
    reads = [(_rc(r) if t % 2 else r).tobytes() for t, r in enumerate(reads)]
    _, got = _oracle_chains_and_maps(al, index, reads)
    assert sum(g is not None for g in got) >= 5


# ------------------------------------------------------------------------------------------------ sizes and host limits
@pytest.mark.parametrize("filler", ["random", "N"])
def test_minimizers_past_one_grid(filler):
    rng = np.random.default_rng(40)
    n_fill = GRID_BASES + 12345
    fill = _rand(rng, n_fill) if filler == "random" else np.full(n_fill, ord("N"), dtype=np.uint8)
    tests = [_rand(rng, 5000), _rand(rng, 36), _rand(rng, 37), _rand(rng, 2000), _rand(rng, 3)]
    tests[3][700:760] = ord("N")
    for k, w in A.PRESETS.values():
        seqs = [fill] + tests
        off = np.concatenate(([0], np.cumsum([len(s) for s in seqs]))).astype(np.int64)
        kmer = torch.empty(off[-1], dtype=torch.int64, device="cuda")
        mm = torch.empty_like(kmer)
        native.map_minimizers(_cuda(np.concatenate(seqs)), _cuda(off), k, w, kmer, mm)
        got = mm.cpu().numpy()
        alone_off = off[1:] - off[1]
        kmer2 = torch.empty(alone_off[-1], dtype=torch.int64, device="cuda")
        mm2 = torch.empty_like(kmer2)
        native.map_minimizers(_cuda(np.concatenate(tests)), _cuda(alone_off), k, w, kmer2, mm2)
        assert np.array_equal(got[off[1]:], mm2.cpu().numpy()), (k, w)
        for s, o in zip(tests, off[1:-1]):
            want = np.full(len(s), -1, dtype=np.int64)
            for p, key in O.minimizers(s.tobytes(), k, w):
                want[p] = key
            assert np.array_equal(got[o:o + len(s)], want), (k, w, len(s))
        assert (got[off[1]:] >= 0).sum() > 100
        if filler == "N":
            assert (got[:n_fill] == -1).all()
    print(f"reached: {off[-1]} bases ({off[-1] / GRID_BASES:.3f} grids) in one map_minimizers launch")


def test_anchors_past_one_grid(indel_genome):
    """map_batch on 34 random reads of 500 000 bases and then reads of chrA (more than 2^24 bases in all) equals
    map_batch over slices of fewer than 2^24 bases, and the oracle on the reads past 2^24."""
    path, contigs = indel_genome
    rng = np.random.default_rng(41)
    al = A.Aligner(path)
    index = O.Index([(n, s.tobytes()) for n, s in contigs], *A.PRESETS["lr:hq"])
    reads = [_rand(rng, A.MAX_READ).tobytes() for _ in range(34)]
    a = contigs[0][1]
    for t in range(16):
        st = int(rng.integers(0, len(a) - 3000))
        r = _mutate(rng, a[st:st + int(rng.integers(1000, 3000))], 0.02, 0.01, 0.01)
        reads.append((_rc(r) if t % 2 else r).tobytes())
    total = sum(len(r) for r in reads)
    assert total > GRID_BASES
    whole = al.map_batch(reads)
    assert whole == al.map_batch(reads[:17]) + al.map_batch(reads[17:34]) + al.map_batch(reads[34:])
    assert all(m is not None for m in whole[34:])
    for t in range(34, len(reads), 3):
        assert tuple(vars(whole[t]).values()) == O.map_read(index, reads[t]), t
    print(f"reached: {total} bases ({total / GRID_BASES:.3f} grids) in one map_batch")


def test_map_read_of_max_read_bases(tmp_path):
    """A read of exactly MAX_READ bases copied from a contig maps full length on both strands (score 2 per base, the end
    cell's key within 5 % of its 20 score bits); one base more and it is not mapped."""
    rng = np.random.default_rng(42)
    ctg = _rand(rng, A.MAX_READ + 30000)
    _fasta(tmp_path / "ref.fa", [("big", ctg)])
    al = A.Aligner(str(tmp_path / "ref.fa"))
    index = O.Index([("big", ctg.tobytes())], *A.PRESETS["lr:hq"])
    st = 12345
    read = ctg[st:st + A.MAX_READ]
    reads = [read.tobytes(), _rc(read).tobytes(), ctg[st:st + A.MAX_READ + 1].tobytes()]
    res, _, _, _ = al.chains(reads)
    got = al.map_batch(reads)
    for t, strand in ((0, 1), (1, -1)):
        anc = O.anchors(index, reads[t], index.k)
        f, pred = O.chain_dp(anc, index.off, index.k)
        ch = O.extract(anc, f, pred, A.MAX_READ, index.k)
        assert res[t, :3].tolist() == [ch["n"], ch["f1"], ch["f2"]]
        assert got[t] == A.Mapping("big", st, st + A.MAX_READ, 0, A.MAX_READ, strand, O.mapq(ch["f1"], ch["f2"], ch["n"]),
                                   f"{A.MAX_READ}M", 0, str(A.MAX_READ))
    assert res[2, 0] == 0 and got[2] is None
    assert 2 * A.MAX_READ < 1 << 20


def test_map_batch_in_several_align_launches(indel_genome, monkeypatch):
    """A trace budget that fits one alignment at a time splits the batch into many map_align launches; the result is the
    same."""
    path, contigs = indel_genome
    rng = np.random.default_rng(43)
    al = A.Aligner(path, preset="map-ont")
    a, b = contigs[0][1], contigs[1][1]
    reads = []
    for t in range(12):
        c = a if t % 3 else b
        st = int(rng.integers(0, len(c) - 2500))
        r = _mutate(rng, c[st:st + int(rng.integers(300, 2500))], 0.03, 0.02, 0.02)
        reads.append((_rc(r) if t % 2 else r).tobytes())
    one = al.map_batch(reads)
    res, _, _, lens = al.chains(reads)
    idx, _, _, _, _, W = al.plan(res, lens)
    sizes = [native.map_align_trace_bytes(m, w) for m, w in zip(lens[idx].tolist(), W.tolist())]
    budget = max(sizes)
    groups = A._budget_groups(sizes, budget)
    assert len(groups) >= 3 and sum(len(g) for g in groups) == len(sizes)
    monkeypatch.setattr(A, "TRACE_BUDGET", budget)
    assert al.map_batch(reads) == one
    assert sum(m is not None for m in one) >= 12
    print(f"reached: {len(groups)} map_align launches for one batch")
