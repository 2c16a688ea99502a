"""
CPU oracle of the mapping rules of bonito_b200/csrc/map.cu, written again from the rules in plain numpy / Python:
minimizers, the index, anchors, the chaining DP and the greedy extraction, MAPQ, the banded local alignment with full
band matrices and a traceback, and CIGAR / NM / MD from the op string.
"""

import math

import numpy as np

NEG = -(1 << 30)
MAX_PRED, MAX_GAP, MAX_OCC, MAX_BAND = 50, 10000, 500, 2048
_CODE = np.full(256, -1, dtype=np.int64)
_CODE[np.frombuffer(b"ACGT", dtype=np.uint8)] = np.arange(4)


def hash64(key, mask):
    key = (~key + (key << 21)) & mask
    key = key ^ key >> 24
    key = ((key + (key << 3)) + (key << 8)) & mask
    key = key ^ key >> 14
    key = ((key + (key << 2)) + (key << 4)) & mask
    key = key ^ key >> 28
    key = (key + (key << 31)) & mask
    return key


def kmer_keys(seq, k):
    """Per k-mer start: hash << 1 | strand, or -1 (an N in the k-mer)."""
    c = _CODE[np.frombuffer(bytes(seq), dtype=np.uint8)]
    nk = len(c) - k + 1
    if nk <= 0:
        return np.zeros(0, dtype=np.int64)
    fwd = np.zeros(nk, dtype=np.uint64)
    rev = np.zeros(nk, dtype=np.uint64)
    bad = np.zeros(nk, dtype=bool)
    for t in range(k):
        ct = c[t:t + nk]
        bad |= ct < 0
        cu = np.where(ct < 0, 0, ct).astype(np.uint64)
        fwd = (fwd << np.uint64(2)) | cu
        rev |= (np.uint64(3) - cu) << np.uint64(2 * t)
    mask = (1 << (2 * k)) - 1
    h = np.array([hash64(int(v), mask) for v in np.minimum(fwd, rev).tolist()], dtype=np.int64)
    keys = (h << 1) | (fwd > rev).astype(np.int64)
    keys[bad] = -1
    return keys


def minimizers(seq, k, w):
    """[(position, key)] in position order."""
    keys = kmer_keys(seq, k)
    if len(keys) < w:
        return []
    hashes = np.where(keys >= 0, keys >> 1, np.iinfo(np.int64).max)
    win = np.lib.stride_tricks.sliding_window_view(hashes, w)
    at = np.argmin(win, axis=1) + np.arange(win.shape[0])      # argmin: the first (leftmost) of equal hashes
    at = np.unique(at[keys[at] >= 0])
    return list(zip(at.tolist(), keys[at].tolist()))


class Index:
    def __init__(self, contigs, k, w):
        self.k, self.w = k, w
        self.names = [n for n, _ in contigs]
        self.seqs = [bytes(s) for _, s in contigs]
        self.off = np.concatenate(([0], np.cumsum([len(s) for s in self.seqs]))).astype(np.int64)
        entries = []
        for c, s in enumerate(self.seqs):
            entries += [(key >> 1, int(self.off[c]) + p, key & 1) for p, key in minimizers(s, k, w)]
        entries.sort(key=lambda e: (e[0], e[1]))
        self.table = {}
        for h, pos, strand in entries:
            self.table.setdefault(h, []).append((pos, strand))


def anchors(index, read, k):
    """[(strand, r, q)] in the sorted order: stable by (strand, r); ties keep (read minimizer, entry) order."""
    out = []
    L = len(read)
    for x, key in minimizers(read, k, index.w):
        hits = index.table.get(key >> 1, [])
        if len(hits) > MAX_OCC:
            continue
        for pos, strand in hits:
            s = (key & 1) ^ strand
            out.append((s, pos, L - x - k if s else x))
    out.sort(key=lambda a: (a[0], a[1]))
    return out


def gamma(d, k):
    return 0 if d == 0 else (k * d) // 100 + (d.bit_length() - 1) // 2


def chain_dp(anc, ctg_off, k):
    n = len(anc)
    f, pred = [0] * n, [-1] * n
    for i in range(n):
        si, ri, qi = anc[i]
        ci = int(np.searchsorted(ctg_off, ri, side="right")) - 1
        best, bj = 0, -1
        for j in range(i - 1, max(-1, i - 1 - MAX_PRED), -1):     # nearest first: a later j wins only when strictly better
            sj, rj, qj = anc[j]
            dr, dq = ri - rj, qi - qj
            if sj != si or rj < ctg_off[ci] or not (0 < dr <= MAX_GAP and 0 < dq <= MAX_GAP):
                continue
            sc = f[j] + min(dq, dr, k) - gamma(abs(dr - dq), k)
            if sc > best:
                best, bj = sc, j
        f[i], pred[i] = k + best, bj
    return f, pred


def extract(anc, f, pred, L, k, max_band=MAX_BAND):
    """-> dict(n, f1, f2, strand, W, chain [(q, r)]) of the primary chain, or None without anchors."""
    if not anc:
        return None
    order = sorted(range(len(anc)), key=lambda i: (-f[i], i))
    taken = [False] * len(anc)
    prim, f2 = None, 0
    for e in order:
        if taken[e]:
            continue
        path, i = [], e
        while i >= 0 and not taken[i]:
            taken[i] = True
            path.append(i)
            i = pred[i]
        score = f[e] - (f[i] if i >= 0 else 0)
        qs, qe = anc[path[-1]][2], anc[e][2] + k
        if anc[e][0]:
            qs, qe = L - qe, L - qs
        if prim is None:
            prim = dict(path=path[::-1], f1=score, span=(qs, qe))
        else:
            ps, pe = prim["span"]
            ov = min(pe, qe) - max(ps, qs)
            if ov > 0 and 2 * ov >= min(pe - ps, qe - qs):
                f2 = max(f2, score)
    chain = [(anc[i][2], anc[i][1]) for i in prim["path"]]
    d = [r - q for q, r in chain]
    W = min(64 + max([abs(a - b) for a, b in zip(d[1:], d[:-1])], default=0), max_band)
    return dict(n=len(chain), f1=prim["f1"], f2=f2, strand=anc[prim["path"][0]][0], W=W, chain=chain)


def mapq(f1, f2, n):
    if f2 >= f1:
        return 0
    return min(60, int(math.floor(40 * (1 - f2 / f1) * min(1.0, n / 10) * math.log(f1))))


def centres(chain, m):
    """c(i) for query bases x = 0..m-1 (chain r relative to the target window)."""
    qs = [q for q, _ in chain]
    out = []
    for x in range(m):
        if x <= qs[0]:
            c = chain[0][1] + x - qs[0]
        elif x >= qs[-1]:
            c = chain[-1][1] + x - qs[-1]
        else:
            a = int(np.searchsorted(qs, x, side="right")) - 1
            (qa, ra), (qb, rb) = chain[a], chain[a + 1]
            c = ra + (x - qa) * (rb - ra) // (qb - qa)
        out.append(c)
    return out


def _score(a, b):
    ca, cb = _CODE[a], _CODE[b]
    return np.where((ca < 0) | (cb < 0), -1, np.where(ca == cb, 2, -4))


def band_align(query, target, chain, W):
    """Local affine alignment in the band -> (score, q_st, q_en, t_st, t_en, ops bytes).  Row by row over the band offsets
    0 .. 2W, with E, F and H from the recurrences cell by cell and the traceback bits of every band cell kept."""
    q = np.frombuffer(bytes(query), dtype=np.uint8)
    t = np.frombuffer(bytes(target), dtype=np.uint8)
    m, n = len(q), len(t)
    cen = centres(chain, m)
    B = 2 * W + 1
    b = np.arange(B)
    src = np.zeros((m + 1, B), dtype=np.uint8)
    eob = np.zeros((m + 1, B), dtype=bool)
    fob = np.zeros((m + 1, B), dtype=bool)
    best = (0, 0, 0)
    hp = fp = None
    lo_prev = 0
    for i in range(1, m + 1):
        lo = cen[i - 1] + 1 - W
        j = lo + b
        inb = (j >= 1) & (j <= n)
        if i == 1:
            up_h, up_f, dg = np.zeros(B, np.int64), np.full(B, NEG, np.int64), np.zeros(B, np.int64)
        else:
            ub = b + (lo - lo_prev)
            ok = ub < B
            up_h = np.where(ok, hp[np.minimum(ub, B - 1)], NEG)
            up_f = np.where(ok, fp[np.minimum(ub, B - 1)], NEG)
            okd = (ub - 1 >= 0) & (ub - 1 < B)
            dg = np.where(j == 1, 0, np.where(okd, hp[np.clip(ub - 1, 0, B - 1)], NEG))
        s = np.where(inb, _score(np.full(B, q[i - 1]), t[np.clip(j - 1, 0, n - 1)]), 0)
        d = dg + s
        fo = up_h - 6 >= up_f - 2
        fv = np.where(fo, up_h - 6, up_f - 2)
        # E by the recurrence, cell by cell (on Python lists: the band is up to 8193 cells wide)
        e, eo, h, sr = [NEG] * B, [False] * B, [NEG] * B, [0] * B
        inb_l, j_l, d_l, fv_l = inb.tolist(), j.tolist(), d.tolist(), fv.tolist()
        for x in range(B):
            if not inb_l[x]:
                continue
            if j_l[x] == 1:
                e[x], eo[x] = max(0 - 6, NEG - 2), True
            elif x > 0 and inb_l[x - 1]:
                eo[x] = h[x - 1] - 6 >= e[x - 1] - 2
                e[x] = h[x - 1] - 6 if eo[x] else e[x - 1] - 2
            m3 = max(d_l[x], e[x], fv_l[x])
            if m3 <= 0:
                h[x], sr[x] = 0, 1
            else:
                h[x], sr[x] = m3, (0 if m3 == d_l[x] else (3 if m3 == e[x] else 2))
            if h[x] > 0 and (h[x], i, j_l[x]) > best:
                best = (h[x], i, j_l[x])
        h = np.array(h, dtype=np.int64)
        src[i], eob[i], fob[i] = sr, eo, fo
        hp, fp = h, np.where(inb, fv, NEG)
        lo_prev = lo
    score, ei, ej = best
    if score <= 0:
        return 0, 0, 0, 0, 0, b""
    ops, i, jj, state = [], ei, ej, 0
    while i > 0 and jj > 0:
        x = jj - (cen[i - 1] + 1 - W)
        if state == 0:
            if src[i, x] == 1:
                break
            if src[i, x] == 0:
                ops.append(b"=" if _CODE[q[i - 1]] >= 0 and _CODE[q[i - 1]] == _CODE[t[jj - 1]] else b"X")
                i, jj = i - 1, jj - 1
            else:
                state = 1 if src[i, x] == 3 else 2
        elif state == 1:
            ops.append(b"D")
            if eob[i, x]:
                state = 0
            jj -= 1
        else:
            ops.append(b"I")
            if fob[i, x]:
                state = 0
            i -= 1
    return score, i, ei, jj, ej, b"".join(ops[::-1])


def cigar_nm_md(ops, ref):
    """Walks the op string base by base."""
    cigar, runs = [], []
    for op in ops.decode():
        c = "M" if op in "=X" else op
        if runs and runs[-1][0] == c:
            runs[-1][1] += 1
        else:
            runs.append([c, 1])
    cigar = "".join(f"{n}{c}" for c, n in runs)
    nm = sum(op != "=" for op in ops.decode())
    md, count, r, in_del = "", 0, 0, False
    for op in ops.decode():
        if op == "I":
            continue
        if op == "=":
            count, in_del = count + 1, False
        elif op == "X":
            md += f"{count}{chr(ref[r])}"
            count, in_del = 0, False
        else:
            md += (chr(ref[r]) if in_del else f"{count}^{chr(ref[r])}")
            count, in_del = 0, True
        r += 1
    return cigar, nm, md + str(count)


_COMP = bytes.maketrans(b"ACGT", b"TGCA")


def revcomp(s):
    return bytes(s).translate(_COMP)[::-1]


def map_read(index, read, max_band=MAX_BAND):
    """The whole rule chain for one read -> a tuple (ctg, r_st, r_en, q_st, q_en, strand, mapq, cigar, NM, MD) or None."""
    read = bytes(read).upper()
    L, k = len(read), index.k
    anc = anchors(index, read, k)
    f, pred = chain_dp(anc, index.off, k)
    ch = extract(anc, f, pred, L, k, max_band)
    if ch is None or ch["n"] < 3 or ch["f1"] < 40:
        return None
    W, (q0, r0), (q1, r1) = ch["W"], ch["chain"][0], ch["chain"][-1]
    c = int(np.searchsorted(index.off, r0, side="right")) - 1
    ts = max(int(index.off[c]), r0 - q0 - W)
    te = min(int(index.off[c + 1]), r1 + (L - q1) + W)
    ref = b"".join(index.seqs)
    query = revcomp(read) if ch["strand"] else read
    score, qs, qe, t_st, t_en, ops = band_align(query, ref[ts:te], [(q, r - ts) for q, r in ch["chain"]], W)
    if score <= 0:
        return None
    cigar, nm, md = cigar_nm_md(ops, ref[ts + t_st:ts + t_en])
    if ch["strand"]:
        qs, qe = L - qe, L - qs
    base = ts - int(index.off[c])
    return (index.names[c], base + t_st, base + t_en, qs, qe, -1 if ch["strand"] else 1,
            mapq(ch["f1"], ch["f2"], ch["n"]), cigar, nm, md)


def nm_md_from_cigar(cigar, query, ref):
    """(NM, MD) recomputed from an M / I / D CIGAR, the aligned query bases (reference orientation, clips removed) and the
    reference bases the alignment covers; also checks that the CIGAR consumes exactly both."""
    import re
    ops = []
    qi = ri = 0
    for n, op in re.findall(r"(\d+)([MID])", cigar):
        n = int(n)
        if op == "M":
            ops += [b"=" if query[qi + t] == ref[ri + t] and chr(ref[ri + t]) in "ACGT" else b"X" for t in range(n)]
            qi, ri = qi + n, ri + n
        elif op == "I":
            ops += [b"I"] * n
            qi += n
        else:
            ops += [b"D"] * n
            ri += n
    assert qi == len(query) and ri == len(ref), (cigar, qi, len(query), ri, len(ref))
    _, nm, md = cigar_nm_md(b"".join(ops), ref)
    return nm, md
