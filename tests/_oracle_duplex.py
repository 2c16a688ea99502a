"""
CPU oracle of b200_pair_align (bonito_b200/csrc/pair_align.cu): full-matrix dynamic programming with an explicit
traceback under the same rules, written for clarity, not speed (numpy rows, a Python walk).

  global_edit(q, r)        -> (distance, ops)   unit cost; ties: diagonal, then I, then D
  semiglobal_affine(q, r)  -> (score, ops)      +5 / -4, gap 10 + 2 (g - 1), free end gaps, ops cover both sequences

ops: one char per op in forward order, '=' 'X' 'I' (consumes q) 'D' (consumes r).
"""

import numpy as np

NEG = -(1 << 30)


def _codes(s):
    return np.frombuffer(s.encode() if isinstance(s, str) else bytes(s), dtype=np.uint8)


def global_edit(q, r):
    qa, ra = _codes(q), _codes(r)
    m, n = len(qa), len(ra)
    D = np.zeros((m + 1, n + 1), dtype=np.int64)
    D[0, :] = np.arange(n + 1)
    D[:, 0] = np.arange(m + 1)
    for i in range(1, m + 1):
        sub = (ra != qa[i - 1]).astype(np.int64)
        for j in range(1, n + 1):
            D[i, j] = min(D[i - 1, j - 1] + sub[j - 1], D[i - 1, j] + 1, D[i, j - 1] + 1)
    ops = []
    i, j = m, n
    while i > 0 and j > 0:
        x = int(qa[i - 1] != ra[j - 1])
        if D[i, j] == D[i - 1, j - 1] + x:
            ops.append("X" if x else "=")
            i, j = i - 1, j - 1
        elif D[i, j] == D[i - 1, j] + 1:
            ops.append("I")
            i -= 1
        else:
            ops.append("D")
            j -= 1
    ops.extend("I" * i)
    ops.extend("D" * j)
    return int(D[m, n]), "".join(reversed(ops))


def semiglobal_affine(q, r):
    qa, ra = _codes(q), _codes(r)
    m, n = len(qa), len(ra)
    if m == 0 or n == 0:
        return 0, "I" * m + "D" * n
    H = np.zeros((m + 1, n + 1), dtype=np.int64)
    E = np.full((m + 1, n + 1), NEG, dtype=np.int64)
    F = np.full((m + 1, n + 1), NEG, dtype=np.int64)
    Eo = np.zeros((m + 1, n + 1), dtype=bool)
    Fo = np.zeros((m + 1, n + 1), dtype=bool)
    src = np.zeros((m + 1, n + 1), dtype=np.int8)        # 0 '=', 1 'X', 2 F, 3 E
    for i in range(1, m + 1):
        for j in range(1, n + 1):
            eo, ee = H[i, j - 1] - 10, E[i, j - 1] - 2
            E[i, j], Eo[i, j] = (eo, True) if eo >= ee else (ee, False)
            fo, fe = H[i - 1, j] - 10, F[i - 1, j] - 2
            F[i, j], Fo[i, j] = (fo, True) if fo >= fe else (fe, False)
            match = qa[i - 1] == ra[j - 1]
            d = H[i - 1, j - 1] + (5 if match else -4)
            h = max(d, E[i, j], F[i, j])
            H[i, j] = h
            src[i, j] = (0 if match else 1) if h == d else (3 if h == E[i, j] else 2)
    # end cell: max over row m and column n, ties to the largest i, then the largest j
    cands = [(H[m, j], m, j) for j in range(n + 1)] + [(H[i, n], i, n) for i in range(m)]
    score, ei, ej = max(cands)
    ops = ["D"] * (n - ej) if ei == m else ["I"] * (m - ei)
    i, j, state = ei, ej, "H"
    while i > 0 and j > 0:
        if state == "H":
            s = src[i, j]
            if s < 2:
                ops.append("X" if s else "=")
                i, j = i - 1, j - 1
            else:
                state = "E" if s == 3 else "F"
        elif state == "E":
            ops.append("D")
            if Eo[i, j]:
                state = "H"
            j -= 1
        else:
            ops.append("I")
            if Fo[i, j]:
                state = "H"
            i -= 1
    ops.extend("I" * i)
    ops.extend("D" * j)
    return int(score), "".join(reversed(ops))


def check_ops(q, r, ops):
    """The op string consumes q and r exactly, and =/X agree with the bases."""
    i = j = 0
    for op in ops:
        if op in "=X":
            assert (q[i] == r[j]) == (op == "="), (i, j, op)
            i, j = i + 1, j + 1
        elif op == "I":
            i += 1
        else:
            assert op == "D", op
            j += 1
    assert (i, j) == (len(q), len(r))


def edit_cost(ops):
    return sum(op != "=" for op in ops)


def affine_score(ops):
    """Score of an op string under SEMIGLOBAL_AFFINE, with the leading and trailing gap runs free."""
    body = ops.strip("ID")
    score, prev = 0, None
    for op in body:
        if op == "=":
            score += 5
        elif op == "X":
            score -= 4
        else:
            score -= 2 if op == prev else 10
        prev = op
    return score
