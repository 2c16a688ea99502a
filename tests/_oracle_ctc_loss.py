"""
Float64 numpy CTC loss with explicit alpha and beta, and the gradient in torch's form (torch's CPU ctc_loss_backward):
  grad[t, n, c] = (exp(lp[t, n, c]) - exp(lcab[t, n, c] + nll[n] - lp[t, n, c])) * g[n] for t < input_lengths[n], else 0,
with lcab the log-sum over the states of class c of alpha + beta (beta includes lp[t] like alpha).  Non-finite values come
out where torch's do: an infeasible sample has nll = inf and NaN on every frame before its input length.

`cases()` lists the shapes the CPU and GPU tests share.
"""
import numpy as np


def _lse(*xs):
    x = np.stack(xs)
    m = x.max(axis=0)
    ms = np.where(np.isfinite(m), m, 0.0)
    with np.errstate(divide="ignore"):
        return np.log(np.exp(x - ms).sum(axis=0)) + ms


def sample(lp, target, blank):
    """lp [T_n, C] float64 of one sample (its first input_length frames), target: its labels -> nll, grad [T_n, C] (g=1)."""
    T, C = lp.shape
    L = len(target)
    S = 2 * L + 1
    cls = np.full(S, blank, dtype=np.int64)
    cls[1::2] = target
    skip = np.zeros(S, dtype=bool)               # s may be entered from s - 2
    skip[3::2] = np.asarray(target[1:]) != np.asarray(target[:-1]) if L > 1 else False
    ninf = np.full(S, -np.inf)
    alpha = np.full((T, S), -np.inf)
    alpha[0, 0] = lp[0, blank]
    if L > 0:
        alpha[0, 1] = lp[0, target[0]]
    for t in range(1, T):
        a = alpha[t - 1]
        a1 = np.concatenate([[-np.inf], a[:-1]])
        a2 = np.where(skip, np.concatenate([[-np.inf, -np.inf], a])[:S], ninf)
        alpha[t] = lp[t, cls] + _lse(a, a1, a2)
    beta = np.full((T, S), -np.inf)
    beta[T - 1, S - 1] = lp[T - 1, blank]
    if L > 0:
        beta[T - 1, S - 2] = lp[T - 1, target[-1]]
    skip_out = np.concatenate([skip[2:], [False, False]])[:S]      # s may leave to s + 2
    for t in range(T - 2, -1, -1):
        b = beta[t + 1]
        b1 = np.concatenate([b[1:], [-np.inf]])
        b2 = np.where(skip_out, np.concatenate([b[2:], [-np.inf, -np.inf]])[:S], ninf)
        beta[t] = lp[t, cls] + _lse(b, b1, b2)
    nll = -_lse(alpha[T - 1, S - 1], alpha[T - 1, S - 2] if L > 0 else -np.inf)
    lcab = np.full((T, C), -np.inf)
    ab = alpha + beta
    for c in range(C):
        sel = cls == c
        if sel.any():
            lcab[:, c] = _lse(*ab[:, sel].T)
    with np.errstate(invalid="ignore", over="ignore"):
        grad = np.exp(lp) - np.exp(lcab + nll - lp)
    return float(nll), grad


def ctc_loss(log_probs, targets, input_lengths, target_lengths, blank=0):
    """log_probs [T, N, C] float64; targets padded [N, S] or concatenated 1-D -> (nll [N], grad [T, N, C]) with g = 1."""
    lp = np.asarray(log_probs, dtype=np.float64)
    T, N, C = lp.shape
    targets = np.asarray(targets)
    nll = np.zeros(N)
    grad = np.zeros((T, N, C))
    off = 0
    for n in range(N):
        il, tl = int(input_lengths[n]), int(target_lengths[n])
        tgt = targets[n, :tl] if targets.ndim == 2 else targets[off:off + tl]
        off += tl
        nll[n], grad[:il, n] = sample(lp[:il, n], [int(x) for x in tgt], blank)
    return nll, grad


def repeats(target):
    return int(sum(a == b for a, b in zip(target[:-1], target[1:])))


def case(name, T, N, C, input_lengths, targets, blank=0, concat=False, seed=0, scale=2.0):
    """One test case: targets is a list of label lists; log-probs are a seeded log_softmax of N(0, scale^2) logits."""
    rng = np.random.default_rng(seed)
    lp = rng.normal(0.0, scale, (T, N, C))
    lp = lp - np.log(np.exp(lp - lp.max(-1, keepdims=True)).sum(-1, keepdims=True)) - lp.max(-1, keepdims=True)
    tl = np.array([len(t) for t in targets], dtype=np.int64)
    if concat:
        tg = np.array([x for t in targets for x in t], dtype=np.int64)
    else:
        tg = np.zeros((N, max(1, int(tl.max()) if N else 1)), dtype=np.int64)
        for n, t in enumerate(targets):
            tg[n, :len(t)] = t
    return dict(name=name, log_probs=lp, targets=tg, input_lengths=np.asarray(input_lengths, dtype=np.int64),
                target_lengths=tl, blank=blank)


def _random_targets(rng, N, lo, hi, C, blank):
    labels = [c for c in range(C) if c != blank]
    return [list(rng.choice(labels, size=int(rng.integers(lo, hi + 1)))) for _ in range(N)]


def cases():
    """The shared cases: reductions and zero_infinity are applied to each by the tests."""
    rng = np.random.default_rng(1234)
    out = []
    # mixed input lengths (1 .. T) and target lengths in one batch, padded and concatenated
    T, N = 40, 6
    tg = _random_targets(rng, N, 0, 12, 5, 0)
    tg[0], tg[1] = [], [2]
    il = [T, 1, 17, T, 33, 25]
    for concat in (False, True):
        out.append(case(f"mixed_{'concat' if concat else 'padded'}", T, N, 5, il, tg, concat=concat, seed=1))
    # input length 1: empty target, one label, one label too many
    out.append(case("input_length_1", 3, 3, 5, [1, 1, 1], [[], [4], [1, 2]], seed=2))
    # repeats and the feasibility boundary: T = L + repeats feasible, one frame below infeasible
    rep = [1, 1, 2, 2, 2, 3, 1, 4, 4]
    need = len(rep) + repeats(rep)
    out.append(case("feasibility_boundary", need + 3, 4, 5, [need, need - 1, need + 3, need], [rep, rep, rep, [1, 2, 3]],
                    seed=3))
    # blank other than 0, and the last class
    out.append(case("blank_2", 30, 4, 5, [30, 30, 21, 9], _random_targets(rng, 4, 1, 9, 5, 2), blank=2, seed=4))
    out.append(case("blank_last", 30, 3, 5, [30, 25, 30], _random_targets(rng, 3, 1, 9, 5, 4), blank=4, seed=5,
                    concat=True))
    # C at the limit
    out.append(case("classes_256", 24, 3, 256, [24, 24, 20], _random_targets(rng, 3, 1, 10, 256, 0), seed=6))
    out.append(case("classes_256_blank_255", 24, 2, 256, [24, 19], _random_targets(rng, 2, 1, 8, 256, 255),
                    blank=255, seed=7))
    # peaked log-probs (scale 8): many entries far below 0, long chain of frames
    out.append(case("peaked", 200, 3, 5, [200, 150, 100], _random_targets(rng, 3, 20, 60, 5, 0), seed=8, scale=8.0))
    return out
