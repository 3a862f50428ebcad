"""Numpy restatement of the reference's CPU CTC forced alignment (forced_align/cpu/compute.cpp), vectorised over the
states of each frame: the band [start, end) and its advance rules, the alphas in the input dtype with every add rounded
to it, the strict comparisons (skip only if strictly above both, neighbour only if strictly above both, else stay),
the final state S - 1 only if strictly above S - 2, and the backtrack over the stored pointers (-1 outside the band).

One deviation, shared with the GPU kernel: where the reference's backtrack would climb above the last state (it
follows -1 pointers of states outside the band, possible only when no alignment has a finite score) and read out of
bounds, the state stops at S - 1.  A row with no targets is all blank.

``case_inputs`` and ``batch_inputs`` rebuild the seeded inputs of the recipes stored in
tests/golden/forced_align_ref_cases.npz.
"""
import numpy as np

DTYPES = (np.float32, np.float16, np.float64)  # recipe dtype codes 0, 1, 2
TDTYPES = (np.int32, np.int64)  # recipe target dtype codes 0, 1


def repeats(tg):
    tg = np.asarray(tg)
    return int(np.count_nonzero(tg[1:] == tg[:-1])) if tg.size > 1 else 0


def align(lp, tg, blank):
    """One sequence: lp (T, C) log-probs in their dtype, tg (L,) targets.  Returns (path int64 (T,), scores (T,))."""
    lp = np.asarray(lp)
    tg = np.asarray(tg, dtype=np.int64)
    dt = lp.dtype.type
    T, L = lp.shape[0], tg.size
    S = 2 * L + 1
    if L == 0:
        path = np.full(T, blank, dtype=np.int64)
        return path, lp[np.arange(T), path]
    R = repeats(tg)
    assert T >= L + R
    ninf = dt(-np.inf)
    labels = np.full(S, blank, dtype=np.int64)
    labels[1::2] = tg
    nd = np.zeros(L + 1, dtype=bool)  # nd[j]: targets[j] != targets[j - 1]; nd[0] and nd[L] false
    nd[1:L] = tg[1:] != tg[:-1]
    skip = np.zeros(S, dtype=bool)
    skip[3::2] = nd[1:L]
    bp = np.full((T, S), -1, dtype=np.int8)
    alpha = np.full(S, ninf, dtype=dt)
    start = 0 if T - (L + R) > 0 else 1
    end = 1 if S == 1 else 2
    alpha[start:end] = lp[0, labels[start:end]]
    idx = np.arange(S)
    for t in range(1, T):
        if T - t <= L + R:
            if start % 2 == 1 and nd[start // 2 + 1]:
                start += 1
            start += 1
        if t <= L + R:
            if end % 2 == 0 and end < 2 * L and nd[end // 2]:
                end += 1
            end += 1
        x0 = alpha
        x1 = np.concatenate(([ninf], alpha[:-1]))
        x2 = np.where(skip, np.concatenate(([ninf, ninf], alpha[:-2])), ninf)
        c2 = (x2 > x1) & (x2 > x0)
        c1 = ~c2 & (x1 > x0) & (x1 > x2)
        res = np.where(c2, x2, np.where(c1, x1, x0))
        band = (idx >= start) & (idx < end)
        with np.errstate(invalid="ignore", over="ignore"):
            new = (res + lp[t, labels]).astype(dt)
        alpha = np.where(band, new, ninf).astype(dt)
        bp[t] = np.where(band, np.where(c2, 2, np.where(c1, 1, 0)), -1)
    s = S - 1 if alpha[S - 1] > alpha[S - 2] else S - 2
    path = np.empty(T, dtype=np.int64)
    for t in range(T - 1, -1, -1):
        path[t] = labels[s]
        s = min(s - int(bp[t, s]), S - 1)
    return path, lp[np.arange(T), path]


def align_batch(lp, tg, tl, ul, blank):
    """Rows aligned alone; frames t >= T_b get path blank and score 0."""
    B, T, _ = lp.shape
    paths = np.full((B, T), blank, dtype=np.int64)
    scores = np.zeros((B, T), dtype=lp.dtype)
    for b in range(B):
        p, s = align(lp[b, : tl[b]], tg[b, : ul[b]], blank)
        paths[b, : tl[b]] = p
        scores[b, : tl[b]] = s
    return paths, scores


def _emission(rng, T, C, kind, dt):
    """kind 0: log-softmax of N(0, 2); 1: a coarse grid of negative multiples of 0.5 (ties everywhere); 2: as 0 with
    every third class masked to -inf (the caller keeps targets off them)."""
    if kind == 1:
        return (-0.5 * rng.integers(0, 4, size=(T, C))).astype(dt)
    x = 2.0 * rng.standard_normal((T, C))
    x = x - x.max(axis=1, keepdims=True)
    x = x - np.log(np.exp(x).sum(axis=1, keepdims=True))
    if kind == 2:
        x[:, 2::3] = -np.inf
    return x.astype(dt)


def _targets(rng, L, C, blank, kind, heavy):
    allowed = np.array([c for c in range(C) if c != blank and not (kind == 2 and c % 3 == 2)])
    if heavy:
        allowed = allowed[:2]
    return rng.choice(allowed, size=L)


def case_inputs(rc):
    """rc = (seed, T, L, C, blank, dtype, tdtype, kind, heavy); T == 0 means T = L + R exactly."""
    seed, T, L, C, blank, dtc, tdc, kind, heavy = (int(v) for v in rc)
    rng = np.random.default_rng(seed)
    tg = _targets(rng, L, C, blank, kind, heavy)
    if T == 0:
        T = L + repeats(tg)
    lp = _emission(rng, T, C, kind, DTYPES[dtc])
    return lp[None], tg[None].astype(TDTYPES[tdc]), blank


def batch_inputs(rc):
    """rc = (seed, B, T, L, C, blank, dtype, tdtype, kind, heavy): ragged lengths with max(T_b) = T, max(L_b) = L."""
    seed, B, T, L, C, blank, dtc, tdc, kind, heavy = (int(v) for v in rc)
    rng = np.random.default_rng(seed)
    ul = rng.integers(1, L + 1, size=B)
    ul[rng.integers(B)] = L
    tg = np.stack([_targets(rng, L, C, blank, kind, heavy) for _ in range(B)])
    need = np.array([ul[b] + repeats(tg[b, : ul[b]]) for b in range(B)])
    assert need.max() <= T, (need, T)
    tl = np.array([rng.integers(n, T + 1) for n in need])
    tl[rng.integers(B)] = T
    lp = _emission(rng, B * T, C, kind, DTYPES[dtc]).reshape(B, T, C)
    return lp, tg.astype(TDTYPES[tdc]), tl.astype(np.int64), ul.astype(np.int64), blank
