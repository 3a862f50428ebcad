"""Float64 numpy restatement of the reference's CPU RNN-T loss (rnnt/cpu/cpu_kernels.h): costs -beta(0, 0) and the
fused and non-fused logit gradients, with the reference's lse (so the lse of two -inf is NaN), its clamp to
[-clamp, clamp] and, for a sequence whose cost is not finite, a zero gradient (what the reference's CUDA path writes;
its CPU path writes NaN there).  The alpha / beta recursions run along anti-diagonals, vectorised over each diagonal.

``case_inputs`` rebuilds the seeded inputs of a recipe stored in tests/golden/rnnt_loss_ref_cases.npz."""
import numpy as np


def lse(x, y):
    with np.errstate(invalid="ignore", over="ignore"):
        return np.where(y > x, y + np.log1p(np.exp(x - y)), x + np.log1p(np.exp(y - x)))


def _log_probs(lg, tgt, blank, fused):
    """(skip, emit, denom) of one sequence's valid block lg (T, U, V); emit is (T, U - 1)."""
    T, U, _ = lg.shape
    if fused:
        m = lg.max(axis=-1)
        with np.errstate(invalid="ignore", divide="ignore"):
            denom = m + np.log(np.exp(lg - m[..., None]).sum(axis=-1))
    else:
        denom = np.zeros((T, U))
    skip = lg[:, :, blank] - denom
    u = np.arange(U - 1)
    emit = lg[:, u, tgt[: U - 1]] - denom[:, : U - 1]
    return skip, emit, denom


def _alpha(skip, emit):
    T, U = skip.shape
    a = np.zeros((T, U))
    for n in range(1, T + U - 1):
        u = np.arange(max(0, n - T + 1), min(n, U - 1) + 1)
        t = n - u
        top = np.where(t > 0, a[np.maximum(t - 1, 0), u] + skip[np.maximum(t - 1, 0), u], 0.0)
        left = np.where(u > 0, a[t, np.maximum(u - 1, 0)] + emit[t, np.maximum(u - 1, 0)] if U > 1 else 0.0, 0.0)
        a[t, u] = np.where(u == 0, top, np.where(t == 0, left, lse(top, left)))
    return a


def _beta(skip, emit):
    T, U = skip.shape
    b = np.zeros((T, U))
    b[T - 1, U - 1] = skip[T - 1, U - 1]
    for n in range(T + U - 3, -1, -1):
        u = np.arange(max(0, n - T + 1), min(n, U - 1) + 1)
        t = n - u
        tn, un = np.minimum(t + 1, T - 1), np.minimum(u + 1, U - 1)
        down = b[tn, u] + skip[t, u]
        right = b[t, un] + (emit[t, np.minimum(u, U - 2)] if U > 1 else 0.0)
        b[t, u] = np.where(u == U - 1, down, np.where(t == T - 1, right, lse(down, right)))
    return b


def _clamp(g, clamp):
    if clamp > 0:
        g = np.where(g > clamp, clamp, g)
        g = np.where(g > -clamp, g, -clamp)
    return g


def sequence(lg, tgt, blank, clamp, fused, grads=True):
    """cost and gradient (T, U, V) of one sequence's valid block lg (float64)."""
    T, U, V = lg.shape
    skip, emit, denom = _log_probs(lg, tgt, blank, fused)
    a, b = _alpha(skip, emit), _beta(skip, emit)
    cost = -b[0, 0]
    if not grads:
        return cost, None
    if not np.isfinite(cost):
        return cost, np.zeros_like(lg)
    tgt = np.asarray(tgt[: U - 1], dtype=np.int64)
    b_next_t = np.vstack([b[1:], np.full((1, U), np.nan)])  # beta(t + 1, u)
    b_next_u = np.hstack([b[:, 1:], np.full((T, 1), np.nan)])  # beta(t, u + 1)
    with np.errstate(invalid="ignore", over="ignore"):
        if fused:
            g = lg + (a + cost - denom)[..., None]
            out = np.exp(g + b[..., None])
            gb = g[:, :, blank]
            blank_val = out[:, :, blank].copy()
            blank_val[: T - 1] -= np.exp(gb[: T - 1] + b_next_t[: T - 1])
            blank_val[T - 1, U - 1] -= np.exp(gb[T - 1, U - 1])
            blank_set = np.zeros((T, U), bool)
            blank_set[: T - 1] = True
            blank_set[T - 1, U - 1] = True
            for u in range(U - 1):
                k = tgt[u]
                rows = ~blank_set[:, u] if k == blank else np.ones(T, bool)
                out[rows, u, k] = out[rows, u, k] - np.exp(g[rows, u, k] + b_next_u[rows, u])
            out[:, :, blank] = np.where(blank_set, blank_val, out[:, :, blank])
        else:
            out = np.full(lg.shape, -0.0)
            g = lg + cost
            blank_set = np.zeros((T, U), bool)
            blank_set[: T - 1] = True
            blank_set[T - 1, U - 1] = True
            bv = g[:, :, blank] + a + np.where(np.arange(T)[:, None] < T - 1, b_next_t, 0.0)
            for u in range(U - 1):
                k = tgt[u]
                rows = ~blank_set[:, u] if k == blank else np.ones(T, bool)
                out[rows, u, k] = -np.exp(g[rows, u, k] + a[rows, u] + b_next_u[rows, u])
            out[:, :, blank] = np.where(blank_set, -np.exp(bv), out[:, :, blank])
    return cost, _clamp(out, clamp)


def rnnt_loss(logits, targets, logit_lengths, target_lengths, blank=-1, clamp=-1.0, fused=True, grads=True):
    """Costs (B,) and unscaled gradients (B, maxT, maxU, V), zero outside each sequence's (T, U) block."""
    lg = np.asarray(logits, dtype=np.float64)
    B, _, _, V = lg.shape
    blank = blank + V if blank < 0 else blank
    costs = np.zeros(B)
    grad = np.zeros_like(lg) if grads else None
    for i in range(B):
        T, U = int(logit_lengths[i]), int(target_lengths[i]) + 1
        costs[i], g = sequence(lg[i, :T, :U], np.asarray(targets[i]), blank, clamp, fused, grads)
        if grads:
            grad[i, :T, :U] = g
    return costs, grad


def case_inputs(recipe):
    """(logits float32 or float16, targets, logit_lengths, target_lengths) of a recipe (seed, B, maxT, maxU, V, blank,
    is_half, scale): ragged lengths in [75 %, 100 %] of the maximum with one sequence at it, targets avoid the blank."""
    seed, B, max_t, max_u, V, blank, is_half = (int(v) for v in recipe[:7])
    scale = float(recipe[7])
    rng = np.random.default_rng(seed)
    logits = (rng.standard_normal((B, max_t, max_u, V)) * scale).astype(np.float16 if is_half else np.float32)
    tl = rng.integers(int(np.ceil(0.75 * max_t)), max_t + 1, size=B).astype(np.int32)
    ul = rng.integers(int(np.ceil(0.75 * (max_u - 1))), max_u, size=B).astype(np.int32)
    tl[0], ul[-1] = max_t, max_u - 1
    tl = np.maximum(tl, 1)
    b = blank + V if blank < 0 else blank
    tg = rng.integers(0, max(V - 1, 1), size=(B, max_u - 1)).astype(np.int32)
    if V > 1:
        tg = tg + (tg >= b)
    return logits, tg, tl, ul
