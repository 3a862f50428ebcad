"""Float64 restatement of fftconvolve and its VJPs (reference functional/functional.py:2189-2258).

The forward is the full linear convolution of the broadcast operands, sliced as ``_apply_convolve_mode`` slices it;
the VJPs are correlations of the upstream gradient (placed at its offset in the full range) with the other operand,
summed over the rows that broadcasting shared.  ``scipy.signal.fftconvolve`` in float64 evaluates the long cases;
``direct=True`` runs ``np.convolve`` per row instead.
"""
import numpy as np
from scipy import signal


def convolve_slice(n, m, mode):
    """(start, length) of the mode's slice of the (n + m - 1)-sample full result, with Python's slice rules."""
    full = n + m - 1
    if mode == "full":
        return 0, full
    target = max(n, m) - min(n, m) + 1 if mode == "valid" else n
    start = (full - target) // 2
    lo, hi, _ = slice(start, start + target).indices(full)
    return lo, max(hi - lo, 0)


def _rows(fn, x, y):
    lead = np.broadcast_shapes(x.shape[:-1], y.shape[:-1])
    xb = np.broadcast_to(x, lead + x.shape[-1:]).reshape(-1, x.shape[-1])
    yb = np.broadcast_to(y, lead + y.shape[-1:]).reshape(-1, y.shape[-1])
    out = np.stack([fn(a, b) for a, b in zip(xb, yb)]) if xb.shape[0] else np.zeros((0, 0))
    return out.reshape(lead + out.shape[-1:])


def full(x, y, direct=False):
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    if direct:
        return _rows(np.convolve, x, y)
    return signal.fftconvolve(x, y, axes=-1)


def fftconvolve(x, y, mode="full", direct=False):
    x, y = np.asarray(x), np.asarray(y)
    start, length = convolve_slice(x.shape[-1], y.shape[-1], mode)
    return full(x, y, direct)[..., start:start + length]


def _sum_to(g, shape):
    """Sum the broadcast leading dimensions of g back to ``shape`` (autograd's reduction of an expand)."""
    lead = len(g.shape) - len(shape)
    g = g.sum(axis=tuple(range(lead))) if lead else g
    axes = tuple(i for i, s in enumerate(shape) if s == 1 and g.shape[i] != 1)
    return g.sum(axis=axes, keepdims=True) if axes else g


def vjp(x, y, g, mode="full", direct=False):
    """(dx, dy) of sum(g * fftconvolve(x, y, mode)):  dx[k] = sum_j gf[k + j] y[j],  dy[j] = sum_k gf[k + j] x[k]."""
    x, y, g = np.asarray(x, np.float64), np.asarray(y, np.float64), np.asarray(g, np.float64)
    n, m = x.shape[-1], y.shape[-1]
    start, length = convolve_slice(n, m, mode)
    gf = np.zeros(g.shape[:-1] + (n + m - 1,))
    gf[..., start:start + length] = g
    if direct:
        dx = _rows(lambda a, b: np.correlate(a, b, "valid"), gf, np.broadcast_to(y, gf.shape[:-1] + (m,)))
        dy = _rows(lambda a, b: np.correlate(a, b, "valid"), gf, np.broadcast_to(x, gf.shape[:-1] + (n,)))
    else:
        dx = signal.fftconvolve(gf, y[..., ::-1], mode="valid", axes=-1)
        dy = signal.fftconvolve(gf, x[..., ::-1], mode="valid", axes=-1)
    return _sum_to(dx, x.shape), _sum_to(dy, y.shape)
