"""Float64 restatement of lfilter / filtfilt and their VJPs (reference functional/filtering.py:926-1099).

The filter runs on the FLOAT32-normalised coefficients a^ = a / a0, b^ = b / a0 (one float32 division each, as the
reference normalises), promoted to float64: an oracle on the exact design would measure the coefficient rounding, not
the recurrence.  Arrays are (..., n_filters, T) with (n_filters, n_order) coefficients, or (..., T) with 1-D ones.
"""
import numpy as np
from scipy import signal


def normalise(a, b):
    a32, b32 = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return (a32 / a32[..., :1]).astype(np.float64), (b32 / a32[..., :1]).astype(np.float64)


def _per_filter(fn, x, a):
    """fn(x_rows (..., T), filter index) over the filter axis of x for 2-D coefficients."""
    if np.ndim(a) == 1:
        return fn(x, None)
    return np.stack([fn(x[..., f, :], f) for f in range(a.shape[0])], axis=-2)


def _iir(x, ah, bh, reverse=False):
    x = np.asarray(x, np.float64)
    if reverse:
        return signal.lfilter(bh, ah, x[..., ::-1], axis=-1)[..., ::-1]
    return signal.lfilter(bh, ah, x, axis=-1)


def lfilter(x, a, b, clamp=True, reverse=False):
    """y (float64) of b200a_lfilter_run; ``reverse`` runs the recurrence from the last sample down."""
    ah, bh = normalise(a, b)
    y = _per_filter(lambda xr, f: _iir(xr, ah if f is None else ah[f], bh if f is None else bh[f], reverse), x, ah)
    return np.clip(y, -1.0, 1.0) if clamp else y


def filtfilt(x, a, b, clamp=True):
    return lfilter(lfilter(x, a, b, clamp=False), a, b, clamp=clamp, reverse=True)


def _lag(z, k, reverse):
    """z[t - k] (z[t + k] when reverse) along the last axis, zero outside."""
    out = np.zeros_like(z)
    if k == 0:
        return z.copy()
    if reverse:
        out[..., :-k] = z[..., k:]
    else:
        out[..., k:] = z[..., :-k]
    return out


def lfilter_vjp(x, a, b, g, clamp=True, reverse=False):
    """(dx, da, db) of sum(g * lfilter(x, a, b, clamp, reverse)) in float64; da and db are for the RAW coefficients,
    summed over the leading dimensions.  The clamp's gradient is torch.clamp's: g where -1 <= y <= 1."""
    a = np.asarray(a, np.float32)
    one_d = a.ndim == 1
    ah, bh = normalise(a, b)
    if one_d:
        ah, bh, a = ah[None], bh[None], a[None]
        x, g = np.asarray(x)[..., None, :], np.asarray(g)[..., None, :]
    x = np.asarray(x, np.float64)
    g = np.asarray(g, np.float64)
    n_f, n = ah.shape
    dx = np.zeros(np.broadcast_shapes(x.shape, g.shape))
    dah, dbh = np.zeros((n_f, n)), np.zeros((n_f, n))
    for f in range(n_f):
        xf, gf = x[..., f, :], g[..., f, :]
        yf = _iir(xf, ah[f], bh[f], reverse)
        gy = gf * ((yf >= -1) & (yf <= 1)) if clamp else gf
        u = _iir(gy, ah[f], np.array([1.0]), not reverse)  # the IIR adjoint runs the other way
        dx[..., f, :] = sum(bh[f][k] * _lag(u, k, not reverse) for k in range(n))
        for k in range(n):
            dah[f, k] = -np.sum(u * _lag(yf, k, reverse))
            dbh[f, k] = np.sum(u * _lag(xf, k, reverse))
    a0 = a[:, :1].astype(np.float64)
    da = dah / a0
    db = dbh / a0
    da[:, 0] = -(np.sum(dah[:, 1:] * ah[:, 1:], axis=1) + np.sum(dbh * bh, axis=1)) / a0[:, 0]
    if one_d:
        return dx[..., 0, :], da[0], db[0]
    return dx, da, db


def filtfilt_vjp(x, a, b, g, clamp=True):
    """(dx, da, db) of sum(g * filtfilt(x, a, b, clamp)): the two passes' VJPs chained."""
    mid = lfilter(x, a, b, clamp=False)
    d_mid, da2, db2 = lfilter_vjp(mid, a, b, g, clamp=clamp, reverse=True)
    dx, da1, db1 = lfilter_vjp(x, a, b, d_mid, clamp=False)
    return dx, da1 + da2, db1 + db2


# the defaults of each *_biquad after the sample rate (reference filtering.py), and the design helper's argument order
_BIQUAD_ARGS = {
    "allpass": (("central_freq", None), ("Q", 0.707)),
    "band": (("central_freq", None), ("Q", 0.707), ("noise", False)),
    "bandpass": (("central_freq", None), ("Q", 0.707), ("const_skirt_gain", False)),
    "bandreject": (("central_freq", None), ("Q", 0.707)),
    "bass": (("gain", None), ("central_freq", 100), ("Q", 0.707)),
    "equalizer": (("center_freq", None), ("gain", None), ("Q", 0.707)),
    "highpass": (("cutoff_freq", None), ("Q", 0.707)),
    "lowpass": (("cutoff_freq", None), ("Q", 0.707)),
    "treble": (("gain", None), ("central_freq", 3000), ("Q", 0.707)),
}


def biquad_coeffs(name, sample_rate, kwargs, device="cpu"):
    """(a, b) float32 numpy arrays of audio_b200's design of ``{name}_biquad`` evaluated on ``device``."""
    import torch

    from audio_b200 import _filtering

    fn = getattr(_filtering, f"_design_{name}")
    if name in ("deemph", "riaa"):
        b, a = fn(sample_rate)
    else:
        args = [kwargs.get(k, d) for k, d in _BIQUAD_ARGS[name]]
        b, a = fn(sample_rate, *args, torch.float32, device)
    as32 = lambda cs: np.array([float(c) for c in cs], dtype=np.float32)  # noqa: E731
    return as32(a), as32(b)
