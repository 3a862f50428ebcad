"""Float64 numpy restatement of the RNN-T feature chain (pipelines/rnnt_pipeline.py:16-23, :35-47, :310-343) and its
vector-Jacobian product, on top of oracle/frontend_oracle.mel_spectrogram and grad_oracle.mel_spectrogram_vjp.

The chain is the reference's, not a cleaned-up one: ``_piecewise_linear_log`` writes ``x`` in place in two statements
and reads the second mask after the first write, so it has three pieces --

    y = x / e        for x <= e
    y = log(x) / e   for e < x <= e^e
    y = log(x)       for x > e^e

-- and jumps at x = e (1 -> 1/e) and at x = e^e (1 -> e).  The model weights were trained on exactly this.  The
pieces can be decided in float32 (``pieces32``, what the reference's float32 run and the kernels decide:
x = fl32(m * fl32(gain)), x > fl32(e), then logf(x) <= fl32(e)) or in float64 (``pieces64``)."""
import math

import numpy as np

from oracle.frontend_oracle import mel_spectrogram

from grad_oracle import mel_spectrogram_vjp

GAIN = pow(10, 0.05 * (2 * 20 * math.log10(32767)))  # rnnt_pipeline.py:16-17, 32767^2 up to rounding
E32 = np.float32(math.e)
GAIN32 = np.float32(GAIN)
MEL_ARGS = dict(sample_rate=16000, n_fft=400, hop_length=160, n_mels=80)


def pieces32(m) -> np.ndarray:
    """Branch of each mel value with the decisions in float32: 1, 2, 3 as above, 0 for a NaN (neither mask)."""
    x = np.asarray(m, dtype=np.float32) * GAIN32
    with np.errstate(divide="ignore", invalid="ignore"):
        lx = np.log(x)
    big = x > E32
    y = np.where(big, lx, x)
    small = y <= E32
    return np.where(small, np.where(big, 2, 1), np.where(big, 3, 0)).astype(np.int8)


def pieces64(m) -> np.ndarray:
    """The same decisions taken in float64 on m * gain."""
    x = np.asarray(m, dtype=np.float64) * GAIN
    with np.errstate(divide="ignore", invalid="ignore"):
        lx = np.log(x)
    big = x > math.e
    y = np.where(big, lx, x)
    small = y <= math.e
    return np.where(small, np.where(big, 2, 1), np.where(big, 3, 0)).astype(np.int8)


def chain(m, mean, invstd, pieces=None) -> np.ndarray:
    """(..., n_mels) mel values -> (m * gain, piecewise log, (y - mean) * invstd) in float64 on the given pieces
    (default: float64 decisions)."""
    m = np.asarray(m, dtype=np.float64)
    p = pieces64(m) if pieces is None else pieces
    x = m * GAIN
    with np.errstate(divide="ignore", invalid="ignore"):
        lx = np.log(x)
    y = np.select([p == 1, p == 2, p == 3], [x / math.e, lx / math.e, lx], x)
    return (y - np.asarray(mean, np.float64)) * np.asarray(invstd, np.float64)


def chain_vjp(m, g, invstd, pieces=None) -> np.ndarray:
    """d/dm of sum(g * chain(m)): g * invstd * gain times 1/e (piece 1), 1/(x e) (piece 2), 1/x (piece 3), 1 (NaN)."""
    m = np.asarray(m, dtype=np.float64)
    p = pieces64(m) if pieces is None else pieces
    x = m * GAIN
    with np.errstate(divide="ignore", invalid="ignore"):
        d = np.select([p == 1, p == 2, p == 3], [1.0 / math.e, 1.0 / (x * math.e), 1.0 / x], 1.0)
    return np.asarray(g, np.float64) * np.asarray(invstd, np.float64) * GAIN * d


def features(x, mean, invstd, fb, right_padding=0, pieces=None) -> np.ndarray:
    """The extractor on (..., L) waveforms: (..., T + right_padding, n_mels), zero padding rows."""
    mel = np.swapaxes(mel_spectrogram(np.asarray(x, np.float64), fb=fb, **MEL_ARGS), -1, -2)
    y = chain(mel, mean, invstd, pieces)
    if right_padding:
        pad = [(0, 0)] * (y.ndim - 2) + [(0, right_padding), (0, 0)]
        y = np.pad(y, pad)
    return y


def features_vjp(x, g, mean, invstd, fb, pieces=None) -> np.ndarray:
    """Gradient of sum(g * features(x)) with respect to x; g: (..., T [+ padding rows], n_mels)."""
    mel = np.swapaxes(mel_spectrogram(np.asarray(x, np.float64), fb=fb, **MEL_ARGS), -1, -2)
    t = mel.shape[-2]
    g_mel = chain_vjp(mel, np.asarray(g)[..., :t, :], invstd, pieces)
    return mel_spectrogram_vjp(x, np.swapaxes(g_mel, -1, -2), fb=fb, **MEL_ARGS)
