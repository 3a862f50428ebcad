"""Float64 oracle of InverseMelScale (reference transforms/_transforms.py:418-503) and of its input gradient.

The forward is a dense minimum-norm least-squares solve with numpy (``numpy.linalg.lstsq``, SVD based), deliberately
not the banded factorisation the kernel uses.  For a full-rank underdetermined system it is the answer of every LAPACK
driver the reference offers."""
import numpy as np


def inverse_mel_scale(mel, fb):
    """relu(lstsq(fb^T, mel).solution): (..., n_mels, T) -> (..., n_stft, T), float64."""
    fb = np.asarray(fb, dtype=np.float64)
    mel = np.asarray(mel, dtype=np.float64)
    lead, (n_mels, frames) = mel.shape[:-2], mel.shape[-2:]
    m2 = np.moveaxis(mel.reshape(-1, n_mels, frames), 1, 0).reshape(n_mels, -1)
    x = np.linalg.lstsq(fb.T, m2, rcond=None)[0]
    x = np.moveaxis(x.reshape(fb.shape[0], -1, frames), 0, 1)
    return np.maximum(x, 0.0).reshape(lead + (fb.shape[0], frames))


def inverse_mel_scale_vjp(mel, fb, grad, mask=None):
    """Mel gradient of inverse_mel_scale for the upstream gradient ``grad`` (..., n_stft, T): the transposed minimum-norm
    map applied to grad * [x > 0] (torch's relu rule), i.e. pinv(fb^T)^T (grad * mask).  ``mask`` overrides the relu mask
    (a kernel's own mask, so that near-zero outputs do not decide the comparison)."""
    fb = np.asarray(fb, dtype=np.float64)
    if mask is None:
        mask = inverse_mel_scale(mel, fb) > 0
    g = np.asarray(grad, dtype=np.float64) * mask
    pinv = np.linalg.pinv(fb.T)  # (n_stft, n_mels)
    return np.einsum("km,...kt->...mt", pinv, g)
