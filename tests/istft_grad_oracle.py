"""Float64 numpy restatement of the spectrogram gradient (vector-Jacobian product) of inverse_spectrogram, next to the
forward restatement in oracle/frontend_oracle.py.  tests/test_istft_grad_oracle.py checks it against torch.autograd
through torch.istft; tests/test_gpu_istft_grad.py checks the kernels against it."""
import numpy as np

from oracle.frontend_oracle import _spec_norms


def inverse_spectrogram_vjp(
    grad: np.ndarray,
    frames: int,
    length,
    pad: int,
    window: np.ndarray,
    n_fft: int,
    hop: int,
    win_length: int,
    normalized=False,
    center: bool = True,
) -> np.ndarray:
    """Gradient of sum(grad * inverse_spectrogram(Z, length, pad, ...)) with respect to the (..., n_fft//2+1, frames)
    complex spectrogram Z, in torch's convention dL/dRe Z + i dL/dIm Z.  With X = scale * DFT(w * frame) the forward
    normalisation and env[s] = sum_t w^2[s - t hop]:
        g_hat[s] = grad[s - start] / env[s] on the returned samples (s < n_fft + hop (frames - 1)), else 0
        grad_Z[t][k] = c_k / (n_fft scale) * sum_n w[n] g_hat[t hop + n] e^(-2 pi i k n / n_fft)
    c_0 = c_{n_fft/2} = 1, c_k = 2 otherwise (the C2R transform ignores the imaginary parts of those two bins).
    start = n_fft/2 when centred, plus the `pad` the reference slices off when `length` is given."""
    g = np.asarray(grad, dtype=np.float64)
    lead = g.shape[:-1]
    gf = g.reshape(-1, g.shape[-1])
    fl_norm, win_norm = _spec_norms(normalized)
    win = np.asarray(window, dtype=np.float64)
    scale = (float(n_fft) ** -0.5 if fl_norm else 1.0) * (1.0 / np.sqrt(np.sum(win**2)) if win_norm else 1.0)
    w = np.zeros(n_fft)
    left = (n_fft - win_length) // 2
    w[left : left + win_length] = win
    expected = n_fft + hop * (frames - 1)
    idx = np.arange(frames)[:, None] * hop + np.arange(n_fft)[None, :]  # (frames, n_fft) sample of each frame position
    env = np.zeros(expected)
    np.add.at(env, idx.ravel(), np.tile(w * w, frames))
    start = (n_fft // 2 if center else 0) + (pad if length is not None and pad > 0 else 0)
    g_hat = np.zeros((gf.shape[0], expected))
    m = max(0, min(gf.shape[1], expected - start))
    g_hat[:, start : start + m] = gf[:, :m] / env[start : start + m]
    spec = np.fft.rfft(g_hat[:, idx] * w, axis=-1)  # (B, frames, n_fft//2+1)
    c = np.full(n_fft // 2 + 1, 2.0)
    c[0] = 1.0
    if n_fft % 2 == 0:
        c[-1] = 1.0
    spec = spec * c / (n_fft * scale)
    spec[..., 0] = spec[..., 0].real
    if n_fft % 2 == 0:
        spec[..., -1] = spec[..., -1].real
    return np.swapaxes(spec, -1, -2).reshape(lead + (n_fft // 2 + 1, frames))
