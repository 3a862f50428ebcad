"""Float64 numpy restatement of the waveform gradients (vector-Jacobian products) of spectrogram / mel_spectrogram,
built on the forward restatements of oracle/frontend_oracle.py.  The tests check it against torch.autograd through
torch.stft (tests/test_grad_oracle.py) and the GPU kernels against it (tests/test_gpu_grad.py)."""
import numpy as np

from oracle.frontend_oracle import _spec_norms, hann_window, melscale_fbanks, pad_index, stft


def _fold_padding(dxp: np.ndarray, length: int, pad: int, n_fft: int, center: bool, pad_mode: str) -> np.ndarray:
    """Adjoint of the constant ``pad`` plus centre padding: (B, L') -> (B, L), every padded sample added onto the
    sample it was copied from."""
    h = n_fft // 2 if center else 0
    ext = length + 2 * pad
    src = np.array([pad_index(i - h, ext, pad_mode if center else "constant") for i in range(dxp.shape[-1])])
    src = np.where(src >= 0, src - pad, -1)
    keep = (src >= 0) & (src < length)
    dx = np.zeros((dxp.shape[0], length))
    for b in range(dxp.shape[0]):
        np.add.at(dx[b], src[keep], dxp[b, keep])
    return dx


def spectrogram_vjp(
    x: np.ndarray,
    grad: np.ndarray,
    pad: int,
    window: np.ndarray,
    n_fft: int,
    hop: int,
    win_length: int,
    power,
    normalized=False,
    center: bool = True,
    pad_mode: str = "reflect",
    onesided: bool = True,
) -> np.ndarray:
    """Gradient of sum(grad * spectrogram(x, ...)) with respect to x, float64 (real part of the pairing for
    ``power=None``, as torch's complex autograd).  With X = scale * DFT(w * frame):
    G = grad (power None) or p |X|^(p-2) X grad, 0 at X = 0 for p >= 1 and NaN for p < 1;
    dframe = scale * w * N * irfft(H), H_k = (G_k + conj G_{N-k}) / 2 with G = 0 outside the output bins; then the
    frames are overlap-added and the padding folded back onto the source samples."""
    x = np.asarray(x, dtype=np.float64)
    lead, length = x.shape[:-1], x.shape[-1]
    flat = x.reshape(-1, length)
    g = np.asarray(grad)
    g = np.swapaxes(g.reshape((-1,) + g.shape[-2:]), -1, -2)  # (B, T, n_freq)
    fl_norm, win_norm = _spec_norms(normalized)
    win = np.asarray(window, dtype=np.float64)
    scale = (float(n_fft) ** -0.5 if fl_norm else 1.0) * (1.0 / np.sqrt(np.sum(win**2)) if win_norm else 1.0)
    w = np.zeros(n_fft)
    left = (n_fft - win_length) // 2
    w[left : left + win_length] = win
    if power is None:
        gk = g.astype(np.complex128)
    else:
        X = np.swapaxes(stft(flat, n_fft, hop, window, center, pad_mode, False, onesided, pad), -1, -2) * scale
        mag = np.abs(X)
        with np.errstate(divide="ignore", invalid="ignore"):
            gk = power * mag ** (power - 2.0) * X * g
        gk[mag == 0] = np.nan if power < 1.0 else 0.0
    full = np.zeros(gk.shape[:-1] + (n_fft,), dtype=np.complex128)
    full[..., : gk.shape[-1]] = gk
    h = 0.5 * (full + np.conj(full[..., (-np.arange(n_fft)) % n_fft]))
    dframes = scale * w * n_fft * np.fft.ifft(h, axis=-1).real  # (B, T, N)
    frames = dframes.shape[1]
    h_pad = n_fft // 2 if center else 0
    lp = length + 2 * pad + 2 * h_pad
    dxp = np.zeros((flat.shape[0], lp))
    for t in range(frames):
        dxp[:, t * hop : t * hop + n_fft] += dframes[:, t]
    return _fold_padding(dxp, length, pad, n_fft, center, pad_mode).reshape(lead + (length,))


def mel_spectrogram_vjp(
    x,
    grad,
    sample_rate=16000,
    n_fft=400,
    win_length=None,
    hop_length=None,
    f_min=0.0,
    f_max=None,
    pad=0,
    n_mels=128,
    window=None,
    power=2.0,
    normalized=False,
    center=True,
    pad_mode="reflect",
    norm=None,
    mel_scale="htk",
    fb=None,
) -> np.ndarray:
    """Gradient of sum(grad * mel_spectrogram(x, ...)) with respect to x: the spectrogram VJP of fb @ grad."""
    win_length = n_fft if win_length is None else win_length
    hop_length = win_length // 2 if hop_length is None else hop_length
    window = hann_window(win_length) if window is None else window
    if fb is None:
        f_max = float(sample_rate // 2) if f_max is None else f_max
        fb = melscale_fbanks(n_fft // 2 + 1, f_min, f_max, n_mels, sample_rate, norm, mel_scale)
    g_spec = np.asarray(fb, dtype=np.float64) @ np.asarray(grad, dtype=np.float64)  # (..., n_freq, T)
    return spectrogram_vjp(x, g_spec, pad, window, n_fft, hop_length, win_length, power, normalized, center, pad_mode,
                           True)
