"""Float64 numpy restatement of the spectrogram gradient (vector-Jacobian product) of phase_vocoder and of the waveform
gradient of pitch_shift, composed from the existing STFT, inverse-STFT and resampler VJPs.
tests/test_vocoder_grad_oracle.py checks them against torch.autograd through the reference's op sequence;
tests/test_gpu_vocoder_grad.py checks the kernel against them."""
import math

import numpy as np

from oracle.frontend_oracle import hann_window, resample_len, sinc_resample_kernel, stft

from grad_oracle import spectrogram_vjp
from istft_grad_oracle import inverse_spectrogram_vjp
from resample_grad_oracle import resample_vjp


def time_grid(frames: int, rate: float, grid=np.float32):
    """The time steps ts of torch.arange(0, frames, rate) and the neighbours the reference takes from them:
    (i0, i1, alpha) with i0 = trunc(ts), i1 = trunc(ts + 1) computed in the grid's dtype (not always i0 + 1 in float32)
    and alpha = ts mod 1.  ``grid`` is a dtype -- ts = rate * t rounded to it, the grid of the GPU kernels -- or the
    time steps themselves, e.g. those of a torch.arange call (whose vectorised fill rounds some steps differently)."""
    if isinstance(grid, np.ndarray):
        ts = grid
    else:
        ts = (rate * np.arange(int(math.ceil(frames / rate)), dtype=np.float64)).astype(grid)
    one = ts.dtype.type(1.0)
    return ts.astype(np.int64), (ts + one).astype(np.int64), np.fmod(ts, one).astype(np.float64)


def phase_vocoder(spec, rate, phase_advance, grid=np.float32):
    """The reference's phase_vocoder (functional.py:713-803) in float64 with a time grid in ``grid`` (see time_grid)."""
    spec = np.asarray(spec, dtype=np.complex128)
    if rate == 1.0:
        return spec
    lead = spec.shape[:-2]
    sp = spec.reshape((-1,) + spec.shape[-2:])
    i0, i1, alpha = time_grid(sp.shape[-1], rate, grid)
    padded = np.concatenate([sp, np.zeros(sp.shape[:-1] + (2,), dtype=sp.dtype)], axis=-1)
    s0, s1 = padded[..., i0], padded[..., i1]
    pa = np.asarray(phase_advance, dtype=np.float64).reshape(-1, 1)
    phase = np.angle(s1) - np.angle(s0) - pa
    phase = phase - 2 * math.pi * np.round(phase / (2 * math.pi))
    phase = np.concatenate([np.angle(sp[..., :1]), (phase + pa)[..., :-1]], axis=-1)
    out = (alpha * np.abs(s1) + (1 - alpha) * np.abs(s0)) * np.exp(1j * np.cumsum(phase, axis=-1))
    return out.reshape(lead + out.shape[1:])


def phase_vocoder_vjp(spec, grad, rate, out=None, phase_advance=None, grid=np.float32) -> np.ndarray:
    """Gradient of Re sum(conj(grad) * phase_vocoder(spec)) with respect to the (..., bins, frames_in) complex ``spec``,
    in torch's convention dL/dRe + i dL/dIm (``grad`` is dL/dRe out + i dL/dIm out).  With the forward's output o:
        a_t = Im g_t Re o_t - Re g_t Im o_t,  m_t = Re(conj(g_t) sgn(o_t)),  S_t = sum_{u >= t} a_u  (S_{frames_out} = 0)
        M_i = sum_{i0(t)=i} (1 - alpha_t) m_t + sum_{i1(t)=i} alpha_t m_t
        P_i = sum_{i1(t)=i} S_{t+1} - sum_{i0(t)=i} S_{t+1} + [i = 0] S_0
        grad_spec[i] = sgn(X_i) M_i + (i X_i / |X_i|^2) P_i   (0 at X_i = 0)
    ``out`` defaults to the float64 forward.  ``phase_advance`` (default zeros) changes that output only by round-off:
    the wrap takes it back out modulo 2 pi."""
    spec = np.asarray(spec, dtype=np.complex128)
    g = np.asarray(grad, dtype=np.complex128)
    if rate == 1.0:
        return g.copy()
    lead = spec.shape[:-2]
    bins, frames = spec.shape[-2:]
    sp = spec.reshape(-1, bins, frames)
    if out is None:
        pa = np.zeros(bins) if phase_advance is None else phase_advance
        out = phase_vocoder(sp, rate, pa, grid)
    o = np.asarray(out, dtype=np.complex128).reshape(sp.shape[0], bins, -1)
    g = g.reshape(o.shape)
    i0, i1, alpha = time_grid(frames, rate, grid)
    n_out = len(i0)
    a = g.imag * o.real - g.real * o.imag
    mo = np.abs(o)
    with np.errstate(divide="ignore", invalid="ignore"):
        m = np.where(mo > 0, (g.real * o.real + g.imag * o.imag) / mo, 0.0)
    S = np.cumsum(a[..., ::-1], axis=-1)[..., ::-1]  # S_t
    S_next = np.concatenate([S[..., 1:], np.zeros(S.shape[:-1] + (1,))], axis=-1)  # S_{t+1}
    M = np.zeros(sp.shape[:-1] + (frames + 2,))
    P = np.zeros_like(M)
    for t in range(n_out):
        M[..., i0[t]] += (1 - alpha[t]) * m[..., t]
        M[..., i1[t]] += alpha[t] * m[..., t]
        P[..., i1[t]] += S_next[..., t]
        P[..., i0[t]] -= S_next[..., t]
    P[..., 0] += S[..., 0]
    M, P = M[..., :frames], P[..., :frames]  # the pad frames are dropped
    mag = np.abs(sp)
    with np.errstate(divide="ignore", invalid="ignore"):
        gx = np.where(mag > 0, sp / mag * M + 1j * sp / mag**2 * P, 0.0)
    return gx.reshape(lead + (bins, frames))


def pitch_shift_vjp(x, grad, sample_rate, n_steps, bins_per_octave=12, n_fft=512, win_length=None, hop_length=None,
                    window=None, grid=np.float32) -> np.ndarray:
    """Gradient of sum(grad * pitch_shift(x)) with respect to the waveform x (reference functional.py:1579-1719): the
    adjoints of crop / zero-pad, resample, inverse STFT, phase vocoder and complex STFT, in that order."""
    x = np.asarray(x, dtype=np.float64)
    hop_length = n_fft // 4 if hop_length is None else hop_length
    win_length = n_fft if win_length is None else win_length
    window = hann_window(win_length) if window is None else np.asarray(window, dtype=np.float64)
    lead, ori_len = x.shape[:-1], x.shape[-1]
    flat = x.reshape(-1, ori_len)
    g = np.asarray(grad, dtype=np.float64).reshape(-1, ori_len)
    rate = 2.0 ** (-float(n_steps) / bins_per_octave)
    spec = stft(flat, n_fft, hop_length, window, center=True, pad_mode="reflect")
    frames_out = len(time_grid(spec.shape[-1], rate, grid)[0]) if rate != 1.0 else spec.shape[-1]
    len_stretch = int(round(ori_len / rate))
    orig_freq = int(sample_rate / rate)
    if orig_freq != sample_rate:
        gcd = math.gcd(orig_freq, int(sample_rate))
        kernel, width = sinc_resample_kernel(orig_freq, sample_rate, gcd)
        shift_len = resample_len(len_stretch, orig_freq // gcd, sample_rate // gcd)
    else:
        shift_len = len_stretch
    g_shift = np.zeros((g.shape[0], shift_len))
    keep = min(shift_len, ori_len)
    g_shift[:, :keep] = g[:, :keep]
    if orig_freq != sample_rate:
        g_stretch = resample_vjp(g_shift, orig_freq, sample_rate, gcd, kernel, width, len_stretch)
    else:
        g_stretch = g_shift
    g_y = inverse_spectrogram_vjp(g_stretch, frames_out, len_stretch, 0, window, n_fft, hop_length, win_length)
    pa = np.linspace(0, math.pi * hop_length, spec.shape[-2])[:, None]
    g_spec = phase_vocoder_vjp(spec, g_y, rate, phase_advance=pa, grid=grid)
    gx = spectrogram_vjp(flat, g_spec, 0, window, n_fft, hop_length, win_length, None)
    return gx.reshape(lead + (ori_len,))
