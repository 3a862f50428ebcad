"""Float64 numpy restatement of the input gradients (vector-Jacobian products) of AmplitudeToDB, MFCC, LFCC, MelScale
and SpectralCentroid, built on oracle/frontend_oracle.py and the waveform VJPs of tests/grad_oracle.py.  The tests check
it against torch.autograd through the reference's op sequence (tests/test_feature_grad_oracle.py) and the GPU kernels
against it (tests/test_gpu_feature_grad.py).  The torch_* functions restate the reference's op sequence in torch: float64
is the autograd reference, float32 on the CPU the yardstick of float32 round-off."""
import math

import numpy as np
import torch

from oracle.frontend_oracle import create_dct, hann_window, linear_fbanks, mel_spectrogram, melscale_fbanks, spectrogram

from grad_oracle import mel_spectrogram_vjp, spectrogram_vjp


def db_groups(shape) -> np.ndarray:
    """Group index of every element of a tensor of this shape under amplitude_to_DB's packing rule (functional.py:
    395-399): one group for dim <= 3, one per element of the flattened leading dims beyond the last three otherwise."""
    groups = int(np.prod(shape[:-3])) if len(shape) > 3 else 1
    return np.repeat(np.arange(groups), int(np.prod(shape)) // groups).reshape(shape)


def amplitude_to_db_vjp(x, grad, multiplier, amin, db_multiplier, top_db=None, d=None, gmax=None) -> np.ndarray:
    """Gradient of sum(grad * amplitude_to_DB(x, ...)) with respect to x, with torch's rules:
    clamp(min=amin) passes the gradient where x >= amin; maximum(d, thr) gives it to d where d > thr, half where
    d == thr, the rest to thr; thr = amax_g(d) - top_db sums that over the group and splits it evenly over the elements
    equal to the maximum.  ``d`` / ``gmax`` (optional): the pre-clamp values and per-group maxima the mask and tie
    decisions use -- e.g. a float32 forward's, whose threshold is then formed in float32 as that forward forms it."""
    x = np.asarray(x, dtype=np.float64)
    g = np.asarray(grad, dtype=np.float64)
    if d is None:
        d = multiplier * np.log10(np.maximum(x, amin)) - multiplier * db_multiplier
    g_d = g.copy()
    if top_db is not None:
        grp = db_groups(x.shape)
        n_groups = int(grp.max()) + 1
        if gmax is None:
            gmax = np.array([d[grp == k].max() for k in range(n_groups)])
            thr = gmax - top_db
        else:
            gmax = np.asarray(gmax)
            thr = (gmax.astype(np.float32) - np.float32(top_db)).astype(np.float64)
        te, me = thr[grp], np.asarray(gmax, dtype=np.float64)[grp]
        own = np.where(d > te, g, np.where(d == te, 0.5 * g, 0.0))
        routed = np.where(d < te, g, np.where(d == te, 0.5 * g, 0.0))
        tie = d == me
        r = np.bincount(grp.ravel(), weights=routed.ravel(), minlength=n_groups)
        count = np.bincount(grp.ravel(), weights=tie.ravel().astype(np.float64), minlength=n_groups)
        share = np.where(count > 0, r / np.maximum(count, 1), 0.0)
        g_d = own + np.where(tie, share[grp], 0.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(x >= amin, g_d * multiplier / (math.log(10.0) * x), 0.0)


def _feature_vjp(mel, g_c, dct, log, d, gmax):
    """Gradient at the filter outputs (..., n, T) of DCT(log(mel + 1e-6)) or DCT(AmplitudeToDB('power', 80)(mel))."""
    g_feat = np.asarray(dct, dtype=np.float64) @ np.asarray(g_c, dtype=np.float64)  # (..., n, T)
    if log:
        return g_feat / (mel + 1e-6)
    return amplitude_to_db_vjp(mel, g_feat, 10.0, 1e-10, 0.0, 80.0, d, gmax)


def mfcc_vjp(x, grad, sample_rate=16000, n_mfcc=40, norm="ortho", log_mels=False, melkwargs=None, fb=None, dct=None,
             d=None, gmax=None) -> np.ndarray:
    """Gradient of sum(grad * MFCC(x)) with respect to the waveform x (transforms.MFCC.forward, _transforms.py:698-709)."""
    kw = dict(melkwargs or {})
    n_fft = kw.get("n_fft", 400)
    if fb is None:
        f_max = kw.get("f_max") or float(sample_rate // 2)
        fb = melscale_fbanks(n_fft // 2 + 1, kw.get("f_min", 0.0), f_max, kw.get("n_mels", 128), sample_rate,
                             kw.get("norm"), kw.get("mel_scale", "htk"))
    mel = mel_spectrogram(x, sample_rate=sample_rate, fb=fb, **kw)
    if dct is None:
        dct = create_dct(n_mfcc, mel.shape[-2], norm)
    g_mel = _feature_vjp(mel, grad, dct, log_mels, d, gmax)
    return mel_spectrogram_vjp(x, g_mel, sample_rate, fb=fb, **kw)


def lfcc_vjp(x, grad, sample_rate=16000, n_filter=128, f_min=0.0, f_max=None, n_lfcc=40, norm="ortho", log_lf=False,
             speckwargs=None, filter_mat=None, dct=None, d=None, gmax=None) -> np.ndarray:
    """Gradient of sum(grad * LFCC(x)) with respect to the waveform x (transforms.LFCC.forward, _transforms.py:802-819)."""
    kw = dict(speckwargs or {})
    n_fft = kw.get("n_fft", 400)
    win = kw.get("win_length", None) or n_fft
    hop = kw.get("hop_length", None) or win // 2
    args = (kw.get("pad", 0), hann_window(win), n_fft, hop, win, kw.get("power", 2.0), kw.get("normalized", False),
            kw.get("center", True), kw.get("pad_mode", "reflect"), True)
    if filter_mat is None:
        f_max = float(sample_rate // 2) if f_max is None else f_max
        filter_mat = linear_fbanks(n_fft // 2 + 1, f_min, f_max, n_filter, sample_rate)
    filter_mat = np.asarray(filter_mat, dtype=np.float64)
    spec = spectrogram(x, *args)
    filt = np.swapaxes(np.swapaxes(spec, -1, -2) @ filter_mat, -1, -2)
    if dct is None:
        dct = create_dct(n_lfcc, filt.shape[-2], norm)
    g_filt = _feature_vjp(filt, grad, dct, log_lf, d, gmax)
    return spectrogram_vjp(x, filter_mat @ g_filt, *args)


def melscale_vjp(grad, fb) -> np.ndarray:
    """Gradient of sum(grad * MelScale(spec)) with respect to spec (..., n_bins, T): fb @ grad."""
    return np.asarray(fb, dtype=np.float64) @ np.asarray(grad, dtype=np.float64)


def spectral_centroid_vjp(x, grad, sample_rate, pad, window, n_fft, hop, win_length) -> np.ndarray:
    """Gradient of sum(grad * spectral_centroid(x, ...)) with respect to x (functional.py:1257-1299): y = N / D with
    N = sum_k f_k |X_k|, D = sum_k |X_k|, so g_N = g / D and g_D = -g N / D^2, then the magnitude-spectrogram VJP."""
    spec = spectrogram(x, pad, window, n_fft, hop, win_length, 1.0, False)
    freqs = np.linspace(0.0, float(sample_rate // 2), 1 + n_fft // 2)[:, None]
    num, den = (freqs * spec).sum(axis=-2), spec.sum(axis=-2)
    g = np.asarray(grad, dtype=np.float64)
    g_n, g_d = g / den, -g * num / (den * den)
    g_spec = freqs * g_n[..., None, :] + g_d[..., None, :]
    return spectrogram_vjp(x, g_spec, pad, window, n_fft, hop, win_length, 1.0)


# ---- the reference's op sequence in torch ------------------------------------------------------------------------
def torch_spectrogram(x, pad, window, n_fft, hop, win_length, power):
    """torchaudio.functional.spectrogram (center, reflect, one-sided, not normalized) in torch."""
    if pad > 0:
        x = torch.nn.functional.pad(x, (pad, pad), "constant")
    shape = x.size()
    spec = torch.stft(x.reshape(-1, shape[-1]), n_fft=n_fft, hop_length=hop, win_length=win_length, window=window,
                      center=True, pad_mode="reflect", normalized=False, onesided=True, return_complex=True)
    spec = spec.reshape(shape[:-1] + spec.shape[-2:])
    return spec.abs() if power == 1.0 else spec.abs().pow(power)


def torch_amplitude_to_db(x, multiplier, amin, db_multiplier, top_db=None):
    """functional.amplitude_to_DB (functional.py:356-404)."""
    x_db = multiplier * torch.log10(torch.clamp(x, min=amin))
    x_db = x_db - multiplier * db_multiplier
    if top_db is not None:
        shape = x_db.size()
        packed_channels = shape[-3] if x_db.dim() > 2 else 1
        x_db = x_db.reshape(-1, packed_channels, shape[-2], shape[-1])
        x_db = torch.max(x_db, (x_db.amax(dim=(-3, -2, -1)) - top_db).view(-1, 1, 1, 1))
        x_db = x_db.reshape(shape)
    return x_db


def torch_cepstrum(filt, dct, log):
    """The tail of MFCC.forward / LFCC.forward (_transforms.py:698-709, :802-819) on the filter outputs."""
    feat = torch.log(filt + 1e-6) if log else torch_amplitude_to_db(filt, 10.0, 1e-10, 0.0, 80.0)
    return torch.matmul(feat.transpose(-1, -2), dct).transpose(-1, -2)


def torch_mfcc(fb, dct, n_fft, hop, log, power=2.0, dtype=torch.float64):
    """MFCC / LFCC of a waveform in torch (x's dtype), with the filterbank ``fb`` and the DCT matrix ``dct``."""
    window = torch.tensor(hann_window(n_fft), dtype=dtype)
    fb_t, dct_t = torch.tensor(fb, dtype=dtype), torch.tensor(dct, dtype=dtype)

    def fn(t):
        spec = torch_spectrogram(t, 0, window, n_fft, hop, n_fft, power)
        mel = torch.matmul(spec.transpose(-1, -2), fb_t).transpose(-1, -2)
        return torch_cepstrum(mel, dct_t, log)

    return fn
