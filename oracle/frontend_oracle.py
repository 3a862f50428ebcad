"""CPU oracle for the DSP front-end hot path  --  TEST INFRASTRUCTURE, NOT PRODUCT.

This file restates, in plain numpy float64, the algorithm that pytorch/audio runs
for Spectrogram / MelSpectrogram / MFCC / Resample.  It exists only so that
``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` / ``--impl
reference`` legs of ``bench.py`` can check the CUDA product; nothing under
``audio_b200/`` may import it.

Parity status: PINNED.  ``tests/test_oracle_golden.py`` checks every function
here against (a) the librosa golden vectors the reference's own test-suite
holds (``test/torchaudio_unittest/assets/librosa_expected_results``, converted
by ``tests/golden/make_golden.py``) and (b) outputs of the reference itself
(``pytorch/audio/src`` imported by the same script).

The arithmetic of the reference lives in PyTorch/ATen (third-party, not under
pytorch/audio; torch 2.11.0 here): ``torch.stft`` -> ``at::stft`` ->
``_fft_r2c`` (MKL DFTI), ``matmul``, ``conv1d``.  Their *published* definitions
are restated below; every function cites the reference call site it follows
(paths relative to pytorch/audio).
"""
from __future__ import annotations

import math

import numpy as np

__all__ = [
    "num_frames",
    "pad_index",
    "hann_window",
    "stft",
    "spectrogram",
    "hz_to_mel",
    "mel_to_hz",
    "melscale_fbanks",
    "create_dct",
    "amplitude_to_db",
    "mel_spectrogram",
    "mfcc",
    "linear_fbanks",
    "lfcc",
    "spectral_centroid",
    "sinc_resample_kernel",
    "resample_len",
    "apply_sinc_resample_kernel",
    "resample",
]


# ----------------------------------------------------------------------------
# integer bookkeeping (must be bit-exact)
# ----------------------------------------------------------------------------
def num_frames(length: int, n_fft: int, hop: int, center: bool, pad: int = 0) -> int:
    """Frame count of torch.stft as called from
    src/torchaudio/functional/functional.py:123-134 (``pad`` applied first, :112-114).
    center pads n_fft//2 on both sides (torch/functional.py:675-680), then
    n_frames = 1 + (L_padded - n_fft) // hop."""
    lp = length + 2 * pad
    if center:
        lp += 2 * (n_fft // 2)
    if lp < n_fft:
        raise ValueError("signal shorter than n_fft")
    return 1 + (lp - n_fft) // hop


def pad_index(i: int, n: int, mode: str) -> int:
    """Source index in [0, n) for a (possibly out-of-range) index ``i`` under a
    torch.nn.functional.pad mode; -1 means "constant zero".  Used by torch.stft's
    centre padding (torch/functional.py:675-680)."""
    if 0 <= i < n:
        return i
    if mode == "constant":
        return -1
    if mode == "reflect":  # single reflection, no edge repeat; requires pad < n
        if i < 0:
            return -i
        return 2 * (n - 1) - i
    if mode == "replicate":
        return 0 if i < 0 else n - 1
    if mode == "circular":
        return i % n
    raise ValueError(mode)


# ----------------------------------------------------------------------------
# STFT -> |.|^p      (functional.py:54-145, torch.stft semantics)
# ----------------------------------------------------------------------------
def hann_window(n: int) -> np.ndarray:
    """torch.hann_window(n) (periodic=True), the default window_fn
    (src/torchaudio/transforms/_transforms.py:70,86)."""
    k = np.arange(n, dtype=np.float64)
    return 0.5 - 0.5 * np.cos(2.0 * np.pi * k / n)


def _padded_signal(x: np.ndarray, pad: int, n_fft: int, center: bool, pad_mode: str) -> np.ndarray:
    """(B, L) -> (B, L') applying the constant ``pad`` then the centre padding."""
    if pad > 0:
        x = np.pad(x, ((0, 0), (pad, pad)))
    if center:
        h = n_fft // 2
        if pad_mode == "reflect":
            if h >= x.shape[-1]:
                raise ValueError("reflect padding needs n_fft//2 < length")
            x = np.pad(x, ((0, 0), (h, h)), mode="reflect")
        elif pad_mode == "constant":
            x = np.pad(x, ((0, 0), (h, h)))
        elif pad_mode == "replicate":
            x = np.pad(x, ((0, 0), (h, h)), mode="edge")
        elif pad_mode == "circular":
            x = np.pad(x, ((0, 0), (h, h)), mode="wrap")
        else:
            raise ValueError(pad_mode)
    return x


def stft(
    x: np.ndarray,
    n_fft: int,
    hop: int,
    window: np.ndarray,
    center: bool = True,
    pad_mode: str = "reflect",
    frame_length_norm: bool = False,
    onesided: bool = True,
    pad: int = 0,
) -> np.ndarray:
    """Complex STFT, shape (B, n_freq, T), float64 math.
    Follows at::stft as invoked at functional.py:123-134: the window (length
    win_length <= n_fft) is zero padded to n_fft with left = (n_fft-win)//2;
    frame t = x_padded[t*hop : t*hop+n_fft]; X[k] = sum_n w[n] x[n] e^{-2 pi i k n / n_fft};
    ``normalized`` multiplies by n_fft**-0.5."""
    x = np.asarray(x, dtype=np.float64)
    squeeze = x.ndim == 1
    x = np.atleast_2d(x)
    win = np.asarray(window, dtype=np.float64)
    if win.shape[0] < n_fft:
        left = (n_fft - win.shape[0]) // 2
        w = np.zeros(n_fft)
        w[left : left + win.shape[0]] = win
        win = w
    xp = _padded_signal(x, pad, n_fft, center, pad_mode)
    t = 1 + (xp.shape[-1] - n_fft) // hop
    idx = np.arange(n_fft)[None, :] + hop * np.arange(t)[:, None]
    frames = xp[:, idx] * win  # (B, T, n_fft)
    spec = np.fft.rfft(frames, axis=-1) if onesided else np.fft.fft(frames, axis=-1)
    if frame_length_norm:
        spec = spec * (float(n_fft) ** -0.5)
    spec = np.swapaxes(spec, -1, -2)  # (B, n_freq, T)
    return spec[0] if squeeze else spec


def _spec_norms(normalized):
    """functional.py:228-242."""
    if isinstance(normalized, str):
        if normalized not in ("frame_length", "window"):
            raise ValueError(f"Invalid normalized parameter: {normalized}")
        return normalized == "frame_length", normalized == "window"
    if isinstance(normalized, bool):
        return False, normalized
    raise TypeError("Input type not supported")


def spectrogram(
    x: np.ndarray,
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
    """functional.spectrogram (functional.py:54-145). Leading dims are packed
    (:119-120), the result is (..., n_freq, T); ``power=None`` returns complex."""
    x = np.asarray(x, dtype=np.float64)
    lead = x.shape[:-1]
    flat = x.reshape(-1, x.shape[-1])
    assert len(window) == win_length
    fl_norm, win_norm = _spec_norms(normalized)
    s = stft(flat, n_fft, hop, window, center, pad_mode, fl_norm, onesided, pad)
    s = s.reshape(lead + s.shape[-2:])
    if win_norm:
        s = s / np.sqrt(np.sum(np.asarray(window, dtype=np.float64) ** 2))
    if power is None:
        return s
    mag = np.abs(s)
    return mag if power == 1.0 else mag**power


# ----------------------------------------------------------------------------
# mel filterbank, DCT, dB   (functional.py:425-587, 636-667, 356-404)
# ----------------------------------------------------------------------------
def hz_to_mel(freq: float, mel_scale: str = "htk") -> float:
    """functional.py:425-455."""
    if mel_scale == "htk":
        return 2595.0 * math.log10(1.0 + freq / 700.0)
    if mel_scale != "slaney":
        raise ValueError('mel_scale should be one of "htk" or "slaney".')
    lin_step = 200.0 / 3
    knee_hz = 1000.0
    knee_mel = knee_hz / lin_step
    if freq >= knee_hz:
        return knee_mel + math.log(freq / knee_hz) / (math.log(6.4) / 27.0)
    return freq / lin_step


def mel_to_hz(mels: np.ndarray, mel_scale: str = "htk") -> np.ndarray:
    """functional.py:458-489."""
    mels = np.asarray(mels, dtype=np.float64)
    if mel_scale == "htk":
        return 700.0 * (10.0 ** (mels / 2595.0) - 1.0)
    if mel_scale != "slaney":
        raise ValueError('mel_scale should be one of "htk" or "slaney".')
    lin_step = 200.0 / 3
    knee_hz = 1000.0
    knee_mel = knee_hz / lin_step
    out = lin_step * mels
    hi = mels >= knee_mel
    out[hi] = knee_hz * np.exp((math.log(6.4) / 27.0) * (mels[hi] - knee_mel))
    return out


def melscale_fbanks(n_freqs, f_min, f_max, n_mels, sample_rate, norm=None, mel_scale="htk") -> np.ndarray:
    """functional.melscale_fbanks (functional.py:518-587) with the triangular
    construction of :492-515; returns (n_freqs, n_mels) float64."""
    if norm is not None and norm != "slaney":
        raise ValueError('norm must be one of None or "slaney"')
    bins_hz = np.linspace(0.0, float(sample_rate // 2), n_freqs)
    edges_mel = np.linspace(hz_to_mel(f_min, mel_scale), hz_to_mel(f_max, mel_scale), n_mels + 2)
    edges_hz = mel_to_hz(edges_mel, mel_scale)
    widths = np.diff(edges_hz)  # n_mels + 1
    delta = edges_hz[None, :] - bins_hz[:, None]  # (n_freqs, n_mels + 2)
    falling = -delta[:, :-2] / widths[:-1]
    rising = delta[:, 2:] / widths[1:]
    fb = np.maximum(0.0, np.minimum(falling, rising))
    if norm == "slaney":
        fb = fb * (2.0 / (edges_hz[2 : n_mels + 2] - edges_hz[:n_mels]))[None, :]
    return fb


def create_dct(n_mfcc: int, n_mels: int, norm) -> np.ndarray:
    """functional.create_dct (functional.py:636-667): DCT-II matrix (n_mels, n_mfcc)."""
    if norm is not None and norm != "ortho":
        raise ValueError('norm must be either "ortho" or None')
    n = np.arange(n_mels, dtype=np.float64)[None, :]
    k = np.arange(n_mfcc, dtype=np.float64)[:, None]
    d = np.cos(math.pi / n_mels * (n + 0.5) * k)
    if norm is None:
        d = d * 2.0
    else:
        d[0] *= 1.0 / math.sqrt(2.0)
        d = d * math.sqrt(2.0 / n_mels)
    return d.T


def amplitude_to_db(x: np.ndarray, multiplier: float, amin: float, db_multiplier: float, top_db=None) -> np.ndarray:
    """functional.amplitude_to_DB (functional.py:356-404).  NOTE the packing rule
    (:395-399): for a tensor of dim <= 3 there is ONE cut-off over the whole tensor
    (for dim == 3 the leading dim is folded into 'channels'); for dim >= 4 there is
    one cut-off per element of the flattened leading dims."""
    x = np.asarray(x, dtype=np.float64)
    db = multiplier * np.log10(np.maximum(x, amin)) - multiplier * db_multiplier
    if top_db is not None:
        shape = db.shape
        ch = shape[-3] if db.ndim > 2 else 1
        packed = db.reshape(-1, ch, shape[-2], shape[-1])
        floor = packed.max(axis=(-3, -2, -1)) - top_db
        db = np.maximum(packed, floor[:, None, None, None]).reshape(shape)
    return db


def mel_spectrogram(
    x,
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
    """transforms.MelSpectrogram.forward (src/torchaudio/transforms/_transforms.py:557-622)
    = Spectrogram (:101-123) then MelScale (:403-415, matmul at :413).
    ``fb`` may be supplied to use the reference's exact (fp32-built) filterbank."""
    win_length = n_fft if win_length is None else win_length
    hop_length = win_length // 2 if hop_length is None else hop_length
    window = hann_window(win_length) if window is None else window
    spec = spectrogram(x, pad, window, n_fft, hop_length, win_length, power, normalized, center, pad_mode, True)
    if fb is None:
        f_max = float(sample_rate // 2) if f_max is None else f_max
        fb = melscale_fbanks(n_fft // 2 + 1, f_min, f_max, n_mels, sample_rate, norm, mel_scale)
    fb = np.asarray(fb, dtype=np.float64)
    return np.swapaxes(np.swapaxes(spec, -1, -2) @ fb, -1, -2)


def mfcc(x, sample_rate=16000, n_mfcc=40, norm="ortho", log_mels=False, melkwargs=None, fb=None, dct=None):
    """transforms.MFCC.forward (_transforms.py:663-709): mel -> log(mel+1e-6) or
    AmplitudeToDB('power', top_db=80) (:680-681,701-705) -> DCT matmul (:708)."""
    melkwargs = dict(melkwargs or {})
    mel = mel_spectrogram(x, sample_rate=sample_rate, fb=fb, **melkwargs)
    n_mels = mel.shape[-2]
    if n_mfcc > n_mels:
        raise ValueError("Cannot select more MFCC coefficients than # mel bins")
    if log_mels:
        feat = np.log(mel + 1e-6)
    else:
        feat = amplitude_to_db(mel, 10.0, 1e-10, math.log10(max(1e-10, 1.0)), 80.0)
    d = create_dct(n_mfcc, n_mels, norm) if dct is None else np.asarray(dct, dtype=np.float64)
    return np.swapaxes(np.swapaxes(feat, -1, -2) @ d, -1, -2)


def linear_fbanks(n_freqs, f_min, f_max, n_filter, sample_rate) -> np.ndarray:
    """functional.linear_fbanks (functional.py:590-633): the triangles of :492-515 on a linear grid."""
    bins_hz = np.linspace(0.0, float(sample_rate // 2), n_freqs)
    edges_hz = np.linspace(f_min, f_max, n_filter + 2)
    widths = np.diff(edges_hz)
    delta = edges_hz[None, :] - bins_hz[:, None]
    return np.maximum(0.0, np.minimum(-delta[:, :-2] / widths[:-1], delta[:, 2:] / widths[1:]))


def lfcc(x, sample_rate=16000, n_filter=128, f_min=0.0, f_max=None, n_lfcc=40, norm="ortho", log_lf=False,
         speckwargs=None, filter_mat=None, dct=None):
    """transforms.LFCC.forward (_transforms.py:712-819): Spectrogram -> linear filterbank -> dB (top_db 80,
    with AmplitudeToDB's packing rule) or log -> DCT."""
    kw = dict(speckwargs or {})
    n_fft = kw.get("n_fft", 400)
    win = kw.get("win_length", None) or n_fft
    hop = kw.get("hop_length", None) or win // 2
    spec = spectrogram(x, kw.get("pad", 0), hann_window(win), n_fft, hop, win, kw.get("power", 2.0),
                       kw.get("normalized", False), kw.get("center", True), kw.get("pad_mode", "reflect"), True)
    if filter_mat is None:
        f_max = float(sample_rate // 2) if f_max is None else f_max
        filter_mat = linear_fbanks(n_fft // 2 + 1, f_min, f_max, n_filter, sample_rate)
    filt = np.swapaxes(np.swapaxes(spec, -1, -2) @ np.asarray(filter_mat, dtype=np.float64), -1, -2)
    feat = np.log(filt + 1e-6) if log_lf else amplitude_to_db(filt, 10.0, 1e-10, 0.0, 80.0)
    d = create_dct(n_lfcc, filt.shape[-2], norm) if dct is None else np.asarray(dct, dtype=np.float64)
    return np.swapaxes(np.swapaxes(feat, -1, -2) @ d, -1, -2)


def spectral_centroid(x, sample_rate, pad, window, n_fft, hop, win_length) -> np.ndarray:
    """functional.spectral_centroid (functional.py:1257-1299)."""
    spec = spectrogram(x, pad, window, n_fft, hop, win_length, 1.0, False)
    freqs = np.linspace(0.0, float(sample_rate // 2), 1 + n_fft // 2)[:, None]
    return (freqs * spec).sum(axis=-2) / spec.sum(axis=-2)


# ----------------------------------------------------------------------------
# polyphase sinc resampler   (functional.py:1305-1490)
# ----------------------------------------------------------------------------
def _i0(x: np.ndarray) -> np.ndarray:
    return np.i0(x)


def sinc_resample_kernel(
    orig_freq: int,
    new_freq: int,
    gcd: int,
    lowpass_filter_width: int = 6,
    rolloff: float = 0.99,
    resampling_method: str = "sinc_interp_hann",
    beta=None,
):
    """functional._get_sinc_resample_kernel (functional.py:1305-1402), float64.
    Returns (kernel[new', 2*width + orig'], width)."""
    if not (int(orig_freq) == orig_freq and int(new_freq) == new_freq):
        raise Exception("Frequencies must be of integer type")
    if resampling_method not in ("sinc_interp_hann", "sinc_interp_kaiser"):
        raise ValueError(f"Invalid resampling method: {resampling_method}")
    o = int(orig_freq) // gcd
    n = int(new_freq) // gcd
    if lowpass_filter_width <= 0:
        raise ValueError("Low pass filter width should be positive.")
    cutoff = min(o, n) * rolloff
    width = math.ceil(lowpass_filter_width * o / cutoff)
    taps = np.arange(-width, width + o, dtype=np.float64)[None, :] / o
    phase = -np.arange(n, dtype=np.float64)[:, None] / n
    t = np.clip((phase + taps) * cutoff, -lowpass_filter_width, lowpass_filter_width)
    if resampling_method == "sinc_interp_hann":
        win = np.cos(t * math.pi / lowpass_filter_width / 2) ** 2
    else:
        b = 14.769656459379492 if beta is None else float(beta)
        win = _i0(b * np.sqrt(1 - (t / lowpass_filter_width) ** 2)) / _i0(np.array(b))
    tp = t * math.pi
    with np.errstate(invalid="ignore", divide="ignore"):
        sinc = np.where(tp == 0, 1.0, np.sin(tp) / tp)
    return sinc * win * (cutoff / o), width


def resample_len(length: int, orig_r: int, new_r: int) -> int:
    """target_length of functional.py:1427: torch.ceil(torch.as_tensor(new' * L / orig')):
    python float division, rounded to float32 by as_tensor (default dtype), then ceil."""
    return int(math.ceil(np.float32(new_r * length / orig_r)))


def apply_sinc_resample_kernel(x, orig_freq, new_freq, gcd, kernel, width) -> np.ndarray:
    """functional._apply_sinc_resample_kernel (functional.py:1405-1432):
    zero pad (width, width+orig'), strided correlation with every phase row,
    interleave phases, cut to ceil(new'*L/orig')."""
    x = np.asarray(x, dtype=np.float64)
    o = int(orig_freq) // gcd
    n = int(new_freq) // gcd
    lead = x.shape[:-1]
    flat = x.reshape(-1, x.shape[-1])
    length = flat.shape[-1]
    xp = np.pad(flat, ((0, 0), (width, width + o)))
    k = np.asarray(kernel, dtype=np.float64).reshape(n, -1)
    taps = k.shape[1]
    frames = (xp.shape[-1] - taps) // o + 1
    idx = np.arange(taps)[None, :] + o * np.arange(frames)[:, None]
    seg = xp[:, idx]  # (B, frames, taps)
    out = np.einsum("bft,pt->bfp", seg, k).reshape(flat.shape[0], -1)
    out = out[:, : resample_len(length, o, n)]
    return out.reshape(lead + out.shape[-1:])


def resample(
    x, orig_freq, new_freq, lowpass_filter_width=6, rolloff=0.99, resampling_method="sinc_interp_hann", beta=None
):
    """functional.resample (functional.py:1435-1490)."""
    if orig_freq <= 0.0 or new_freq <= 0.0:
        raise ValueError("Original frequency and desired frequecy should be positive")
    if orig_freq == new_freq:
        return np.asarray(x)
    g = math.gcd(int(orig_freq), int(new_freq))
    k, w = sinc_resample_kernel(orig_freq, new_freq, g, lowpass_filter_width, rolloff, resampling_method, beta)
    return apply_sinc_resample_kernel(x, orig_freq, new_freq, g, k, w)


def istft(spec, n_fft, hop_length, win_length, window, center=True, normalized=False, length=None):
    """torch.istft restated (ATen `istft`, the third-party arithmetic F.inverse_spectrogram calls at
    functional.py:198-209): spec (..., n_fft//2+1, T) complex -> (..., time).

    irfft of every frame (C2R: imaginary parts of bins 0 and n_fft/2 ignored; `normalized` multiplies by sqrt(n_fft)),
    times the centre-padded window, overlap-add at hop_length, division by the overlap-added squared window, the
    slice [n_fft/2, n_fft/2 + length) when centred (zero tail if `length` exceeds what the frames cover)."""
    spec = np.asarray(spec, dtype=np.complex128)
    lead = spec.shape[:-2]
    frames = spec.shape[-1]
    sp = spec.reshape((-1,) + spec.shape[-2:])
    w = np.zeros(n_fft)
    left = (n_fft - win_length) // 2
    w[left:left + win_length] = np.asarray(window, dtype=np.float64)
    if normalized:
        sp = sp * math.sqrt(n_fft)
    fr = np.fft.irfft(np.swapaxes(sp, 1, 2), n=n_fft, axis=-1) * w  # (rows, T, n_fft)
    expected = n_fft + hop_length * (frames - 1)
    y = np.zeros((sp.shape[0], expected))
    env = np.zeros(expected)
    for t in range(frames):
        y[:, t * hop_length:t * hop_length + n_fft] += fr[:, t]
        env[t * hop_length:t * hop_length + n_fft] += w * w
    start = n_fft // 2 if center else 0
    if length is not None:
        end = start + length
    else:
        end = expected - n_fft // 2 if center else expected
    seg_end = min(end, expected)
    assert np.abs(env[start:seg_end]).min() > 1e-11, "window overlap add min"
    out = y[:, start:seg_end] / env[start:seg_end]
    if end > expected:
        out = np.concatenate([out, np.zeros((out.shape[0], end - expected))], axis=1)
    return out.reshape(lead + (out.shape[-1],))


def inverse_spectrogram(spec, length, pad, window, n_fft, hop_length, win_length, normalized=False, center=True):
    """reference functional.py:148-225."""
    spec = np.asarray(spec, dtype=np.complex128)
    frame_norm = normalized == "frame_length"
    if normalized is True or normalized == "window":
        spec = spec * np.sqrt((np.asarray(window, dtype=np.float64) ** 2).sum())
    y = istft(spec, n_fft, hop_length, win_length, window, center=center, normalized=frame_norm,
              length=length + 2 * pad if length is not None else None)
    if length is not None and pad > 0:
        y = y[..., pad:-pad]
    return y


def griffinlim(specgram, window, n_fft, hop_length, win_length, power, n_iter, momentum, length):
    """reference functional.py:255-353 with rand_init=False: fast Griffin-Lim phase recovery.

    specgram (..., freq, time) holds |X|^power; every iteration inverts the current estimate (istft), rebuilds its STFT
    (centred, reflect), and keeps only the phase of `rebuilt - m/(1+m) * previous rebuilt`."""
    if not 0 <= momentum < 1:
        raise ValueError("momentum must be in range [0, 1). Found: {}".format(momentum))
    momentum = momentum / (1 + momentum)
    spec = np.asarray(specgram, dtype=np.float64)
    lead = spec.shape[:-2]
    mag = spec.reshape((-1,) + spec.shape[-2:]) ** (1.0 / power)
    angles = np.ones(mag.shape, dtype=np.complex128)
    tprev = 0.0
    for _ in range(n_iter):
        inverse = istft(mag * angles, n_fft, hop_length, win_length, window, length=length)
        rebuilt = stft(inverse, n_fft, hop_length, window, center=True, pad_mode="reflect")
        angles = rebuilt
        if momentum:
            angles = angles - tprev * momentum
        angles = angles / (np.abs(angles) + 1e-16)
        tprev = rebuilt
    out = istft(mag * angles, n_fft, hop_length, win_length, window, length=length)
    return out.reshape(lead + out.shape[-1:])


def phase_vocoder(spec, rate, phase_advance):
    """reference functional.py:713-803 in float64, with the reference's float32 time grid
    (`torch.arange(0, T, rate, dtype=float32)`: value i is float32(rate * i), neighbours by truncation)."""
    spec = np.asarray(spec, dtype=np.complex128)
    if rate == 1.0:
        return spec
    lead = spec.shape[:-2]
    sp = spec.reshape((-1,) + spec.shape[-2:])
    frames = sp.shape[-1]
    n_out = int(math.ceil(frames / rate))
    ts = (rate * np.arange(n_out, dtype=np.float64)).astype(np.float32)
    alphas = np.fmod(ts, np.float32(1.0)).astype(np.float64)
    i0 = ts.astype(np.int64)
    i1 = (ts + np.float32(1.0)).astype(np.int64)
    phase_0 = np.angle(sp[..., :1])
    padded = np.concatenate([sp, np.zeros(sp.shape[:-1] + (2,), dtype=sp.dtype)], axis=-1)
    s0, s1 = padded[..., i0], padded[..., i1]
    pa = np.asarray(phase_advance, dtype=np.float64).reshape(-1, 1)
    phase = np.angle(s1) - np.angle(s0) - pa
    phase = phase - 2 * math.pi * np.round(phase / (2 * math.pi))
    phase = phase + pa
    phase = np.concatenate([phase_0, phase[..., :-1]], axis=-1)
    acc = np.cumsum(phase, axis=-1)
    mag = alphas * np.abs(s1) + (1 - alphas) * np.abs(s0)
    out = mag * np.exp(1j * acc)
    return out.reshape(lead + out.shape[1:])


def pitch_shift(x, sample_rate, n_steps, bins_per_octave=12, n_fft=512, win_length=None, hop_length=None, window=None):
    """reference functional.py:1579-1719."""
    x = np.asarray(x, dtype=np.float64)
    hop_length = n_fft // 4 if hop_length is None else hop_length
    win_length = n_fft if win_length is None else win_length
    window = hann_window(win_length) if window is None else np.asarray(window, dtype=np.float64)
    lead = x.shape[:-1]
    flat = x.reshape(-1, x.shape[-1])
    ori_len = x.shape[-1]
    rate = 2.0 ** (-float(n_steps) / bins_per_octave)
    spec = stft(flat, n_fft, hop_length, window, center=True, pad_mode="reflect")
    pa = np.linspace(0, math.pi * hop_length, spec.shape[-2])[:, None]
    stretched = istft(phase_vocoder(spec, rate, pa), n_fft, hop_length, win_length, window, length=int(round(ori_len / rate)))
    shifted = resample(stretched, int(sample_rate / rate), sample_rate)
    n = shifted.shape[-1]
    shifted = shifted[..., :ori_len] if n > ori_len else np.concatenate([shifted, np.zeros((shifted.shape[0], ori_len - n))], -1)
    return shifted.reshape(lead + (ori_len,))
