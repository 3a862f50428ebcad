"""Host-side builders of the constant tables the kernels consume.

The tables (mel filterbank, DCT matrix, polyphase sinc taps) are *inputs* to the CUDA
kernels, built once at module construction.  They are evaluated with the same torch
CPU op sequence and dtypes as the reference so the resulting buffers are bit-identical
and ``state_dict``s interchange with torchaudio's (tests/test_constants.py checks this
against tests/golden/ref_cases.npz).

Reference (relative to pytorch/audio/src/torchaudio/functional/functional.py):
  melscale_fbanks 518-587 (+ _hz_to_mel 425-455, _mel_to_hz 458-489, triangles 492-515),
  create_dct 636-667, _get_sinc_resample_kernel 1305-1402.
"""
from __future__ import annotations

import math
import warnings
from typing import Optional

import torch

_KAISER_BETA_DEFAULT = 14.769656459379492
_SLANEY_LIN_HZ_PER_MEL = 200.0 / 3
_SLANEY_KNEE_HZ = 1000.0
_SLANEY_LOG_STEP = math.log(6.4) / 27.0


def _check_mel_scale(mel_scale: str) -> None:
    if mel_scale not in ("slaney", "htk"):
        raise ValueError('mel_scale should be one of "htk" or "slaney".')


def hz_to_mel(freq: float, mel_scale: str = "htk") -> float:
    _check_mel_scale(mel_scale)
    if mel_scale == "htk":
        return 2595.0 * math.log10(1.0 + (freq / 700.0))
    knee_mel = (_SLANEY_KNEE_HZ - 0.0) / _SLANEY_LIN_HZ_PER_MEL
    if freq >= _SLANEY_KNEE_HZ:
        return knee_mel + math.log(freq / _SLANEY_KNEE_HZ) / _SLANEY_LOG_STEP
    return (freq - 0.0) / _SLANEY_LIN_HZ_PER_MEL


def mel_to_hz(mels: torch.Tensor, mel_scale: str = "htk") -> torch.Tensor:
    _check_mel_scale(mel_scale)
    if mel_scale == "htk":
        return 700.0 * (10.0 ** (mels / 2595.0) - 1.0)
    knee_mel = (_SLANEY_KNEE_HZ - 0.0) / _SLANEY_LIN_HZ_PER_MEL
    hz = 0.0 + _SLANEY_LIN_HZ_PER_MEL * mels
    upper = mels >= knee_mel
    hz[upper] = _SLANEY_KNEE_HZ * torch.exp(_SLANEY_LOG_STEP * (mels[upper] - knee_mel))
    return hz


def triangular_filterbank(bin_hz: torch.Tensor, edge_hz: torch.Tensor) -> torch.Tensor:
    """(n_freqs,), (n_filter+2,) -> (n_freqs, n_filter) overlapping triangles."""
    span = edge_hz[1:] - edge_hz[:-1]
    offs = edge_hz.unsqueeze(0) - bin_hz.unsqueeze(1)
    falling = (-1.0 * offs[:, :-2]) / span[:-1]
    rising = offs[:, 2:] / span[1:]
    return torch.max(torch.zeros(1), torch.min(falling, rising))


def melscale_fbanks(
    n_freqs: int,
    f_min: float,
    f_max: float,
    n_mels: int,
    sample_rate: int,
    norm: Optional[str] = None,
    mel_scale: str = "htk",
) -> torch.Tensor:
    if norm is not None and norm != "slaney":
        raise ValueError('norm must be one of None or "slaney"')
    bin_hz = torch.linspace(0, sample_rate // 2, n_freqs)
    lo = hz_to_mel(f_min, mel_scale=mel_scale)
    hi = hz_to_mel(f_max, mel_scale=mel_scale)
    edge_hz = mel_to_hz(torch.linspace(lo, hi, n_mels + 2), mel_scale=mel_scale)
    fb = triangular_filterbank(bin_hz, edge_hz)
    if norm == "slaney":
        fb *= (2.0 / (edge_hz[2 : n_mels + 2] - edge_hz[:n_mels])).unsqueeze(0)
    if (fb.max(dim=0).values == 0.0).any():
        warnings.warn(
            "At least one mel filterbank has all zero values. "
            f"The value for `n_mels` ({n_mels}) may be set too high. "
            f"Or, the value for `n_freqs` ({n_freqs}) may be set too low."
        )
    return fb


def linear_fbanks(n_freqs: int, f_min: float, f_max: float, n_filter: int, sample_rate: int) -> torch.Tensor:
    """functional.linear_fbanks (functional.py:590-633) -- same triangles on a linear grid."""
    bin_hz = torch.linspace(0, sample_rate // 2, n_freqs)
    return triangular_filterbank(bin_hz, torch.linspace(f_min, f_max, n_filter + 2))


def create_dct(n_mfcc: int, n_mels: int, norm: Optional[str]) -> torch.Tensor:
    if norm is not None and norm != "ortho":
        raise ValueError('norm must be either "ortho" or None')
    pos = torch.arange(float(n_mels))
    order = torch.arange(float(n_mfcc)).unsqueeze(1)
    basis = torch.cos(math.pi / float(n_mels) * (pos + 0.5) * order)
    if norm is None:
        basis *= 2.0
    else:
        basis[0] *= 1.0 / math.sqrt(2.0)
        basis *= math.sqrt(2.0 / float(n_mels))
    return basis.t()


def sinc_resample_kernel(
    orig_freq: int,
    new_freq: int,
    gcd: int,
    lowpass_filter_width: int = 6,
    rolloff: float = 0.99,
    resampling_method: str = "sinc_interp_hann",
    beta: Optional[float] = None,
    device: torch.device = torch.device("cpu"),
    dtype: Optional[torch.dtype] = None,
):
    """Polyphase windowed-sinc taps, shape (new', 1, 2*width + orig'), and ``width``.

    dtype=None (the ``transforms.Resample`` default) evaluates in float64 and casts to
    float32 -- except the phase term, which the reference forms from a default-dtype
    (int64) arange divided by an int, i.e. float32 (functional.py:1378).  That quirk is
    reproduced so cached kernels are bit-identical.
    """
    if not (int(orig_freq) == orig_freq and int(new_freq) == new_freq):
        raise Exception(
            "Frequencies must be of integer type to ensure quality resampling computation. "
            "To work around this, manually convert both frequencies to integer values "
            "that maintain their resampling rate ratio before passing them into the function. "
            "Example: To downsample a 44100 hz waveform by a factor of 8, use "
            "`orig_freq=8` and `new_freq=1` instead of `orig_freq=44100` and `new_freq=5512.5`. "
            "For more information, please refer to https://github.com/pytorch/audio/issues/1487."
        )
    renamed = {"sinc_interpolation": "sinc_interp_hann", "kaiser_window": "sinc_interp_kaiser"}
    if resampling_method in renamed:
        warnings.warn(
            f'"{resampling_method}" resampling method name is being deprecated and replaced by '
            f'"{renamed[resampling_method]}" in the next release. '
            "The default behavior remains unchanged.",
            stacklevel=3,
        )
    elif resampling_method not in ("sinc_interp_hann", "sinc_interp_kaiser"):
        raise ValueError("Invalid resampling method: {}".format(resampling_method))

    orig_r = int(orig_freq) // gcd
    new_r = int(new_freq) // gcd
    if lowpass_filter_width <= 0:
        raise ValueError("Low pass filter width should be positive.")
    cutoff = min(orig_r, new_r)
    cutoff *= rolloff
    width = math.ceil(lowpass_filter_width * orig_r / cutoff)

    tap_dtype = torch.float64 if dtype is None else dtype
    tap_pos = torch.arange(-width, width + orig_r, dtype=tap_dtype, device=device)[None, None] / orig_r
    t = torch.arange(0, -new_r, -1, dtype=dtype, device=device)[:, None, None] / new_r + tap_pos
    t *= cutoff
    t = t.clamp_(-lowpass_filter_width, lowpass_filter_width)
    is_kaiser = resampling_method in ("sinc_interp_kaiser", "kaiser_window")
    if not is_kaiser:
        taper = torch.cos(t * math.pi / lowpass_filter_width / 2) ** 2
    else:
        b = torch.tensor(float(_KAISER_BETA_DEFAULT if beta is None else beta))
        taper = torch.i0(b * torch.sqrt(1 - (t / lowpass_filter_width) ** 2)) / torch.i0(b)
    t *= math.pi
    gain = cutoff / orig_r
    taps = torch.where(t == 0, torch.tensor(1.0).to(t), t.sin() / t)
    taps *= taper * gain
    if dtype is None:
        taps = taps.to(dtype=torch.float32)
    return taps, width
