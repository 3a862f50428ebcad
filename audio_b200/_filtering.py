"""IIR filtering on the GPU: ``lfilter``, ``filtfilt``, the twelve ``*_biquad`` filters and pre-/de-emphasis, with the
signatures, defaults and errors of the reference (pytorch/audio/src/torchaudio/functional/filtering.py and
functional.py:2426-2473).  Every filter runs the chunked-scan kernels of ``csrc/lfilter.cu`` (b200audio::lfilter);
inside ``audio_b200.differentiable(filtering=True)`` the waveform and coefficient gradients run b200audio::lfilter_backward.

The biquad designs are the Audio-EQ-Cookbook and SoX formulas, evaluated with torch scalar ops in the waveform's dtype
and device, so a tensor ``cutoff_freq`` / ``Q`` / ``gain`` that requires grad gets its gradient through the
coefficient gradient.  The ``_design_*`` helpers return ``(b, a)`` as lists of three coefficients and run on any device.
"""
from __future__ import annotations

import math
from typing import List, Tuple

import torch
from torch import Tensor
from torch.autograd.function import once_differentiable

from . import _lib, _ops
from ._plans import _no_autograd, _require_cuda_f32, is_filtering_differentiable, pack_rows


class _LfilterFunction(torch.autograd.Function):
    """b200audio::lfilter on the (batch, n_filters, T) rows with b200audio::lfilter_backward as its backward.  Saved
    (save_for_backward, so in-place edits are detected): the input rows, the unclamped output and the coefficients --
    not the FIR output the reference's autograd keeps."""

    @staticmethod
    def forward(ctx, x3, a, b, clamp, reverse):
        y, raw = _ops.lfilter(x3, a, b, clamp, reverse, clamp)
        ctx.save_for_backward(x3, raw if clamp else y, a, b)
        ctx.clamp, ctx.reverse = clamp, reverse
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x3, raw, a, b = ctx.saved_tensors
        gx, ga, gb = _ops.lfilter_backward(g, x3, raw, a, b, ctx.clamp, ctx.reverse)
        need = ctx.needs_input_grad
        return gx if need[0] else None, ga if need[1] else None, gb if need[2] else None, None, None


def _lfilter(waveform: Tensor, a_coeffs: Tensor, b_coeffs: Tensor, clamp: bool, batching: bool,
             reverse: bool = False) -> Tensor:
    if a_coeffs.size() != b_coeffs.size():
        raise ValueError(
            "Expected coeffs to be the same size."
            f"Found: a_coeffs size: {a_coeffs.size()}, b_coeffs size: {b_coeffs.size()}"
        )
    if a_coeffs.ndim > 2:
        raise ValueError(f"Expected coeffs to have greater than 1 dimension. Found: {a_coeffs.ndim}")
    if a_coeffs.ndim > 1 and batching:
        if waveform.ndim <= 0:
            raise ValueError("Expected waveform to have a positive number of dimensions." f"Found: {waveform.ndim}")
        if waveform.shape[-2] != a_coeffs.shape[0]:
            raise ValueError(
                "Expected number of batches in waveform and coeffs to be the same."
                f"Found: coeffs batches: {a_coeffs.shape[0]}, waveform batches: {waveform.shape[-2]}"
            )
    _require_cuda_f32(waveform, "waveform")
    _require_cuda_f32(a_coeffs, "a_coeffs")
    _require_cuda_f32(b_coeffs, "b_coeffs")
    for name, t in (("a_coeffs", a_coeffs), ("b_coeffs", b_coeffs)):
        if t.device != waveform.device:
            raise RuntimeError(f"audio_b200: {name} is on {t.device} but the waveform is on {waveform.device}")
    length = waveform.shape[-1]
    if a_coeffs.ndim > 1:
        n_filters = a_coeffs.shape[0]
        if batching:
            lead = waveform.shape[:-1]
            x3 = waveform.reshape(-1, n_filters, length)
        else:
            # one waveform row for every filter: a stride-0 view instead of the reference's stacked copy; autograd of
            # the view sums the waveform gradient over the filters
            lead = waveform.shape[:-1] + (n_filters,)
            x3 = pack_rows(waveform)[0].unsqueeze(1).expand(-1, n_filters, length)
    else:
        a_coeffs, b_coeffs = a_coeffs.unsqueeze(0), b_coeffs.unsqueeze(0)
        lead = waveform.shape[:-1]
        x3 = waveform.reshape(-1, 1, length)
    n_order = a_coeffs.shape[1]
    if n_order - 1 > _lib.LFILTER_MAX_ORDER:
        raise RuntimeError(
            f"audio_b200: lfilter of order {n_order - 1} ({n_order} coefficients) is not supported: the filter order is "
            f"capped at {_lib.LFILTER_MAX_ORDER} (B200A_LFILTER_MAX_ORDER); split the filter into second-order sections")
    if length > 1 and x3.stride(2) != 1:
        x3 = x3.contiguous()
    a2, b2 = a_coeffs.contiguous(), b_coeffs.contiguous()
    grad = torch.is_grad_enabled() and (waveform.requires_grad or a2.requires_grad or b2.requires_grad)
    if grad and not is_filtering_differentiable():
        for t in (waveform, a2, b2):
            _no_autograd(t)
    if grad:
        y = _LfilterFunction.apply(x3, a2, b2, bool(clamp), bool(reverse))
    else:
        y = _ops.lfilter(x3, a2, b2, bool(clamp), bool(reverse), False)[0]
    return y.reshape(lead + (length,))


def lfilter(waveform: Tensor, a_coeffs: Tensor, b_coeffs: Tensor, clamp: bool = True, batching: bool = True) -> Tensor:
    """IIR filter by its difference equation (reference filtering.py:1032-1099): ``(..., time)`` with 1-D
    ``(n_order,)`` coefficients, or ``(..., n_filters, time)`` with 2-D ``(n_filters, n_order)`` coefficients
    (``batching=False``: every filter on the same ``(..., time)`` waveform).  Coefficients are normalised by ``a0`` in
    float32, as the reference does; the output is clamped to [-1, 1] when ``clamp``.  Filter orders up to 16."""
    return _lfilter(waveform, a_coeffs, b_coeffs, clamp, batching)


def filtfilt(waveform: Tensor, a_coeffs: Tensor, b_coeffs: Tensor, clamp: bool = True) -> Tensor:
    """Forward-backward IIR filter (reference filtering.py:672-710): an unclamped forward pass, then the same filter
    run from the last sample down (no flipped copies), clamped when ``clamp``."""
    forward_filtered = _lfilter(waveform, a_coeffs, b_coeffs, False, True)
    return _lfilter(forward_filtered, a_coeffs, b_coeffs, clamp, True, reverse=True)


def biquad(waveform: Tensor, b0, b1, b2, a0, a1, a2) -> Tensor:
    """Second-order IIR filter with zero initial conditions (reference filtering.py:295-333); clamps to [-1, 1]."""
    dtype, device = waveform.dtype, waveform.device

    def vec(*cs):
        return torch.cat([torch.as_tensor(c, dtype=dtype, device=device).view(1) for c in cs])

    return lfilter(waveform, vec(a0, a1, a2), vec(b0, b1, b2))


# ---- designs (Audio-EQ-Cookbook, SoX) ----------------------------------------------------------------------------
Coeffs = Tuple[List, List]


def _scalar(v, dtype, device) -> Tensor:
    return torch.as_tensor(v, dtype=dtype, device=device)


def _angle(sample_rate, freq, Q, dtype, device):
    """w0 = 2 pi f0 / fs, cos(w0) and the cookbook's alpha = sin(w0) / (2 Q), as tensors."""
    freq, Q = _scalar(freq, dtype, device), _scalar(Q, dtype, device)
    w0 = 2 * math.pi * freq / sample_rate
    return w0, torch.cos(w0), torch.sin(w0) / 2 / Q


def _design_lowpass(sample_rate, cutoff_freq, Q, dtype, device) -> Coeffs:
    _, cw, alpha = _angle(sample_rate, cutoff_freq, Q, dtype, device)
    b0 = (1 - cw) / 2
    return [b0, 1 - cw, b0], [1 + alpha, -2 * cw, 1 - alpha]


def _design_highpass(sample_rate, cutoff_freq, Q, dtype, device) -> Coeffs:
    _, cw, alpha = _angle(sample_rate, cutoff_freq, Q, dtype, device)
    b0 = (1 + cw) / 2
    return [b0, -1 - cw, b0], [1 + alpha, -2 * cw, 1 - alpha]


def _design_allpass(sample_rate, central_freq, Q, dtype, device) -> Coeffs:
    _, cw, alpha = _angle(sample_rate, central_freq, Q, dtype, device)
    return [1 - alpha, -2 * cw, 1 + alpha], [1 + alpha, -2 * cw, 1 - alpha]


def _design_bandpass(sample_rate, central_freq, Q, const_skirt_gain, dtype, device) -> Coeffs:
    w0, cw, alpha = _angle(sample_rate, central_freq, Q, dtype, device)
    peak = torch.sin(w0) / 2 if const_skirt_gain else alpha  # constant skirt gain: peak gain Q instead of 0 dB
    return [peak, 0.0, -peak], [1 + alpha, -2 * cw, 1 - alpha]


def _design_bandreject(sample_rate, central_freq, Q, dtype, device) -> Coeffs:
    _, cw, alpha = _angle(sample_rate, central_freq, Q, dtype, device)
    return [1.0, -2 * cw, 1.0], [1 + alpha, -2 * cw, 1 - alpha]


def _design_band(sample_rate, central_freq, Q, noise, dtype, device) -> Coeffs:
    # SoX "band": a two-pole resonator whose pole radius follows the bandwidth f0 / Q
    central_freq, Q = _scalar(central_freq, dtype, device), _scalar(Q, dtype, device)
    w0 = 2 * math.pi * central_freq / sample_rate
    r2 = torch.exp(-2 * math.pi * (central_freq / Q) / sample_rate)
    a1 = -4 * r2 / (1 + r2) * torch.cos(w0)
    g = torch.sqrt(1 - a1 * a1 / (4 * r2)) * (1 - r2)
    if noise:  # unpitched mode: unit gain for white noise rather than at the centre frequency
        g = torch.sqrt(((1 + r2) * (1 + r2) - a1 * a1) * (1 - r2) / (1 + r2)) / g * g
    return [g, 0.0, 0.0], [1.0, a1, r2]


def _design_equalizer(sample_rate, center_freq, gain, Q, dtype, device) -> Coeffs:
    _, cw, alpha = _angle(sample_rate, center_freq, Q, dtype, device)
    A = torch.exp(_scalar(gain, dtype, device) / 40.0 * math.log(10))
    return [1 + alpha * A, -2 * cw, 1 - alpha * A], [1 + alpha / A, -2 * cw, 1 - alpha / A]


def _shelf_terms(A, cw, alpha):
    return 2 * torch.sqrt(A) * alpha, (A - 1) * cw, (A + 1) * cw


def _design_bass(sample_rate, gain, central_freq, Q, dtype, device) -> Coeffs:
    # low shelf, normalised by a0 before filtering (SoX's bass)
    _, cw, alpha = _angle(sample_rate, central_freq, Q, dtype, device)
    A = torch.exp(_scalar(gain, dtype, device) / 40 * math.log(10))
    sa, am, ap = _shelf_terms(A, cw, alpha)
    b = [A * ((A + 1) - am + sa), 2 * A * ((A - 1) - ap), A * ((A + 1) - am - sa)]
    a = [(A + 1) + am + sa, -2 * ((A - 1) + ap), (A + 1) + am - sa]
    a0 = a[0]
    return [c / a0 for c in b], [c / a0 for c in a]


def _design_treble(sample_rate, gain, central_freq, Q, dtype, device) -> Coeffs:
    # high shelf (SoX's treble)
    _, cw, alpha = _angle(sample_rate, central_freq, Q, dtype, device)
    A = torch.exp(_scalar(gain, dtype, device) / 40 * math.log(10))
    sa, am, ap = _shelf_terms(A, cw, alpha)
    b = [A * ((A + 1) + am + sa), -2 * A * ((A - 1) + ap), A * ((A + 1) + am - sa)]
    a = [(A + 1) - am + sa, 2 * ((A - 1) - ap), (A + 1) - am - sa]
    return b, a


_DEEMPH = {44100: (5283, 0.4845, -9.477), 48000: (5356, 0.479, -9.62)}  # ISO 908: (f0, shelf slope, gain dB)


def _design_deemph(sample_rate) -> Coeffs:
    if sample_rate not in _DEEMPH:
        raise ValueError("Sample rate must be 44100 (audio-CD) or 48000 (DAT)")
    f0, slope, gain = _DEEMPH[sample_rate]
    w0 = 2 * math.pi * f0 / sample_rate
    A = math.exp(gain / 40.0 * math.log(10))
    alpha = math.sin(w0) / 2 * math.sqrt((A + 1 / A) * (1 / slope - 1) + 2)  # the cookbook's shelf-slope form
    sa, am, ap = 2 * math.sqrt(A) * alpha, (A - 1) * math.cos(w0), (A + 1) * math.cos(w0)
    b = [A * ((A + 1) + am + sa), -2 * A * ((A - 1) + ap), A * ((A + 1) + am - sa)]
    a = [(A + 1) - am + sa, 2 * ((A - 1) - ap), (A + 1) - am - sa]
    return b, a


# RIAA playback: the (zeros, poles) of SoX's bilinear designs per sample rate
_RIAA = {
    44100: ((-0.2014898, 0.9233820), (0.7083149, 0.9924091)),
    48000: ((-0.1766069, 0.9321590), (0.7396325, 0.9931330)),
    88200: ((-0.1168735, 0.9648312), (0.8590646, 0.9964002)),
    96000: ((-0.1141486, 0.9676817), (0.8699137, 0.9966946)),
}


def _design_riaa(sample_rate) -> Coeffs:
    if sample_rate not in _RIAA:
        raise ValueError("Sample rate must be 44.1k, 48k, 88.2k, or 96k")
    (z0, z1), (p0, p1) = _RIAA[sample_rate]
    b = [1.0, -(z0 + z1), z0 * z1]  # monic polynomials with those roots
    a = [1.0, -(p0 + p1), p0 * p1]
    # scale b for 0 dB at 1 kHz: |H(e^{-iy})| = 1
    y = 2 * math.pi * 1000 / sample_rate
    b_re = b[0] + b[1] * math.cos(-y) + b[2] * math.cos(-2 * y)
    a_re = a[0] + a[1] * math.cos(-y) + a[2] * math.cos(-2 * y)
    b_im = b[1] * math.sin(-y) + b[2] * math.sin(-2 * y)
    a_im = a[1] * math.sin(-y) + a[2] * math.sin(-2 * y)
    g = 1 / math.sqrt((b_re**2 + b_im**2) / (a_re**2 + a_im**2))
    return [c * g for c in b], a


def _run(waveform: Tensor, coeffs: Coeffs) -> Tensor:
    b, a = coeffs
    return biquad(waveform, *b, *a)


def allpass_biquad(waveform: Tensor, sample_rate: int, central_freq: float, Q: float = 0.707) -> Tensor:
    return _run(waveform, _design_allpass(sample_rate, central_freq, Q, waveform.dtype, waveform.device))


def band_biquad(waveform: Tensor, sample_rate: int, central_freq: float, Q: float = 0.707, noise: bool = False) -> Tensor:
    return _run(waveform, _design_band(sample_rate, central_freq, Q, noise, waveform.dtype, waveform.device))


def bandpass_biquad(waveform: Tensor, sample_rate: int, central_freq: float, Q: float = 0.707,
                    const_skirt_gain: bool = False) -> Tensor:
    return _run(waveform, _design_bandpass(sample_rate, central_freq, Q, const_skirt_gain, waveform.dtype,
                                           waveform.device))


def bandreject_biquad(waveform: Tensor, sample_rate: int, central_freq: float, Q: float = 0.707) -> Tensor:
    return _run(waveform, _design_bandreject(sample_rate, central_freq, Q, waveform.dtype, waveform.device))


def bass_biquad(waveform: Tensor, sample_rate: int, gain: float, central_freq: float = 100, Q: float = 0.707) -> Tensor:
    return _run(waveform, _design_bass(sample_rate, gain, central_freq, Q, waveform.dtype, waveform.device))


def deemph_biquad(waveform: Tensor, sample_rate: int) -> Tensor:
    return _run(waveform, _design_deemph(sample_rate))


def equalizer_biquad(waveform: Tensor, sample_rate: int, center_freq: float, gain: float, Q: float = 0.707) -> Tensor:
    return _run(waveform, _design_equalizer(sample_rate, center_freq, gain, Q, waveform.dtype, waveform.device))


def highpass_biquad(waveform: Tensor, sample_rate: int, cutoff_freq: float, Q: float = 0.707) -> Tensor:
    return _run(waveform, _design_highpass(sample_rate, cutoff_freq, Q, waveform.dtype, waveform.device))


def lowpass_biquad(waveform: Tensor, sample_rate: int, cutoff_freq: float, Q: float = 0.707) -> Tensor:
    return _run(waveform, _design_lowpass(sample_rate, cutoff_freq, Q, waveform.dtype, waveform.device))


def riaa_biquad(waveform: Tensor, sample_rate: int) -> Tensor:
    return _run(waveform, _design_riaa(sample_rate))


def treble_biquad(waveform: Tensor, sample_rate: int, gain: float, central_freq: float = 3000, Q: float = 0.707) -> Tensor:
    return _run(waveform, _design_treble(sample_rate, gain, central_freq, Q, waveform.dtype, waveform.device))


def preemphasis(waveform: Tensor, coeff: float = 0.97) -> Tensor:
    """y[i] = x[i] - coeff * x[i - 1] along the last dimension (reference functional.py:2426-2446): an unclamped
    two-tap FIR through the same kernel."""
    _require_cuda_f32(waveform, "waveform")
    a = torch.tensor([1.0, 0.0], dtype=waveform.dtype, device=waveform.device)
    b = torch.tensor([1.0, -coeff], dtype=waveform.dtype, device=waveform.device)
    return lfilter(waveform, a, b, clamp=False)


def deemphasis(waveform: Tensor, coeff: float = 0.97) -> Tensor:
    """y[i] = x[i] + coeff * y[i - 1] (reference functional.py:2449-2473).  Clamped to [-1, 1], because the reference
    calls lfilter with its default ``clamp=True``."""
    _require_cuda_f32(waveform, "waveform")
    a = torch.tensor([1.0, -coeff], dtype=waveform.dtype, device=waveform.device)
    b = torch.tensor([1.0, 0.0], dtype=waveform.dtype, device=waveform.device)
    return lfilter(waveform, a, b)
