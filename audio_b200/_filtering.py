"""IIR filtering on the GPU: ``lfilter``, ``filtfilt``, the twelve ``*_biquad`` filters and pre-/de-emphasis, with the
signatures, defaults and errors of the reference (pytorch/audio/src/torchaudio/functional/filtering.py and
functional.py:2426-2473).  Every filter runs the chunked-scan kernels of ``csrc/lfilter.cu`` (b200audio::lfilter);
inside ``audio_b200.differentiable(filtering=True)`` the waveform and coefficient gradients run b200audio::lfilter_backward.

The biquad designs are the Audio-EQ-Cookbook and SoX formulas, evaluated with torch scalar ops in the waveform's dtype
and device, so a tensor ``cutoff_freq`` / ``Q`` / ``gain`` that requires grad gets its gradient through the
coefficient gradient.  The ``_design_*`` helpers return ``(b, a)`` as lists of three coefficients and run on any device.

``vad`` (filtering.py:1414-1702) measures on two front-end passes around the per-bin walk and the trigger kernel of
``csrc/vad.cu`` (b200audio::vad_walk, b200audio::vad_trigger) and returns a view of its input.
"""
from __future__ import annotations

import math
import warnings
from typing import List, Optional, Tuple

import torch
from torch import Tensor
from torch.autograd.function import once_differentiable

from . import _lib, _ops
from ._plans import FrontendPlan, _no_autograd, _require_cuda_f32, is_filtering_differentiable, pack_rows


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


# ---- vad (reference filtering.py:1414-1702) -----------------------------------------------------------------------
VAD_CHUNK = 1024  # measurement frames per chunk: 51 s at the default 20 Hz; the status is read back once per chunk


class VadPlan:
    """The host constants of one vad parameter set, computed with the reference's own Python-float and CPU-tensor
    arithmetic (filtering.py:1579-1629, so its errors are raised here, in its order), and per device the uploaded
    windows and the two prepared front-end workspaces: the measurement FFT (|X|, power 1) and the cepstrum FFT (power 2
    summed over the lifter band by a one-column indicator bank)."""

    def __init__(self, sample_rate, trigger_level=7.0, trigger_time=0.25, search_time=1.0, allowed_gap=0.25,
                 pre_trigger_time=0.0, boot_time=0.35, noise_up_time=0.1, noise_down_time=0.01,
                 noise_reduction_amount=1.35, measure_freq=20.0, measure_duration=None, measure_smooth_time=0.4,
                 hp_filter_freq=50.0, lp_filter_freq=6000.0, hp_lifter_freq=150.0, lp_lifter_freq=2000.0):
        measure_duration = 2.0 / measure_freq if measure_duration is None else measure_duration
        self.measure_len_ws = measure_len_ws = int(sample_rate * measure_duration + 0.5)
        dft_len_ws = 16
        while dft_len_ws < measure_len_ws:
            dft_len_ws *= 2
        self.dft_len_ws = dft_len_ws
        self.measure_period_ns = int(sample_rate / measure_freq + 0.5)
        self.measures_len = math.ceil(search_time * measure_freq)
        self.gap_len = int(allowed_gap * measure_freq + 0.5)
        self.fixed_pre_trigger_len_ns = int(pre_trigger_time * sample_rate + 0.5)
        self.samples_len_ns = (self.fixed_pre_trigger_len_ns + self.measures_len * self.measure_period_ns
                               + measure_len_ws)
        self.spectrum_window = torch.zeros(measure_len_ws)
        self.spectrum_window[:] = 2.0 / math.sqrt(float(measure_len_ws))
        self.spectrum_window *= torch.hann_window(measure_len_ws, dtype=torch.float)
        s0 = max(int(hp_filter_freq / sample_rate * dft_len_ws + 0.5), 1)
        s1 = min(int(lp_filter_freq / sample_rate * dft_len_ws + 0.5), dft_len_ws // 2)
        self.spectrum_start, self.spectrum_end = s0, s1
        self.cepstrum_window = torch.zeros(s1 - s0)
        self.cepstrum_window[:] = 2.0 / math.sqrt(float(s1) - s0)
        self.cepstrum_window *= torch.hann_window(s1 - s0, dtype=torch.float)
        c0 = math.ceil(sample_rate * 0.5 / lp_lifter_freq)
        c1 = min(math.floor(sample_rate * 0.5 / hp_lifter_freq), dft_len_ws // 4)
        if c1 <= c0:
            raise ValueError(
                "Expected cepstrum_start to be smaller than cepstrum_end."
                f"Found: cepstrum_start: {c0}, cepstrum_end: {c1}."
            )
        self.cepstrum_start, self.cepstrum_end = c0, c1
        self.noise_up_time_mult = math.exp(-1.0 / (noise_up_time * measure_freq))
        self.noise_down_time_mult = math.exp(-1.0 / (noise_down_time * measure_freq))
        self.measure_smooth_time_mult = math.exp(-1.0 / (measure_smooth_time * measure_freq))
        self.trigger_meas_time_mult = math.exp(-1.0 / (trigger_time * measure_freq))
        self.boot_count_max = int(boot_time * measure_freq - 0.5)
        self.noise_reduction_amount = noise_reduction_amount
        self.trigger_level = trigger_level
        self._devices = {}

    def desc(self, channels: int) -> "_lib.VadDesc":
        return _lib.VadDesc(
            channels=channels, dft_len=self.dft_len_ws, spectrum_start=self.spectrum_start,
            spectrum_end=self.spectrum_end, cepstrum_start=self.cepstrum_start, cepstrum_end=self.cepstrum_end,
            measures_len=self.measures_len, gap_len=self.gap_len, boot_count_max=self.boot_count_max,
            period=self.measure_period_ns, fixed_pre_trigger=self.fixed_pre_trigger_len_ns,
            noise_up_mult=self.noise_up_time_mult, noise_down_mult=self.noise_down_time_mult,
            noise_reduction_amount=self.noise_reduction_amount, measure_smooth_mult=self.measure_smooth_time_mult,
            trigger_mult=self.trigger_meas_time_mult, trigger_level=self.trigger_level)

    def num_frames(self, length: int) -> int:
        """Measurement frames the reference runs on `length` samples: len(range(measure_len_ws, length, period))."""
        return len(range(self.measure_len_ws, length, self.measure_period_ns))

    def device_state(self, device: torch.device):
        """(measurement plan, its workspace, cepstrum plan, its workspace, cepstrum window) on ``device``."""
        key = str(device)
        state = self._devices.get(key)
        if state is not None:
            return state
        if self.dft_len_ws > _lib.VAD_MAX_DFT:
            raise RuntimeError(
                f"audio_b200: vad with dft_len_ws = {self.dft_len_ws} (sample_rate * measure_duration = "
                f"{self.measure_len_ws} samples) is not supported: the measurement FFT is capped at {_lib.VAD_MAX_DFT} "
                "points (about 82 kHz at the default measure_duration); resample the input first")
        half = self.dft_len_ws // 2
        measure = FrontendPlan(FrontendPlan.make_desc(self.dft_len_ws, self.measure_len_ws, self.measure_period_ns, 0,
                                                      False, "constant", True, False, False, 1.0))
        cepstrum = FrontendPlan(FrontendPlan.make_desc(half, half, half, 0, False, "constant", True, False, False, 2.0,
                                                       n_mels=1))
        lifter = torch.zeros(half // 2 + 1, 1)
        lifter[self.cepstrum_start:self.cepstrum_end] = 1.0
        ones = torch.ones(half, device=device)
        state = (measure, measure.workspace(self.spectrum_window.to(device), None, None), cepstrum,
                 cepstrum.workspace(ones, lifter.to(device), None), self.cepstrum_window.to(device))
        self._devices[key] = state
        return state

    def run(self, x: Tensor, chunk: int = VAD_CHUNK, keep_measures: bool = False):
        """Measure the (C, L) CUDA float32 rows chunk by chunk until a frame triggers.  Returns (trigger frame or -1,
        trim start, the float32 measures of the frames run as a (C, frames) tensor or None)."""
        channels, length = x.shape
        frames = self.num_frames(length)
        if channels == 0 or frames == 0:
            return -1, 0, x.new_zeros(channels, 0) if keep_measures else None
        if self.measures_len < 1:
            raise RuntimeError(f"audio_b200: vad with search_time * measure_freq <= 0 (a measure ring of "
                               f"{self.measures_len} frames) is not supported")
        measure, ws_measure, cepstrum, ws_cepstrum, cep_window = self.device_state(x.device)
        m_i, m_f = measure._packed_desc()
        c_i, c_f = cepstrum._packed_desc()
        desc_i, desc_f = _ops.pack(self.desc(channels))
        dft, period, half = self.dft_len_ws, self.measure_period_ns, self.dft_len_ws // 2
        chunk = min(int(chunk), frames)
        lib = _lib.lib()
        nbytes = lib.b200a_vad_workspace_bytes(self.desc(channels), chunk)
        if nbytes == 0:
            raise _lib.B200AudioError(_lib.EUNSUPPORTED, "vad_workspace_bytes (descriptor rejected)")
        # the measured signal: (dft - ws) // 2 leading zeros centre the window in the FFT buffer as the reference's
        # left-aligned one (|X| is the same under the circular shift), trailing zeros complete the last frame
        left = (dft - self.measure_len_ws) // 2
        padded = x.new_zeros(channels, (frames - 1) * period + dft)
        n_copy = min(length, padded.shape[1] - left)
        padded[:, left:left + n_copy] = x[:, :n_copy]
        rows = x.new_zeros(channels, chunk * half)  # cepstrum rows; bins outside [s0, s1) stay zero
        ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
        kept = []
        for f0 in range(0, frames, chunk):
            k = min(chunk, frames - f0)
            span = padded[:, f0 * period:f0 * period + (k - 1) * period + dft]
            spec = _ops.frontend_run(span, ws_measure, m_i, m_f, _lib.STAGE_POWER, k, half + 1, padded.stride(0), None, 1)
            _ops.vad_walk(spec, cep_window, rows, ws, desc_i, desc_f, chunk, f0)
            power = _ops.frontend_run(rows[:, :k * half], ws_cepstrum, c_i, c_f, _lib.STAGE_MEL, k, 1, chunk * half,
                                      None, 1)
            meas = _ops.vad_trigger(power.view(channels, k), ws, desc_i, desc_f, chunk, f0)
            if keep_measures:
                kept.append(meas)
            trigger, start = ws[:16].view(torch.int64).tolist()
            if trigger >= 0:
                break
        return trigger, start, torch.cat(kept, 1) if keep_measures else None


_VAD_PLANS: "dict[tuple, VadPlan]" = {}


def vad_plan(sample_rate, *args) -> VadPlan:
    """One VadPlan per parameter tuple (the plan keeps one device state per device)."""
    key = (sample_rate,) + tuple(args)
    plan = _VAD_PLANS.get(key)
    if plan is None:
        plan = VadPlan(sample_rate, *args)
        if len(_VAD_PLANS) >= 64:
            _VAD_PLANS.pop(next(iter(_VAD_PLANS)))
        _VAD_PLANS[key] = plan
    return plan


def _warn_batch(waveform: Tensor) -> None:
    if waveform.ndim > 2:
        warnings.warn(
            "Expected input tensor dimension of 1 for single channel"
            f" or 2 for multi-channel. Got {waveform.ndim} instead. "
            "Batch semantics is not supported. "
            "Please refer to https://github.com/pytorch/audio/issues/1348"
            " and https://github.com/pytorch/audio/issues/1468."
        )


def _vad_trim(waveform: Tensor, plan: VadPlan, chunk: int = VAD_CHUNK) -> Tensor:
    """The reference's batch packing and output slicing (filtering.py:1632-1702) around ``plan.run``: the result is a
    view of ``waveform``, so autograd through the trim is the reference's."""
    _require_cuda_f32(waveform, "waveform")
    shape = waveform.size()
    waveform = waveform.view(-1, shape[-1])
    trigger, start, _ = plan.run(waveform.detach(), chunk)
    fixed_pre = plan.fixed_pre_trigger_len_ns
    if trigger < 0:
        if shape[-1] >= fixed_pre:
            return waveform[..., :fixed_pre].view(shape[:-1] + torch.Size([fixed_pre]))
        frames = plan.num_frames(shape[-1])
        pos = plan.measure_len_ws + (frames - 1) * plan.measure_period_ns if frames > 0 else 0
        start = max(pos - plan.samples_len_ns, 0)
    res = waveform[:, start:]
    return res.view(shape[:-1] + res.shape[-1:])


def vad(waveform: Tensor, sample_rate: int, trigger_level: float = 7.0, trigger_time: float = 0.25,
        search_time: float = 1.0, allowed_gap: float = 0.25, pre_trigger_time: float = 0.0, boot_time: float = 0.35,
        noise_up_time: float = 0.1, noise_down_time: float = 0.01, noise_reduction_amount: float = 1.35,
        measure_freq: float = 20.0, measure_duration: Optional[float] = None, measure_smooth_time: float = 0.4,
        hp_filter_freq: float = 50.0, lp_filter_freq: float = 6000.0, hp_lifter_freq: float = 150.0,
        lp_lifter_freq: float = 2000.0) -> Tensor:
    """Voice-activity trim from the front of ``(..., time)`` audio, as SoX's vad (reference filtering.py:1485-1702):
    every leading dimension is one channel of a single recording, trimmed jointly to the earliest activity in any
    channel.  Returns a view of ``waveform``; a waveform that requires grad gets 1 on the kept samples and 0 on the
    trimmed ones.  The measurements run on the GPU in chunks of frames and stop at the first triggering chunk;
    ``sample_rate * measure_duration`` is capped at 8192 samples (the measurement FFT)."""
    _warn_batch(waveform)
    plan = vad_plan(sample_rate, trigger_level, trigger_time, search_time, allowed_gap, pre_trigger_time, boot_time,
                    noise_up_time, noise_down_time, noise_reduction_amount, measure_freq, measure_duration,
                    measure_smooth_time, hp_filter_freq, lp_filter_freq, hp_lifter_freq, lp_lifter_freq)
    return _vad_trim(waveform, plan)
