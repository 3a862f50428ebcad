"""Drop-in ``torchaudio.functional`` surface of the hot path, backed by libb200audio.so.

Same names, argument order, defaults and error behaviour as the reference
(pytorch/audio/src/torchaudio/functional/functional.py):
``spectrogram`` (54-145), ``melscale_fbanks`` (518-587), ``linear_fbanks`` (590-633),
``create_dct`` (636-667), ``amplitude_to_DB`` (356-404), ``resample`` (1435-1490) and the two
private helpers ``transforms`` imports (``_get_sinc_resample_kernel`` 1305-1402,
``_apply_sinc_resample_kernel`` 1405-1432).

Differences, all explicit (never a silent fallback): CUDA float32 tensors only, forward only except the waveform
gradient of ``spectrogram`` (and of the MelSpectrogram path) inside ``audio_b200.differentiable()``, the spectrogram
gradient of ``inverse_spectrogram`` inside ``audio_b200.differentiable(inverse=True)``, the waveform gradient of
``resample`` / ``speed`` inside ``audio_b200.differentiable(resample=True)``, and the input gradients of
``amplitude_to_DB``, ``spectral_centroid`` and the MFCC / LFCC / MelScale paths inside
``audio_b200.differentiable(features=True)``, and the spectrogram gradient of ``phase_vocoder`` and the waveform
gradient of ``pitch_shift`` inside ``audio_b200.differentiable(vocoder=True)``, and the waveform and coefficient
gradients of ``lfilter``, ``filtfilt``, the ``*_biquad`` filters, ``preemphasis`` and ``deemphasis``, and the input
gradients of ``fftconvolve`` and ``convolve``, inside ``audio_b200.differentiable(filtering=True)``.  ``griffinlim`` is
forward-only.

IIR filtering (reference functional/filtering.py): ``lfilter`` (1032-1099), ``filtfilt`` (672-710), ``biquad`` and the
``allpass`` / ``band`` / ``bandpass`` / ``bandreject`` / ``bass`` / ``deemph`` / ``equalizer`` / ``highpass`` /
``lowpass`` / ``riaa`` / ``treble`` ``_biquad`` designs, and ``preemphasis`` / ``deemphasis`` (functional.py:2426-2473),
all on one chunked-scan kernel family; filter orders up to 16.  ``vad`` (filtering.py:1485-1702): SoX's voice-activity
trim, measured on the GPU (the front end's FFT passes around a per-bin walk kernel), returning a view of its input.

FFT convolution: ``fftconvolve`` (functional.py:2222-2258), uniformly partitioned overlap-save on the kernels of
``csrc/convolve.cu``.  Direct convolution: ``convolve`` (functional.py:2261-2314), a banded TF32 x 3 tensor-core
product on the kernels of ``csrc/convolve_direct.cu``, for filters up to 4096 taps.

RNN-T loss: ``rnnt_loss`` (functional.py:1747-1796) on the kernels of ``csrc/rnnt_loss.cu``, float32 or float16 logits,
differentiable with respect to the logits without a switch.

CTC forced alignment: ``forced_align`` (functional/_alignment.py) on the kernels of ``csrc/forced_align.cu``, batched
with ragged lengths, bit-identical to the reference CPU per sequence; ``merge_tokens`` and ``TokenSpan`` on the host.

SpecAugment masking: ``mask_along_axis_iid`` (functional.py:813-882) and ``mask_along_axis`` (885-957) on the kernel of
``csrc/masking.cu``, with the reference's random draws, values bit for bit and output strides; differentiable with
respect to the input and a tensor ``mask_value`` without a switch.
"""
from __future__ import annotations

import collections
import math
import warnings
from dataclasses import dataclass
from typing import List, Optional, Tuple, Union

import torch
from torch import Tensor

from torch.autograd.function import once_differentiable

from . import _lib, _ops
from ._bookkeeping import resample_ratio
from ._constants import create_dct, linear_fbanks, melscale_fbanks, sinc_resample_kernel
from ._filtering import (allpass_biquad, band_biquad, bandpass_biquad, bandreject_biquad, bass_biquad,  # noqa: F401
                         biquad, deemph_biquad, deemphasis, equalizer_biquad, filtfilt, highpass_biquad, lfilter,
                         lowpass_biquad, preemphasis, riaa_biquad, treble_biquad, vad)
from ._masking import mask_along_axis, mask_along_axis_iid  # noqa: F401
from ._plans import (FrontendPlan, ResamplePlan, _no_autograd, _require_cuda_f32, _stream_ptr, _wants_grad,
                     is_feature_differentiable, is_filtering_differentiable, is_inverse_differentiable,
                     is_vocoder_differentiable, new_group_max, pack_rows, vocoder_chain)

__all__ = [
    "spectrogram",
    "inverse_spectrogram",
    "griffinlim",
    "phase_vocoder",
    "pitch_shift",
    "melscale_fbanks",
    "linear_fbanks",
    "create_dct",
    "amplitude_to_DB",
    "resample",
    "speed",
    "spectral_centroid",
    "mel_spectrogram",
    "mfcc",
    "lfilter",
    "filtfilt",
    "biquad",
    "allpass_biquad",
    "band_biquad",
    "bandpass_biquad",
    "bandreject_biquad",
    "bass_biquad",
    "deemph_biquad",
    "equalizer_biquad",
    "highpass_biquad",
    "lowpass_biquad",
    "riaa_biquad",
    "treble_biquad",
    "preemphasis",
    "deemphasis",
    "fftconvolve",
    "convolve",
    "vad",
    "rnnt_loss",
    "forced_align",
    "merge_tokens",
    "TokenSpan",
    "mask_along_axis",
    "mask_along_axis_iid",
]


_PLAN_CACHE: "dict[tuple, FrontendPlan]" = {}


def _plan_for(desc, device) -> FrontendPlan:
    """One FrontendPlan per (descriptor, device) for the functional entry points, so that repeated calls reuse the
    prepared workspace (the plan itself re-prepares when the window / filterbank tensors change)."""
    key = (tuple(None if (isinstance(v, float) and v != v) else v for v in desc.key()), str(device))  # NaN power -> None
    plan = _PLAN_CACHE.get(key)
    if plan is None:
        if len(_PLAN_CACHE) >= 64:
            _PLAN_CACHE.pop(next(iter(_PLAN_CACHE)))
        plan = _PLAN_CACHE[key] = FrontendPlan(desc)
    return plan


def _get_spec_norms(normalized: Union[str, bool]):
    """(frame_length_norm, window_norm) -- reference functional.py:228-242."""
    if isinstance(normalized, str):
        if normalized not in ("frame_length", "window"):
            raise ValueError("Invalid normalized parameter: {}".format(normalized))
        return normalized == "frame_length", normalized == "window"
    if isinstance(normalized, bool):
        return False, normalized
    raise TypeError("Input type not supported")


def _unpack(out: Tensor, waveform: Tensor) -> Tensor:
    """(rows, T, W[,2]) frame-major -> logical (..., W, T) view, as the reference returns it."""
    lead = waveform.shape[:-1]
    if out.dim() == 4:  # complex
        out = torch.view_as_complex(out)
    return out.reshape(lead + out.shape[-2:]).transpose(-1, -2)


def spectrogram(
    waveform: Tensor,
    pad: int,
    window: Tensor,
    n_fft: int,
    hop_length: int,
    win_length: int,
    power: Optional[float],
    normalized: Union[bool, str],
    center: bool = True,
    pad_mode: str = "reflect",
    onesided: bool = True,
    return_complex: Optional[bool] = None,
) -> Tensor:
    """``(..., time) -> (..., freq, time)``; one fused kernel (pad, frame, window, FFT, |.|^p)."""
    if return_complex is not None:
        warnings.warn(
            "`return_complex` argument is now deprecated and is not effective."
            "`torchaudio.functional.spectrogram(power=None)` always returns a tensor with "
            "complex dtype. Please remove the argument in the function call."
        )
    fl_norm, win_norm = _get_spec_norms(normalized)
    desc = FrontendPlan.make_desc(n_fft, win_length, hop_length, pad, center, pad_mode, onesided, fl_norm, win_norm, power)
    plan = _plan_for(desc, waveform.device)
    ws = plan.workspace(window, None, None)
    stage = _lib.STAGE_COMPLEX if power is None else _lib.STAGE_POWER
    return _unpack(plan.run(ws, stage, waveform, constants=(("window", window),)), waveform)


# ---- inverse spectrogram ------------------------------------------------------------------------------------
_ENVELOPE_OK: "collections.OrderedDict[tuple, Tensor]" = collections.OrderedDict()
_ENVELOPE_CACHE_SIZE = 64


def _check_window_envelope(window: Tensor, n_fft: int, win_length: int, hop: int, frames: int, start: int, end: int) -> None:
    """torch.istft refuses windows whose overlap-added square dips below 1e-11 inside the returned range
    ("window overlap add min"); it finds out with a device synchronisation, and so does this check -- once per
    (window tensor, geometry).  The cache entry HOLDS the window tensor, so its (data_ptr, _version) key cannot
    be matched by a different window that was handed the recycled allocation; the cache is a bounded LRU."""
    key = (window.data_ptr(), -1 if window.is_inference() else window._version, str(window.device), n_fft, win_length,
           hop, frames, start, end)
    if key in _ENVELOPE_OK:
        _ENVELOPE_OK.move_to_end(key)
        return
    import numpy as np

    w = np.zeros(n_fft, dtype=np.float64)
    left = (n_fft - win_length) // 2
    w[left:left + win_length] = window.detach().double().cpu().numpy()
    expected = n_fft + hop * (frames - 1)
    # overlap-added w^2 without a Python loop over frames: scatter-add over the (frames, n_fft) index grid
    env = np.zeros(expected)
    idx = (np.arange(frames)[:, None] * hop + np.arange(n_fft)[None, :]).ravel()
    np.add.at(env, idx, np.tile(w * w, frames))
    seg = env[start:min(end, expected)]
    if seg.size and np.abs(seg).min() < 1e-11:
        raise RuntimeError("istft(...) window overlap add min: 1 (the window envelope is zero inside the output range)")
    _ENVELOPE_OK[key] = window
    if len(_ENVELOPE_OK) > _ENVELOPE_CACHE_SIZE:
        _ENVELOPE_OK.popitem(last=False)


def inverse_spectrogram(
    spectrogram: Tensor,
    length: Optional[int],
    pad: int,
    window: Tensor,
    n_fft: int,
    hop_length: int,
    win_length: int,
    normalized: Union[bool, str],
    center: bool = True,
    pad_mode: str = "reflect",
    onesided: bool = True,
) -> Tensor:
    """``(..., freq, time)`` complex64 -> ``(..., time)``: least-squares inverse of ``spectrogram(power=None)``
    (reference functional.py:148-225 over ``torch.istft``).  Two kernels: Hermitian inverse FFT x window per frame pair,
    then overlap-add with window-envelope normalisation."""
    fl_norm, win_norm = _get_spec_norms(normalized)
    if not spectrogram.is_complex():
        raise ValueError("Expected `spectrogram` to be complex dtype.")
    if not spectrogram.is_cuda:
        raise RuntimeError(
            f"audio_b200: spectrogram is on '{spectrogram.device}'. This package runs only hand-written sm_90a CUDA "
            "kernels; there is no CPU or ATen fallback -- move the tensor (and the module) to a CUDA device."
        )
    if spectrogram.dtype != torch.complex64:
        raise TypeError(f"audio_b200: spectrogram must be complex64 (got {spectrogram.dtype})")
    if not onesided:
        raise NotImplementedError("audio_b200: inverse_spectrogram(onesided=False) is not implemented")
    grad = _wants_grad(spectrogram, (("window", window),), is_inverse_differentiable, "spectrogram")
    if not grad:
        _no_autograd(spectrogram)
    shape = spectrogram.size()
    n_bins, frames = shape[-2], shape[-1]
    if n_bins != n_fft // 2 + 1:
        raise RuntimeError(f"istft: expected {n_fft // 2 + 1} frequency bins for n_fft={n_fft}, got {n_bins}")
    spec3 = spectrogram.reshape(-1, n_bins, frames)
    desc = FrontendPlan.make_desc(n_fft, win_length, hop_length, 0, center, "reflect", True, fl_norm, win_norm, 2.0)
    plan = _plan_for(desc, spectrogram.device)
    ws = plan.workspace(window, None, None)
    expected = n_fft + hop_length * (frames - 1)
    start = n_fft // 2 if center else 0
    if length is not None:
        out_len = length + 2 * pad
    else:
        out_len = expected - 2 * start if center else expected
    if out_len <= 0:
        raise RuntimeError(f"istft: the requested signal is empty (frames={frames}, n_fft={n_fft})")
    _check_window_envelope(window, n_fft, win_length, hop_length, frames, start, start + out_len)
    if start + out_len > expected:
        warnings.warn("The length of signal is shorter than the length parameter. Result is being padded with zeros in "
                      "the tail. Please check your center and hop_length settings.")
    cut = pad if length is not None and pad > 0 else 0
    if grad:
        out = _IstftFunction.apply(spec3, ws, desc, start, out_len, cut)
    else:
        out = _istft_run(spec3, ws, desc, start, out_len, cut)
    return out.reshape(shape[:-2] + out.shape[-1:])


def _istft_run(spec3: Tensor, ws: Tensor, desc, start: int, out_len: int, cut: int) -> Tensor:
    """b200a_istft_run on the packed (rows, bins, frames) spectrogram: samples [start, start + out_len) of the
    overlap-added signal, less ``cut`` samples at each end."""
    rows, _, frames = spec3.shape
    dev = spec3.device
    real = torch.view_as_real(spec3)  # (rows, bins, frames, 2) float32 view, same storage
    with torch.cuda.device(dev):
        frame_buf = torch.empty((rows, frames, desc.n_fft), dtype=torch.float32, device=dev)
        out = torch.empty((rows, out_len), dtype=torch.float32, device=dev)
        rc = _lib.lib().b200a_istft_run(
            desc, ws.data_ptr(), real.data_ptr(), rows, frames, spec3.stride(0), spec3.stride(1), spec3.stride(2),
            frame_buf.data_ptr(), out.data_ptr(), out_len, start, out_len, _stream_ptr(dev),
        )
    _lib.check(rc, "istft_run")
    return out[:, cut:-cut] if cut > 0 else out


class _IstftFunction(torch.autograd.Function):
    """_istft_run with b200audio::istft_backward as its backward.  The map is linear, so nothing is saved but the
    forward's workspace: a window edited before backward does not change the gradient.  The ``cut`` slice happens
    inside, so autograd adds no slice_backward fill of the full-length gradient."""

    @staticmethod
    def forward(ctx, spec3, ws, desc, start, out_len, cut):
        ctx.ws, ctx.desc_lists, ctx.start, ctx.frames = ws, _ops.pack(desc), start + cut, spec3.shape[2]
        return _istft_run(spec3, ws, desc, start, out_len, cut)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        gz = _ops.istft_backward(g, ctx.ws, *ctx.desc_lists, ctx.start, ctx.frames)  # (rows, frames, bins, 2)
        return torch.view_as_complex(gz).transpose(1, 2), None, None, None, None, None


def griffinlim(
    specgram: Tensor,
    window: Tensor,
    n_fft: int,
    hop_length: int,
    win_length: int,
    power: float,
    n_iter: int,
    momentum: float,
    length: Optional[int],
    rand_init: bool,
) -> Tensor:
    """Fast Griffin-Lim phase recovery: ``(..., freq, time)`` |X|^power -> ``(..., time)`` (reference
    functional.py:255-353).  Every iteration is four launches on device-resident buffers: the phase step
    (``b200a_griffinlim_update``), the two inverse-STFT kernels, and the fused forward STFT (complex stage)."""
    if not 0 <= momentum < 1:
        raise ValueError("momentum must be in range [0, 1). Found: {}".format(momentum))
    momentum = momentum / (1 + momentum)
    _require_cuda_f32(specgram, "specgram")
    _no_autograd(specgram)
    shape = specgram.size()
    n_bins, frames = shape[-2], shape[-1]
    spec3 = specgram.reshape(-1, n_bins, frames)
    rows = spec3.shape[0]
    dev = specgram.device
    desc = FrontendPlan.make_desc(n_fft, win_length, hop_length, 0, True, "reflect", True, False, False, None)
    plan = _plan_for(desc, dev)
    ws = plan.workspace(window, None, None)
    expected = n_fft + hop_length * (frames - 1)
    start = n_fft // 2
    out_len = length if length is not None else expected - 2 * start
    _check_window_envelope(window, n_fft, win_length, hop_length, frames, start, start + out_len)
    lib = _lib.lib()
    stream = _stream_ptr(dev)
    with torch.cuda.device(dev):
        proj = torch.empty((rows, frames, n_bins, 2), dtype=torch.float32, device=dev)
        frame_buf = torch.empty((rows, frames, n_fft), dtype=torch.float32, device=dev)
        wave = torch.empty((rows, out_len), dtype=torch.float32, device=dev)
        rebuilt, tprev = None, None
        first_raw = False
        if rand_init:
            # the reference's own call (functional.py:310-311): uniform real and imaginary parts from torch's generator
            # on this device, in the (rows, freq, time) element order; used un-normalised for the first inversion
            init = torch.rand(spec3.size(), dtype=torch.complex64, device=dev)
            rebuilt = torch.view_as_real(init.transpose(1, 2).contiguous())
            first_raw = True

        def invert():
            rc = lib.b200a_istft_run(desc, ws.data_ptr(), proj.data_ptr(), rows, frames, frames * n_bins, 1, n_bins,
                                     frame_buf.data_ptr(), wave.data_ptr(), out_len, start, out_len, stream)
            _lib.check(rc, "istft_run")

        def step(raw=False):
            rc = lib.b200a_griffinlim_update(
                spec3.data_ptr(), spec3.stride(0), spec3.stride(1), spec3.stride(2), 1.0 / float(power),
                None if rebuilt is None else rebuilt.data_ptr(), None if tprev is None or not momentum else tprev.data_ptr(),
                float(momentum), 0 if raw else 1, proj.data_ptr(), rows, n_bins, frames, stream)
            _lib.check(rc, "griffinlim_update")

        for it in range(n_iter):
            step(raw=first_raw and it == 0)
            invert()
            new = plan.run(ws, _lib.STAGE_COMPLEX, wave)  # (rows, T', bins, 2) frame-major
            if new.shape[1] != frames:
                raise RuntimeError(
                    f"griffinlim: the rebuilt spectrogram has {new.shape[1]} frames, the input {frames} "
                    "(`length` is inconsistent with hop_length and the number of frames)"
                )
            tprev, rebuilt = (None if (first_raw and it == 0) else rebuilt), new
        step(raw=first_raw and n_iter == 0)
        invert()
    return wave.reshape(shape[:-2] + wave.shape[-1:])


def phase_vocoder(complex_specgrams: Tensor, rate: float, phase_advance: Tensor) -> Tensor:
    """Stretch a complex spectrogram in time by ``rate`` without modifying pitch: ``(..., freq, num_frame)`` ->
    ``(..., freq, ceil(num_frame / rate))`` (reference functional.py:713-803)."""
    if rate == 1.0:
        return complex_specgrams
    if not complex_specgrams.is_complex():
        raise ValueError("audio_b200: phase_vocoder expects a complex spectrogram")
    if not complex_specgrams.is_cuda:
        raise RuntimeError(
            f"audio_b200: complex_specgrams is on '{complex_specgrams.device}'. This package runs only hand-written "
            "sm_90a CUDA kernels; there is no CPU or ATen fallback -- move the tensor (and the module) to a CUDA device."
        )
    if complex_specgrams.dtype != torch.complex64:
        raise TypeError(f"audio_b200: complex_specgrams must be complex64 (got {complex_specgrams.dtype})")
    grad = _wants_grad(complex_specgrams, (("phase_advance", phase_advance),), is_vocoder_differentiable, "spectrogram")
    if not grad:
        _no_autograd(complex_specgrams)
    _require_cuda_f32(phase_advance, "phase_advance")
    shape = complex_specgrams.size()
    n_bins, frames = shape[-2], shape[-1]
    spec3 = complex_specgrams.reshape(-1, n_bins, frames)
    pa = phase_advance.reshape(-1).contiguous()
    if pa.numel() != n_bins:
        raise RuntimeError(f"phase_advance must have one entry per frequency bin ({n_bins}), got {pa.numel()}")
    if grad:
        res = _PhaseVocoderFunction.apply(spec3, float(rate), pa)
    else:
        res = _phase_vocoder_run(spec3, rate, pa)[1]
    return res.reshape(shape[:-2] + res.shape[1:])


def _phase_vocoder_run(spec3: Tensor, rate: float, pa: Tensor):
    """b200a_phase_vocoder on the packed (rows, bins, frames) spectrogram: the (rows, frames_out, bins, 2) frame-major
    buffer and the logical (rows, bins, frames_out) complex view of it."""
    rows, n_bins, frames = spec3.shape
    frames_out = int(math.ceil(frames / rate))  # len(torch.arange(0, frames, rate))
    dev = spec3.device
    with torch.cuda.device(dev):
        out = torch.empty((rows, frames_out, n_bins, 2), dtype=torch.float32, device=dev)
        rc = _lib.lib().b200a_phase_vocoder(
            torch.view_as_real(spec3).data_ptr(), spec3.stride(0), spec3.stride(1), spec3.stride(2), rows, n_bins, frames,
            float(rate), pa.data_ptr(), out.data_ptr(), frames_out, _stream_ptr(dev))
    _lib.check(rc, "phase_vocoder")
    return out, torch.view_as_complex(out).transpose(-1, -2)  # logical (rows, freq, frames_out) over the buffer


class _PhaseVocoderFunction(torch.autograd.Function):
    """_phase_vocoder_run with b200audio::phase_vocoder_backward as its backward.  The backward needs the forward's input
    and output and nothing else (no angles, no phase_advance, no recompute); both go through save_for_backward, so an
    in-place edit of either before backward is an error."""

    @staticmethod
    def forward(ctx, spec3, rate, pa):
        out, res = _phase_vocoder_run(spec3, rate, pa)
        ctx.save_for_backward(spec3, out)
        ctx.rate = rate
        return res

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        spec3, out = ctx.saved_tensors
        gx = _ops.phase_vocoder_backward(spec3, out, g, ctx.rate)  # (rows, frames_in, bins, 2)
        return torch.view_as_complex(gx).transpose(1, 2), None, None


def pitch_shift(
    waveform: Tensor,
    sample_rate: int,
    n_steps: int,
    bins_per_octave: int = 12,
    n_fft: int = 512,
    win_length: Optional[int] = None,
    hop_length: Optional[int] = None,
    window: Optional[Tensor] = None,
) -> Tensor:
    """Shift the pitch of a waveform by ``n_steps`` steps (reference functional.py:1579-1719): STFT -> phase vocoder
    (rate 2^(-n_steps / bins_per_octave)) -> inverse STFT -> resample back to the original duration -> crop / zero-pad
    to the input length.  Five kernels of this library, no host round trip.  Inside
    ``audio_b200.differentiable(vocoder=True)`` the waveform gradient runs their five adjoints."""
    _require_cuda_f32(waveform, "waveform")
    if hop_length is None:
        hop_length = n_fft // 4
    if win_length is None:
        win_length = n_fft
    if window is None:
        window = torch.hann_window(window_length=win_length, device=waveform.device)
    with vocoder_chain(waveform):
        return _pitch_shift(waveform, sample_rate, n_steps, bins_per_octave, n_fft, win_length, hop_length, window)


def _pitch_shift(waveform, sample_rate, n_steps, bins_per_octave, n_fft, win_length, hop_length, window) -> Tensor:
    shape = waveform.size()
    flat = waveform.reshape(-1, shape[-1])
    ori_len = shape[-1]
    rate = 2.0 ** (-float(n_steps) / bins_per_octave)
    spec_f = spectrogram(flat, 0, window, n_fft, hop_length, win_length, None, False)
    phase_advance = torch.linspace(0, math.pi * hop_length, spec_f.shape[-2], device=spec_f.device)[..., None]
    spec_stretch = phase_vocoder(spec_f, rate, phase_advance)
    len_stretch = int(round(ori_len / rate))
    stretched = inverse_spectrogram(spec_stretch, len_stretch, 0, window, n_fft, hop_length, win_length, False)
    shifted = resample(stretched, int(sample_rate / rate), sample_rate)
    shift_len = shifted.size()[-1]
    if shift_len > ori_len:
        shifted = shifted[..., :ori_len]
    else:
        shifted = torch.nn.functional.pad(shifted, [0, ori_len - shift_len])
    return shifted.reshape(shape[:-1] + shifted.shape[-1:])


def _db_groups(shape) -> int:
    """How many independent top_db cut-offs the reference uses for a tensor of this shape
    (functional.py:395-399: dims beyond the last three are separate items)."""
    groups = 1
    for s in shape[:-3]:
        groups *= s
    return groups


def amplitude_to_DB(
    x: Tensor, multiplier: float, amin: float, db_multiplier: float, top_db: Optional[float] = None
) -> Tensor:
    _require_cuda_f32(x, "x")
    if _wants_grad(x, (), is_feature_differentiable, "x"):
        return _AmplitudeToDBFunction.apply(x, float(multiplier), float(amin), float(multiplier) * float(db_multiplier),
                                            top_db)
    _no_autograd(x)
    return _amplitude_to_db_run(x.contiguous(), multiplier, amin, float(multiplier) * float(db_multiplier), top_db)[0]


def _amplitude_to_db_run(xc: Tensor, multiplier: float, amin: float, offset: float, top_db: Optional[float]):
    """b200a_amplitude_to_db on the contiguous ``xc``: (output, group maxima or None, groups)."""
    out = torch.empty_like(xc)
    if xc.numel() == 0:
        return out, None, 0
    groups = _db_groups(xc.shape) if top_db is not None else 1
    dev = xc.device
    with torch.cuda.device(dev):
        scratch = torch.empty(groups, dtype=torch.float32, device=dev)
        rc = _lib.lib().b200a_amplitude_to_db(
            xc.data_ptr(), groups, xc.numel() // groups, float(multiplier), float(amin), float(offset),
            -1.0 if top_db is None else float(top_db), scratch.data_ptr(), out.data_ptr(), _stream_ptr(dev),
        )
    _lib.check(rc, "amplitude_to_db")
    return out, scratch if top_db is not None else None, groups


class _AmplitudeToDBFunction(torch.autograd.Function):
    """amplitude_to_DB with b200audio::amplitude_to_db_backward as its backward.  Saved: the input (save_for_backward,
    so in-place edits of it are detected) and the forward's group maxima, against which the backward's recomputed dB
    values tie exactly."""

    @staticmethod
    def forward(ctx, x, multiplier, amin, offset, top_db):
        xc = x.contiguous()
        out, gmax, groups = _amplitude_to_db_run(xc, multiplier, amin, offset, top_db)
        ctx.save_for_backward(x)
        ctx.xc = None if xc is x else xc
        ctx.gmax, ctx.args = gmax, (groups, multiplier, amin, offset, -1.0 if top_db is None else float(top_db))
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        xc = x if ctx.xc is None else ctx.xc
        if xc.numel() == 0:
            return torch.zeros_like(xc), None, None, None, None
        return _ops.amplitude_to_db_backward(g, xc, ctx.gmax, *ctx.args), None, None, None, None


def _apply_fbank(specgram: Tensor, fb: Tensor) -> Tensor:
    """MelScale.forward on an existing spectrogram of logical shape (..., n_bins, T)."""
    _require_cuda_f32(specgram, "specgram")
    _require_cuda_f32(fb, "fb")
    grad = _wants_grad(specgram, (("fb", fb),), is_feature_differentiable, "spectrogram")
    if not grad:
        _no_autograd(specgram)
    n_bins, frames = specgram.shape[-2], specgram.shape[-1]
    if fb.shape[0] != n_bins:
        raise RuntimeError(f"mat1 and mat2 shapes cannot be multiplied: n_bins={n_bins} vs fb {tuple(fb.shape)}")
    lead = specgram.shape[:-2]
    s3 = specgram.reshape((-1, n_bins, frames))
    out = _MelScaleFunction.apply(s3, fb) if grad else _apply_fbank_run(s3, fb)
    return out.reshape(lead + out.shape[-2:]).transpose(-1, -2)


def _apply_fbank_run(s3: Tensor, fb: Tensor) -> Tensor:
    """b200a_apply_fbank on the (rows, n_bins, T) spectrogram: the frame-major (rows, T, n_filters) product."""
    rows, n_bins, frames = s3.shape
    fbc = fb.contiguous()
    dev = s3.device
    with torch.cuda.device(dev):
        out = torch.empty((rows, frames, fb.shape[1]), dtype=torch.float32, device=dev)
        rc = _lib.lib().b200a_apply_fbank(
            s3.data_ptr(), rows, n_bins, frames, s3.stride(0), s3.stride(1), s3.stride(2),
            fbc.data_ptr(), fb.shape[1], out.data_ptr(), _stream_ptr(dev),
        )
    _lib.check(rc, "apply_fbank")
    return out


class _MelScaleFunction(torch.autograd.Function):
    """MelScale on its own with b200audio::apply_fbank_backward as its backward.  The map is linear in the spectrogram:
    only the filterbank is saved (save_for_backward, so an in-place edit of it before backward is an error, as it is for
    torch's matmul)."""

    @staticmethod
    def forward(ctx, s3, fb):
        ctx.save_for_backward(fb)
        return _apply_fbank_run(s3, fb)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        (fb,) = ctx.saved_tensors
        return _ops.apply_fbank_backward(g, fb.contiguous()).transpose(1, 2), None


# ---- fused MelSpectrogram / MFCC (what the transforms call) -----------------------------------
def mel_spectrogram(plan: FrontendPlan, window: Tensor, fb: Tensor, waveform: Tensor) -> Tensor:
    """Spectrogram + MelScale in ONE kernel: ``(..., time) -> (..., n_mels, time)``."""
    ws = plan.workspace(window, fb, None)
    return _unpack(plan.run(ws, _lib.STAGE_MEL, waveform, constants=(("window", window), ("fb", fb))), waveform)


def mfcc(
    plan: FrontendPlan,
    window: Tensor,
    fb: Tensor,
    dct_mat: Tensor,
    waveform: Tensor,
    top_db: Optional[float],
    log_mels: bool,
    process_group=None,
    fb_name: str = "fb",
) -> Tensor:
    """MelSpectrogram -> dB/log -> DCT: fused front-end kernel + clamp/DCT kernel.

    The only cross-utterance coupling on the path is AmplitudeToDB's ``top_db`` clamp
    (reference functional.py:395-399): for a waveform of dim <= 2 ONE maximum is shared by the
    whole batch, for dim >= 3 each leading item has its own.  ``process_group`` (optional)
    extends the shared maximum across ranks with one all-reduce(MAX) of that scalar.

    Inside ``audio_b200.differentiable(features=True)`` a waveform that requires grad gets its gradient
    (``_MfccFunction``); ``fb_name`` names the filterbank buffer in the error for one that requires grad.
    """
    ws = plan.workspace(window, fb, dct_mat)
    rows = 1
    for s in waveform.shape[:-1]:
        rows *= s
    clamp = (not log_mels) and top_db is not None
    if clamp:
        rows_per_group = waveform.shape[-2] if waveform.dim() >= 2 else 1
        rows_per_group = max(int(rows_per_group), 1)
        groups = max((rows + rows_per_group - 1) // rows_per_group, 1)
    else:
        rows_per_group, groups = 1, 0
    _require_cuda_f32(waveform, "waveform")
    if _wants_grad(waveform, (("window", window), (fb_name, fb), ("dct_mat", dct_mat)), is_feature_differentiable):
        if process_group is not None:
            raise RuntimeError(
                "audio_b200: MFCC / LFCC gradients with a process_group are not implemented (the sharded backward would "
                "need the routed top_db sums all-reduced and the group maximum located across ranks); set "
                "process_group = None, or detach() the waveform"
            )
        out = plan.mfcc_grad(ws, waveform, groups, rows_per_group, top_db if clamp else None)
        return _unpack(out, waveform)
    gmax = new_group_max(groups, waveform.device) if clamp else None
    feat = plan.run(ws, _lib.STAGE_FEAT, waveform, gmax, rows_per_group)
    if clamp and waveform.dim() <= 2:
        gmax = _exchange_group_max(gmax, process_group)
    out = plan.mfcc_finish(ws, feat, gmax, rows_per_group, top_db if clamp else None)
    return _unpack(out, waveform)


def _exchange_group_max(gmax: Tensor, process_group) -> Tensor:
    """The path's only cross-rank message: all-reduce(MAX) of the running dB maximum of a 2-D batch that is sharded
    over ``process_group`` (reference semantics: ONE ``amax`` over the whole batch, functional.py:395-399).
    In place; a ``None`` group (single process) is the identity."""
    if process_group is not None:
        import torch.distributed as dist

        dist.all_reduce(gmax, op=dist.ReduceOp.MAX, group=process_group)
    return gmax


# ---- resampling ---------------------------------------------------------------------------------
def _get_sinc_resample_kernel(
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
    return sinc_resample_kernel(
        orig_freq, new_freq, gcd, lowpass_filter_width, rolloff, resampling_method, beta, device, dtype
    )


def _apply_sinc_resample_kernel(
    waveform: Tensor, orig_freq: int, new_freq: int, gcd: int, kernel: Tensor, width: int, plan: Optional[ResamplePlan] = None
) -> Tensor:
    if not waveform.is_floating_point():
        raise TypeError(f"Expected floating point type for waveform tensor, but received {waveform.dtype}.")
    if plan is None:
        plan = ResamplePlan(int(orig_freq) // gcd, int(new_freq) // gcd, width)
    return plan.run(kernel, waveform)


def resample(
    waveform: Tensor,
    orig_freq: int,
    new_freq: int,
    lowpass_filter_width: int = 6,
    rolloff: float = 0.99,
    resampling_method: str = "sinc_interp_hann",
    beta: Optional[float] = None,
) -> Tensor:
    if orig_freq <= 0.0 or new_freq <= 0.0:
        raise ValueError("Original frequency and desired frequecy should be positive")
    if orig_freq == new_freq:
        return waveform
    if not waveform.is_floating_point():
        raise TypeError(f"Expected floating point type for waveform tensor, but received {waveform.dtype}.")
    _require_cuda_f32(waveform, "waveform")
    gcd = math.gcd(int(orig_freq), int(new_freq))
    # the reference builds the taps on the waveform's device in its dtype (functional.py:1478-1488);
    # that is a handful of tiny torch elementwise launches at call time -- table building, not the hot path
    kernel, width = sinc_resample_kernel(
        orig_freq, new_freq, gcd, lowpass_filter_width, rolloff, resampling_method, beta, waveform.device, waveform.dtype
    )
    return _apply_sinc_resample_kernel(waveform, orig_freq, new_freq, gcd, kernel, width)


def speed(waveform: Tensor, orig_freq: int, factor: float, lengths: Optional[Tensor] = None):
    """Adjusts waveform speed (reference functional.py:2384-2423): ``resample`` from ``int(factor * orig_freq)`` to
    ``orig_freq``; returns ``(waveform', lengths')``."""
    source, target = int(factor * orig_freq), int(orig_freq)
    g = math.gcd(source, target)
    source, target = source // g, target // g
    out_lengths = None if lengths is None else torch.ceil(lengths * target / source).to(lengths.dtype)
    return resample(waveform, source, target), out_lengths


# ---- spectral centroid (SURVEY.md 8f: a weighted-sum epilogue of the same fused kernel) --------------
def spectral_centroid(
    waveform: Tensor,
    sample_rate: int,
    pad: int,
    window: Tensor,
    n_fft: int,
    hop_length: int,
    win_length: int,
) -> Tensor:
    """``(..., time) -> (..., frames)``: sum_k f_k |X_k| / sum_k |X_k| (reference functional.py:1257-1299).

    The magnitude spectrogram is contracted inside the fused kernel with the two-column matrix
    ``[bin frequency | 1]`` (the mel stage with a 2-filter bank), then one tiny kernel divides the pair.
    """
    _require_cuda_f32(waveform, "waveform")
    desc = FrontendPlan.make_desc(n_fft, win_length, hop_length, pad, True, "reflect", True, False, False, 1.0, n_mels=2)
    plan = FrontendPlan(desc)
    dev = waveform.device
    freqs = torch.linspace(0, sample_rate // 2, steps=1 + n_fft // 2, device=dev)
    fb = torch.stack([freqs, torch.ones_like(freqs)], dim=1).contiguous()
    ws = plan.workspace(window, fb, None)
    # with the feature switch on, the mel stage differentiates (_FrontendFunction) and so does the ratio
    constants = (("window", window),)
    grad = _wants_grad(waveform, constants, is_feature_differentiable)
    pairs = plan.run(ws, _lib.STAGE_MEL, waveform, constants=constants if grad else None,
                     switch=is_feature_differentiable)  # (rows, T, 2)
    out = _RatioFunction.apply(pairs) if grad else _ratio_run(pairs)
    return out.reshape(waveform.shape[:-1] + (out.shape[1],))


def _ratio_run(pairs: Tensor) -> Tensor:
    """b200a_ratio_f32 on the (rows, T, 2) pairs: (rows, T) ratios."""
    rows, frames, _ = pairs.shape
    dev = pairs.device
    with torch.cuda.device(dev):
        out = torch.empty((rows, frames), dtype=torch.float32, device=dev)
        rc = _lib.lib().b200a_ratio_f32(pairs.data_ptr(), rows * frames, out.data_ptr(), _stream_ptr(dev))
    _lib.check(rc, "ratio_f32")
    return out


class _RatioFunction(torch.autograd.Function):
    """SpectralCentroid's N / D per frame with b200audio::ratio_backward as its backward; the pairs are saved."""

    @staticmethod
    def forward(ctx, pairs):
        ctx.save_for_backward(pairs)
        return _ratio_run(pairs)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        (pairs,) = ctx.saved_tensors
        return _ops.ratio_backward(g, pairs)


# ---- FFT convolution (reference functional.py:2189-2258) -------------------------------------------------------
def _check_shape_compatible(x: Tensor, y: Tensor) -> None:
    if x.ndim != y.ndim:
        raise ValueError(f"The operands must be the same dimension (got {x.ndim} and {y.ndim}).")
    for i in range(x.ndim - 1):
        xi, yi = x.size(i), y.size(i)
        if xi == yi or xi == 1 or yi == 1:
            continue
        raise ValueError(f"Leading dimensions of x and y are not broadcastable (got {x.shape} and {y.shape}).")


def _check_convolve_mode(mode: str) -> None:
    valid_convolve_modes = ["full", "valid", "same"]
    if mode not in valid_convolve_modes:
        raise ValueError(f"Unrecognized mode value '{mode}'. Please specify one of {valid_convolve_modes}.")


def _convolve_slice(n: int, m: int, mode: str):
    """(start, length) of ``_apply_convolve_mode``'s slice of the full (n + m - 1)-sample result, with Python's slice
    rules (a negative start counts from the end, as the reference's slicing does for an empty operand)."""
    full = n + m - 1
    if mode == "full":
        return 0, full
    target = max(n, m) - min(n, m) + 1 if mode == "valid" else n
    start = (full - target) // 2
    lo, hi, _ = slice(start, start + target).indices(full)
    return lo, max(hi - lo, 0)


def _conv_function(name: str, run, backward_op):
    """An autograd Function for an operand-row convolution op (``run``: b200audio::fftconvolve or b200audio::convolve)
    with ``backward_op`` as its backward.  Saved (save_for_backward): the two operands' rows only.  The per-output-row
    gradients are summed onto the operand rows that broadcasting shared (``sum_to_size``: a fixed-order reduction, no
    atomics)."""

    class Fn(torch.autograd.Function):
        @staticmethod
        def forward(ctx, x2, y2, ix, iy, start, out_len, shapes):
            ctx.save_for_backward(x2, y2)
            ctx.ix, ctx.iy, ctx.start, ctx.shapes = ix, iy, start, shapes
            return run(x2, y2, ix, iy, start, out_len)

        @staticmethod
        @once_differentiable
        def backward(ctx, g):
            x2, y2 = ctx.saved_tensors
            gx, gy = backward_op(g, x2, y2, ctx.ix, ctx.iy, ctx.start)
            lo, lx, ly = ctx.shapes
            need = ctx.needs_input_grad
            gx = gx.reshape(lo + (x2.shape[1],)).sum_to_size(lx + (x2.shape[1],)).reshape(x2.shape) if need[0] else None
            gy = gy.reshape(lo + (y2.shape[1],)).sum_to_size(ly + (y2.shape[1],)).reshape(y2.shape) if need[1] else None
            return gx, gy, None, None, None, None, None

    Fn.__name__ = Fn.__qualname__ = name
    Fn.run = staticmethod(run)
    return Fn


_FFTConvolveFunction = _conv_function("_FFTConvolveFunction", _ops.fftconvolve, _ops.fftconvolve_backward)
_ConvolveFunction = _conv_function("_ConvolveFunction", _ops.convolve, _ops.convolve_backward)


def _convolve_operands(x: Tensor, y: Tensor, mode: str):
    """The checks fftconvolve and convolve share, in the reference's order, then the package's: shapes, mode, CUDA
    float32, one device.  Returns (n, m, lx, ly, lo): the lengths, both operands' leading shapes and the output's."""
    _check_shape_compatible(x, y)
    _check_convolve_mode(mode)
    _require_cuda_f32(x, "x")
    _require_cuda_f32(y, "y")
    if y.device != x.device:
        raise RuntimeError(f"audio_b200: y is on {y.device} but x is on {x.device}")
    lx, ly = tuple(x.shape[:-1]), tuple(y.shape[:-1])
    return x.shape[-1], y.shape[-1], lx, ly, tuple(torch.broadcast_shapes(lx, ly))


def _convolve_rows(fn, x: Tensor, y: Tensor, lx, ly, lo, start: int, out_len: int) -> Tensor:
    """Runs ``fn`` (a _conv_function) on the operands' rows for the output slice [start, start + out_len) of every
    output row, under the filtering gradient switch; returns the (lo..., out_len) output."""
    x2, _ = pack_rows(x)
    y2, _ = pack_rows(y)
    dev = x.device
    # output row -> operand row, by broadcasting the operands' row numbers on the device (no host synchronisation); the
    # kernels read one int64 per output row, so the vectors are materialised (a broadcast view may have stride 0)
    ix = torch.arange(x2.shape[0], device=dev).reshape(lx).broadcast_to(lo).contiguous().reshape(-1)
    iy = torch.arange(y2.shape[0], device=dev).reshape(ly).broadcast_to(lo).contiguous().reshape(-1)
    grad = torch.is_grad_enabled() and (x.requires_grad or y.requires_grad)
    if grad and not is_filtering_differentiable():
        _no_autograd(x)
        _no_autograd(y)
    if grad:
        out = fn.apply(x2, y2, ix, iy, start, out_len, (lo, lx, ly))
    else:
        out = fn.run(x2, y2, ix, iy, start, out_len)
    return out.reshape(lo + (out_len,))


def fftconvolve(x: Tensor, y: Tensor, mode: str = "full") -> Tensor:
    """Convolves ``x (..., N)`` and ``y (..., M)`` along their last dimension (reference functional.py:2222-2258): the
    true convolution, leading dimensions broadcast, output ``(..., L)`` with L = N + M - 1 (``"full"``),
    max(N, M) - min(N, M) + 1 (``"valid"``) or N (``"same"``).  Runs uniformly partitioned overlap-save
    (``csrc/convolve.cu``): the shorter operand is cut into blocks of B = 256 .. 2048 samples, and only the output
    blocks the mode returns are computed.  The shorter operand may have up to 128 * 2048 = 262144 samples."""
    n, m, lx, ly, lo = _convolve_operands(x, y, mode)
    if n + m - 1 <= 0:  # what torch.fft.rfft reports for the reference's n = N + M - 1 points
        raise RuntimeError(f"Invalid number of data points ({n + m - 1}) specified")
    start, out_len = _convolve_slice(n, m, mode)
    if n == 0 or m == 0:
        return x.new_zeros(lo + (out_len,))  # the transform of an empty operand is zero
    k = min(n, m)
    block = min(max(1 << (k - 1).bit_length(), 256), _lib.FFTCONVOLVE_MAX_BLOCK)
    if -(-k // block) > _lib.FFTCONVOLVE_MAX_PARTITIONS:
        raise RuntimeError(
            f"audio_b200: fftconvolve of a {k}-sample shorter operand is not supported: it is capped at "
            f"{_lib.FFTCONVOLVE_MAX_PARTITIONS} partitions of {block} samples (B200A_FFTCONVOLVE_MAX_PARTITIONS), "
            f"{_lib.FFTCONVOLVE_MAX_PARTITIONS * block} samples")
    if math.prod(lo) == 0:
        return x.new_empty(lo + (out_len,))
    return _convolve_rows(_FFTConvolveFunction, x, y, lx, ly, lo, start, out_len)


def convolve(x: Tensor, y: Tensor, mode: str = "full") -> Tensor:
    """Convolves ``x (..., N)`` and ``y (..., M)`` along their last dimension using the direct method (reference
    functional.py:2261-2314): the true convolution, leading dimensions broadcast, output ``(..., L)`` with
    L = N + M - 1 (``"full"``), max(N, M) - min(N, M) + 1 (``"valid"``) or N (``"same"``).  Runs a banded Toeplitz
    product on TF32 x 3 tensor-core MMAs at float32 grade (``csrc/convolve_direct.cu``), and only the outputs the mode
    returns are computed.  The shorter operand (the filter) may have up to 4096 taps; longer filters are the job of
    ``fftconvolve``."""
    n, m, lx, ly, lo = _convolve_operands(x, y, mode)
    if lx != ly:  # the reference broadcasts to the per-dimension maximum, which refuses a 0 against a 1
        big, small = (y, x) if n < m else (x, y)
        new = [max(i, j) for i, j in zip(big.shape[:-1], small.shape[:-1])]
        big.broadcast_to(new + [big.shape[-1]])
        small.broadcast_to(new + [small.shape[-1]])
    if math.prod(lo) == 0:  # the reference's grouped conv1d with zero groups
        raise RuntimeError("non-positive groups is not supported")
    if n == 0 or m == 0:  # and with padding min(N, M) - 1 < 0
        raise RuntimeError("negative padding is not supported")
    k = min(n, m)
    if k > _lib.CONVOLVE_MAX_TAPS:
        raise RuntimeError(
            f"audio_b200: convolve of a {k}-sample shorter operand is not supported: the direct method is capped at "
            f"{_lib.CONVOLVE_MAX_TAPS} taps (B200A_CONVOLVE_MAX_TAPS); use fftconvolve for longer filters")
    start, out_len = _convolve_slice(n, m, mode)
    return _convolve_rows(_ConvolveFunction, x, y, lx, ly, lo, start, out_len)


def _rnnt_check_device(t: Tensor, name: str, logits: Tensor) -> None:
    if not isinstance(t, Tensor):
        raise TypeError(f"{name} must be a torch.Tensor")
    if not t.is_cuda or t.device != logits.device:
        raise RuntimeError(f"logits and {name} must be on the same device")


def _rnnt_inputs(logits: Tensor, targets: Tensor, logit_lengths: Tensor, target_lengths: Tensor, blank: int):
    """The reference's checks (rnnt/gpu/compute.cu:25-85) in its order and with its messages, then the ones where the
    reference reads out of bounds.  The lengths are checked on the device by one launch and read back once."""
    if not isinstance(logits, Tensor):
        raise TypeError("logits must be a torch.Tensor")
    if not logits.is_cuda:
        raise RuntimeError(
            f"audio_b200: logits is on '{logits.device}'. This package runs only hand-written sm_90a CUDA "
            "kernels; there is no CPU or ATen fallback -- move the tensor (and the module) to a CUDA device."
        )
    _rnnt_check_device(targets, "targets", logits)
    _rnnt_check_device(logit_lengths, "logit_lengths", logits)
    _rnnt_check_device(target_lengths, "target_lengths", logits)
    if logits.dtype not in (torch.float32, torch.float16):
        raise RuntimeError("logits must be float32 or float16 (half) type")
    if targets.dtype != torch.int32:
        raise RuntimeError("targets must be int32 type")
    if logit_lengths.dtype != torch.int32:
        raise RuntimeError("logit_lengths must be int32 type")
    if target_lengths.dtype != torch.int32:
        raise RuntimeError("target_lengths must be int32 type")
    for t, name in ((logits, "logits"), (targets, "targets"), (logit_lengths, "logit_lengths"),
                    (target_lengths, "target_lengths")):
        if not t.is_contiguous():
            raise RuntimeError(f"{name} must be contiguous")
    if logits.dim() != 4:
        raise RuntimeError("logits must be 4-D (batch, time, target, class)")
    if targets.dim() != 2:
        raise RuntimeError("targets must be 2-D (batch, max target length)")
    if logit_lengths.dim() != 1:
        raise RuntimeError("logit_lengths must be 1-D")
    if target_lengths.dim() != 1:
        raise RuntimeError("target_lengths must be 1-D")
    batch, max_t, max_u, classes = logits.shape
    if logit_lengths.size(0) != batch:
        raise RuntimeError("batch dimension mismatch between logits and logit_lengths")
    if target_lengths.size(0) != batch:
        raise RuntimeError("batch dimension mismatch between logits and target_lengths")
    if targets.size(0) != batch:
        raise RuntimeError("batch dimension mismatch between logits and targets")
    if not 0 <= blank < classes:
        raise RuntimeError("blank must be within [0, logits.shape[-1])")
    dev = logits.device
    with torch.cuda.device(dev):
        stats = torch.empty(5, dtype=torch.int32, device=dev)
        rc = _lib.lib().b200a_rnnt_loss_check(batch, classes, targets.data_ptr(), targets.size(1),
                                              logit_lengths.data_ptr(), target_lengths.data_ptr(), stats.data_ptr(),
                                              _stream_ptr(dev))
    _lib.check(rc, "rnnt_loss check")
    t_max, t_min, u_max, u_min, bad_target = stats.tolist()
    if max_t != t_max:
        raise RuntimeError("input length mismatch")
    if max_u != u_max + 1:
        raise RuntimeError("output length mismatch")
    if targets.size(1) + 1 != max_u:
        raise RuntimeError("target length mismatch")
    if t_min < 1:
        raise ValueError(f"rnnt_loss: every logit_lengths entry must be at least 1 (got {t_min})")
    if u_min < 0:
        raise ValueError(f"rnnt_loss: target_lengths entries must be non-negative (got {u_min})")
    if bad_target:
        raise ValueError(f"rnnt_loss: a target within its sequence's target_length lies outside [0, {classes})")
    if max_u > _lib.RNNT_MAX_U:
        raise ValueError(f"rnnt_loss: logits.shape[2] = {max_u} is above the supported {_lib.RNNT_MAX_U}")


def _rnnt_desc(logits: Tensor, blank: int, clamp: float, fused: bool):
    batch, max_t, max_u, classes = logits.shape
    return _lib.RnntLossDesc(batch, max_t, max_u, classes, blank,
                             _lib.DTYPE_F16 if logits.dtype == torch.float16 else _lib.DTYPE_F32, int(bool(fused)),
                             float(clamp))


def _rnnt_forward(logits, targets, logit_lengths, target_lengths, desc, save: bool):
    """b200a_rnnt_loss_forward: the costs, and the float32 (denom, alpha, beta) of the gradient when ``save``."""
    dev = logits.device
    batch, max_t, max_u, _ = logits.shape
    with torch.cuda.device(dev):
        costs = torch.empty(batch, dtype=logits.dtype, device=dev)
        ws = torch.empty(_lib.lib().b200a_rnnt_loss_workspace_bytes(desc), dtype=torch.uint8, device=dev)
        saved = [torch.empty((batch, max_t, max_u), dtype=torch.float32, device=dev) if save and (k or desc.fused)
                 else None for k in range(3)]
        denom, alpha, beta = saved
        rc = _lib.lib().b200a_rnnt_loss_forward(
            desc, logits.data_ptr(), targets.data_ptr(), logit_lengths.data_ptr(), target_lengths.data_ptr(),
            costs.data_ptr(), 0 if denom is None else denom.data_ptr(), 0 if alpha is None else alpha.data_ptr(),
            0 if beta is None else beta.data_ptr(), ws.data_ptr(), ws.numel(), _stream_ptr(dev))
    _lib.check(rc, "rnnt_loss")
    return costs, denom, alpha, beta


class _RnntLossFunction(torch.autograd.Function):
    """_rnnt_forward with the logit gradient.  Saved: the inputs through save_for_backward (so an in-place edit of the
    logits before backward is an error) and per-(b, t, u) float32 denom / alpha / beta; nothing joint-sized."""

    @staticmethod
    def forward(ctx, logits, targets, logit_lengths, target_lengths, desc):
        costs, denom, alpha, beta = _rnnt_forward(logits, targets, logit_lengths, target_lengths, desc, True)
        ctx.desc = desc
        ctx.fused = denom is not None
        ctx.save_for_backward(logits, targets, logit_lengths, target_lengths, alpha, beta,
                              *((denom,) if denom is not None else ()))
        return costs

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        logits, targets, logit_lengths, target_lengths, alpha, beta, *rest = ctx.saved_tensors
        denom = rest[0] if ctx.fused else None
        dev = logits.device
        if dy.dim() != 1 or dy.dtype != logits.dtype:
            dy = dy.reshape(-1).to(logits.dtype)
        with torch.cuda.device(dev):
            grad = torch.empty_like(logits)
            rc = _lib.lib().b200a_rnnt_loss_backward(
                ctx.desc, logits.data_ptr(), targets.data_ptr(), logit_lengths.data_ptr(), target_lengths.data_ptr(),
                0 if denom is None else denom.data_ptr(), alpha.data_ptr(), beta.data_ptr(), dy.data_ptr(),
                dy.stride(0), grad.data_ptr(), _stream_ptr(dev))
        _lib.check(rc, "rnnt_loss backward")
        return grad, None, None, None, None


def rnnt_loss(
    logits: Tensor,
    targets: Tensor,
    logit_lengths: Tensor,
    target_lengths: Tensor,
    blank: int = -1,
    clamp: float = -1,
    reduction: str = "mean",
    fused_log_softmax: bool = True,
):
    """The RNN Transducer loss of Graves (2012) (reference functional.py:1747-1796): logits ``(batch, max seq length,
    max target length + 1, class)`` in float32 or float16, int32 targets ``(batch, max target length)`` and lengths
    ``(batch,)``, all contiguous on one CUDA device.  Returns the costs (``reduction="none"``, shape ``(batch,)``) or
    their mean or sum, in the logits' dtype; the arithmetic is float32.

    Differentiable with respect to ``logits`` whenever grad mode is on and ``logits.requires_grad``, with no
    ``audio_b200.differentiable`` switch: a loss exists to be differentiated.  Otherwise nothing is saved and no gradient
    kernel runs.  ``clamp > 0`` clamps each unscaled gradient element to ``[-clamp, clamp]`` (as the reference's CPU
    path) before the upstream gradient scales it.  A sequence whose paths all have probability 0 costs NaN (or inf when
    T or U + 1 is 1) and gets a zero gradient.  Beyond the reference's checks, raises ``ValueError`` for a
    ``logit_lengths`` entry below 1, a negative ``target_lengths`` entry and a target outside ``[0, class)`` within its
    sequence's length, where the reference reads out of bounds.
    """
    if reduction not in ["none", "mean", "sum"]:
        raise ValueError('reduction should be one of "none", "mean", or "sum"')
    if blank < 0:  # reinterpret blank index if blank < 0.
        blank = logits.shape[-1] + blank
    _rnnt_inputs(logits, targets, logit_lengths, target_lengths, blank)
    desc = _rnnt_desc(logits, blank, clamp, fused_log_softmax)
    if torch.is_grad_enabled() and logits.requires_grad:
        costs = _RnntLossFunction.apply(logits, targets, logit_lengths, target_lengths, desc)
    else:
        costs = _rnnt_forward(logits, targets, logit_lengths, target_lengths, desc, False)[0]
    if reduction == "mean":
        return costs.mean()
    elif reduction == "sum":
        return costs.sum()
    return costs


_FA_DTYPES = {torch.float32: _lib.DTYPE_F32, torch.float16: _lib.DTYPE_F16, torch.float64: _lib.DTYPE_F64}
_INDEX_DTYPES = {torch.int32: _lib.INDEX_I32, torch.int64: _lib.INDEX_I64}


def _fa_tensor(t, name: str, log_probs: Tensor) -> None:
    if not isinstance(t, Tensor):
        raise TypeError(f"{name} must be a torch.Tensor")
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor")
    if t.device != log_probs.device:
        raise RuntimeError(f"log_probs and {name} need to be on the same device")


def forced_align(
    log_probs: Tensor,
    targets: Tensor,
    input_lengths: Optional[Tensor] = None,
    target_lengths: Optional[Tensor] = None,
    blank: int = 0,
) -> Tuple[Tensor, Tensor]:
    """Align CTC label sequences to emissions (reference functional/_alignment.py): the Viterbi path of
    ``targets`` ``(B, L)`` (int32 or int64) through ``log_probs`` ``(B, T, C)`` (float32, float16 or float64), both
    contiguous on one CUDA device, with optional ``(B,)`` int32 / int64 lengths of any strides (the full sizes when
    ``None``).

    Returns ``(paths, scores)``, both ``(B, T)``: the label of every frame in the targets' dtype and its log-probability
    in the log-probs' dtype.  Row ``b`` is exactly the reference CPU's alignment of ``log_probs[b:b+1, :T_b]`` and
    ``targets[b:b+1, :L_b]`` (same path, same scores, same tie-breaking); frames ``t >= T_b`` hold ``blank`` and 0, and a
    row with ``L_b = 0`` is all blank.  The reference takes ``B == 1`` only.  The outputs do not require grad.

    Raises as the reference does, with its messages; the blank and range checks cover each sequence's first ``L_b``
    targets.  Beyond them, raises ``ValueError`` for a negative target, an ``input_lengths`` entry below 1, a negative
    ``target_lengths`` entry, and ``L`` above ``B200A_FORCED_ALIGN_MAX_L`` (8191).  One launch checks the inputs and
    its result is read back once; the alignment itself is one more launch.
    """
    if not isinstance(log_probs, Tensor):
        raise TypeError("log_probs must be a torch.Tensor")
    if not log_probs.is_cuda:
        raise RuntimeError(
            f"audio_b200: log_probs is on '{log_probs.device}'. This package runs only hand-written sm_90a CUDA "
            "kernels; there is no CPU or ATen fallback -- move the tensor (and the module) to a CUDA device."
        )
    _fa_tensor(targets, "targets", log_probs)
    dev = log_probs.device
    for t, name in ((input_lengths, "input_lengths"), (target_lengths, "target_lengths")):
        if t is not None:
            _fa_tensor(t, name, log_probs)
    if log_probs.dtype not in _FA_DTYPES:
        raise RuntimeError("log_probs must be float64, float32 or float16 (half) type")
    if targets.dtype not in _INDEX_DTYPES:
        raise RuntimeError("targets must be int32 or int64 type")
    for t, name in ((input_lengths, "input_lengths"), (target_lengths, "target_lengths")):
        if t is not None and t.dtype not in _INDEX_DTYPES:
            raise RuntimeError(f"{name} must be int32 or int64 type")
    if not log_probs.is_contiguous():
        raise RuntimeError("log_probs must be contiguous")
    if not targets.is_contiguous():
        raise RuntimeError("targets must be contiguous")
    if log_probs.dim() != 3:
        raise RuntimeError("log_probs must be 3-D (batch_size, input length, num classes)")
    if targets.dim() != 2:
        raise RuntimeError("targets must be 2-D (batch_size, target length,)")
    if input_lengths is None:
        input_lengths = torch.full((log_probs.size(0),), log_probs.size(1), dtype=torch.int64, device=dev)
    if target_lengths is None:
        target_lengths = torch.full((targets.size(0),), targets.size(1), dtype=torch.int64, device=dev)
    if input_lengths.dim() != 1:
        raise RuntimeError("input_lengths must be 1-D (batch_size,)")
    if target_lengths.dim() != 1:
        raise RuntimeError("target_lengths must be 1-D (batch_size,)")
    batch, max_t, classes = log_probs.shape
    if targets.size(0) != batch or input_lengths.size(0) != batch or target_lengths.size(0) != batch:
        raise RuntimeError("log_probs, targets, input_lengths and target_lengths must have the same batch size")
    if targets.numel() == 0:  # the reference's torch.max(targets)
        raise RuntimeError("max(): Expected reduction dim to be specified for input.numel() == 0. "
                           "Specify the reduction dim with the 'dim' argument.")
    if batch == 0 or max_t == 0:
        raise ValueError("forced_align: log_probs must have at least one sequence and one frame")
    # The kernels read both lengths as dense (B,) vectors of one dtype.  Like the reference (which takes their max()),
    # any 1-D strides are accepted: a strided or expanded vector is copied, B elements.
    len_dtype = input_lengths.dtype if input_lengths.dtype == target_lengths.dtype else torch.int64
    input_lengths = input_lengths.to(len_dtype).contiguous()
    target_lengths = target_lengths.to(len_dtype).contiguous()
    max_l = targets.size(1)
    # a blank outside int32 reaches the check as -1, whose blank flag then means nothing and is ignored below
    blank_fits = -(2**31) <= blank < 2**31
    blank32 = blank if blank_fits else -1
    desc = _lib.ForcedAlignDesc(batch, max_t, min(max_l, 2**31 - 1), classes, blank32, _FA_DTYPES[log_probs.dtype],
                                _INDEX_DTYPES[targets.dtype], _INDEX_DTYPES[input_lengths.dtype])
    lib = _lib.lib()
    with torch.cuda.device(dev):
        ws = torch.empty(max(lib.b200a_forced_align_workspace_bytes(desc), 4 * batch), dtype=torch.uint8, device=dev)
        stats = torch.empty(11, dtype=torch.int64, device=dev)
        rc = lib.b200a_forced_align_check(desc, targets.data_ptr(), input_lengths.data_ptr(),
                                          target_lengths.data_ptr(), stats.data_ptr(), ws.data_ptr(), ws.numel(),
                                          _stream_ptr(dev))
        _lib.check(rc, "forced_align check")
        t_max, t_min, l_max, l_min, out_of_range, negative, has_blank, bad, bad_t, bad_l, bad_r = stats.tolist()
    if has_blank and blank_fits:
        raise ValueError(f"targets Tensor shouldn't contain blank index. Found {targets}.")
    if out_of_range:
        raise ValueError("targets values must be less than the CTC dimension")
    if not 0 <= blank < classes:
        raise RuntimeError("blank must be within [0, num classes)")
    if negative:
        raise ValueError("forced_align: a target within its sequence's target_length is negative")
    if max_t != t_max:
        raise RuntimeError("input length mismatch")
    if max_l != l_max:
        raise RuntimeError("target length mismatch")
    if t_min < 1:
        raise ValueError(f"forced_align: every input_lengths entry must be at least 1 (got {t_min})")
    if l_min < 0:
        raise ValueError(f"forced_align: target_lengths entries must be non-negative (got {l_min})")
    if bad >= 0:
        raise RuntimeError(f"targets length is too long for CTC. Found log_probs length: {bad_t}, targets length: "
                           f"{bad_l}, and number of repeats: {bad_r}")
    if max_l > _lib.FORCED_ALIGN_MAX_L:
        raise ValueError(f"forced_align: targets.shape[1] = {max_l} is above the supported {_lib.FORCED_ALIGN_MAX_L}")
    with torch.cuda.device(dev):
        paths = torch.empty((batch, max_t), dtype=targets.dtype, device=dev)
        scores = torch.empty((batch, max_t), dtype=log_probs.dtype, device=dev)
        rc = lib.b200a_forced_align_run(desc, log_probs.data_ptr(), targets.data_ptr(), input_lengths.data_ptr(),
                                        target_lengths.data_ptr(), paths.data_ptr(), scores.data_ptr(), ws.data_ptr(),
                                        ws.numel(), _stream_ptr(dev))
    _lib.check(rc, "forced_align")
    return paths, scores


@dataclass
class TokenSpan:
    """One token of an alignment with its frame span and score, as :func:`merge_tokens` returns it."""

    token: int
    """The token."""
    start: int
    """The first frame of the span (inclusive)."""
    end: int
    """The frame after the span (exclusive)."""
    score: float
    """The mean of the frame scores over the span."""

    def __len__(self) -> int:
        """The span's length in frames."""
        return self.end - self.start


def merge_tokens(tokens: Tensor, scores: Tensor, blank: int = 0) -> List[TokenSpan]:
    """Collapse an unbatched alignment (a row of :func:`forced_align`'s ``paths`` and ``scores``, shape ``(T,)``) into
    spans of repeated non-blank tokens, each scored by the mean of its frames' scores (reference
    functional/_alignment.py).  Both tensors are copied to the host once; every span is built there."""
    if tokens.ndim != 1 or scores.ndim != 1:
        raise ValueError("`tokens` and `scores` must be 1D Tensor.")
    if len(tokens) != len(scores):
        raise ValueError("`tokens` and `scores` must be the same length.")
    scores = scores.detach().cpu()
    ids = tokens.tolist()
    spans = []
    start = 0
    for t in range(1, len(ids) + 1):
        if t == len(ids) or ids[t] != ids[start]:
            if ids[start] != blank:
                spans.append(TokenSpan(token=ids[start], start=start, end=t, score=scores[start:t].mean().item()))
            start = t
    return spans
