"""Drop-in ``torchaudio.transforms`` modules of the hot path, backed by libb200audio.so.

Class names, constructor signatures, attribute / buffer / sub-module names and error
behaviour follow pytorch/audio/src/torchaudio/transforms/_transforms.py
(Spectrogram 25-123, AmplitudeToDB 300-346, MelScale 349-415, InverseMelScale 418-503,
MelSpectrogram 506-622, MFCC 625-709, Resample 899-980), so ``state_dict``s interchange with torchaudio's and
existing call sites keep working after ``import audio_b200.transforms as T``.

``forward`` launches hand-written sm_90a kernels through the C ABI; MelSpectrogram and MFCC
do NOT chain their sub-modules' forwards (that would round-trip the (B, T, n_fft/2+1) power
spectrum through HBM) -- they read the sub-modules' buffers and launch the fused kernel.

Gradients are opt-in, per thread: Spectrogram and MelSpectrogram inside ``audio_b200.differentiable()``,
InverseSpectrogram with ``inverse=True``, Resample / Speed / SpeedPerturbation with ``resample=True``, and MFCC,
LFCC, AmplitudeToDB, MelScale, InverseMelScale and SpectralCentroid with ``features=True``, the Kaldi features
(``audio_b200.compliance.kaldi``) with ``kaldi=True``, TimeStretch (spectrogram gradient) and PitchShift
(waveform gradient) with ``vocoder=True``, and Preemphasis and Deemphasis (waveform gradient) and Convolve and
FFTConvolve (input gradients) with ``filtering=True``.
GriffinLim is forward-only.  RNNTLoss is differentiable with respect to the logits without a switch, and FrequencyMasking,
TimeMasking and SpecAugment with respect to the input and a tensor mask value.
"""
from __future__ import annotations

import math
import warnings
from typing import Callable, Optional, Union

import torch
from torch import Tensor

from . import _filtering, _lib, _masking, _ops
from . import functional as F
from ._plans import (FrontendPlan, InverseMelPlan, ResamplePlan, _InverseMelFunction, _no_autograd, _require_cuda_f32,
                     _wants_grad, is_feature_differentiable, vocoder_chain)

__all__ = ["Spectrogram", "InverseSpectrogram", "GriffinLim", "AmplitudeToDB", "MelScale", "InverseMelScale", "MelSpectrogram", "MFCC", "LFCC",
           "SpectralCentroid", "Resample", "Speed", "SpeedPerturbation", "TimeStretch", "PitchShift", "Preemphasis",
           "Deemphasis", "FFTConvolve", "Convolve", "Vad", "RNNTLoss", "FrequencyMasking", "TimeMasking",
           "SpecAugment"]


def _setup_framing(mod, n_fft, win_length, hop_length, window_fn=None, wkwargs=None, hop_div=2):
    """The STFT geometry every transform here derives the same way (reference _transforms.py:79-87 and siblings):
    win_length defaults to n_fft, hop_length to win_length // hop_div, and the window buffer is window_fn(win_length)."""
    mod.n_fft = n_fft
    mod.win_length = n_fft if win_length is None else win_length
    mod.hop_length = mod.win_length // hop_div if hop_length is None else hop_length
    if window_fn is not None:
        mod.register_buffer("window", window_fn(mod.win_length, **(wkwargs or {})))


class Spectrogram(torch.nn.Module):
    r"""Create a spectrogram from an audio signal: ``(..., time) -> (..., n_fft // 2 + 1, n_frames)``.

    Args are those of ``torchaudio.transforms.Spectrogram`` (reference _transforms.py:64-78).
    """

    __constants__ = ["n_fft", "win_length", "hop_length", "pad", "power", "normalized"]

    def __init__(
        self,
        n_fft: int = 400,
        win_length: Optional[int] = None,
        hop_length: Optional[int] = None,
        pad: int = 0,
        window_fn: Callable[..., Tensor] = torch.hann_window,
        power: Optional[float] = 2.0,
        normalized: Union[bool, str] = False,
        wkwargs: Optional[dict] = None,
        center: bool = True,
        pad_mode: str = "reflect",
        onesided: bool = True,
        return_complex: Optional[bool] = None,
    ) -> None:
        super().__init__()
        _setup_framing(self, n_fft, win_length, hop_length, window_fn, wkwargs)
        self.pad = pad
        self.power = power
        self.normalized = normalized
        self.center = center
        self.pad_mode = pad_mode
        self.onesided = onesided
        if return_complex is not None:
            warnings.warn(
                "`return_complex` argument is now deprecated and is not effective."
                "`torchaudio.transforms.Spectrogram(power=None)` always returns a tensor with "
                "complex dtype. Please remove the argument in the function call."
            )
        self._plan: Optional[FrontendPlan] = None

    def _frontend_plan(self, n_mels: int = 0, n_mfcc: int = 0, log_mels: bool = False) -> FrontendPlan:
        fl_norm, win_norm = F._get_spec_norms(self.normalized)
        desc = FrontendPlan.make_desc(
            self.n_fft, self.win_length, self.hop_length, self.pad, self.center, self.pad_mode,
            self.onesided, fl_norm, win_norm, self.power, n_mels, n_mfcc, log_mels,
        )
        return FrontendPlan(desc)

    def forward(self, waveform: Tensor) -> Tensor:
        plan = self._frontend_plan()
        if self._plan is None or self._plan.desc.key() != plan.desc.key():
            self._plan = plan
        ws = self._plan.workspace(self.window, None, None)
        stage = _lib.STAGE_COMPLEX if self.power is None else _lib.STAGE_POWER
        return F._unpack(self._plan.run(ws, stage, waveform, constants=(("window", self.window),)), waveform)


class InverseSpectrogram(torch.nn.Module):
    r"""Recover an audio signal from a complex spectrogram: ``(..., n_fft // 2 + 1, frames) -> (..., time)``.

    Args are those of ``torchaudio.transforms.InverseSpectrogram`` (reference _transforms.py:126-212); buffer ``window``.
    """

    __constants__ = ["n_fft", "win_length", "hop_length", "pad", "power", "normalized"]

    def __init__(
        self,
        n_fft: int = 400,
        win_length: Optional[int] = None,
        hop_length: Optional[int] = None,
        pad: int = 0,
        window_fn: Callable[..., Tensor] = torch.hann_window,
        normalized: Union[bool, str] = False,
        wkwargs: Optional[dict] = None,
        center: bool = True,
        pad_mode: str = "reflect",
        onesided: bool = True,
    ) -> None:
        super().__init__()
        _setup_framing(self, n_fft, win_length, hop_length, window_fn, wkwargs)
        self.pad = pad
        self.normalized = normalized
        self.center = center
        self.pad_mode = pad_mode
        self.onesided = onesided

    def forward(self, spectrogram: Tensor, length: Optional[int] = None) -> Tensor:
        return F.inverse_spectrogram(
            spectrogram, length, self.pad, self.window, self.n_fft, self.hop_length, self.win_length, self.normalized,
            self.center, self.pad_mode, self.onesided,
        )


class GriffinLim(torch.nn.Module):
    r"""Compute a waveform from a linear-scale magnitude spectrogram with the fast Griffin-Lim transformation
    (reference _transforms.py:215-297): ``(..., n_fft // 2 + 1, frames) -> (..., time)``; buffer ``window``."""

    __constants__ = ["n_fft", "n_iter", "win_length", "hop_length", "power", "length", "momentum", "rand_init"]

    def __init__(
        self,
        n_fft: int = 400,
        n_iter: int = 32,
        win_length: Optional[int] = None,
        hop_length: Optional[int] = None,
        window_fn: Callable[..., Tensor] = torch.hann_window,
        power: float = 2.0,
        wkwargs: Optional[dict] = None,
        momentum: float = 0.99,
        length: Optional[int] = None,
        rand_init: bool = True,
    ) -> None:
        super().__init__()
        if not (0 <= momentum < 1):
            raise ValueError("momentum must be in the range [0, 1). Found: {}".format(momentum))
        self.n_fft = n_fft
        self.n_iter = n_iter
        self.win_length = win_length if win_length is not None else n_fft
        self.hop_length = hop_length if hop_length is not None else self.win_length // 2
        window = window_fn(self.win_length) if wkwargs is None else window_fn(self.win_length, **wkwargs)
        self.register_buffer("window", window)
        self.length = length
        self.power = power
        self.momentum = momentum
        self.rand_init = rand_init

    def forward(self, specgram: Tensor) -> Tensor:
        return F.griffinlim(
            specgram, self.window, self.n_fft, self.hop_length, self.win_length, self.power, self.n_iter, self.momentum,
            self.length, self.rand_init,
        )


class AmplitudeToDB(torch.nn.Module):
    r"""Power/amplitude -> decibel scale (reference _transforms.py:300-346)."""

    __constants__ = ["multiplier", "amin", "ref_value", "db_multiplier"]

    def __init__(self, stype: str = "power", top_db: Optional[float] = None) -> None:
        super().__init__()
        self.stype = stype
        if top_db is not None and top_db < 0:
            raise ValueError("top_db must be positive value")
        self.top_db = top_db
        self.multiplier = 10.0 if stype == "power" else 20.0
        self.amin = 1e-10
        self.ref_value = 1.0
        self.db_multiplier = math.log10(max(self.amin, self.ref_value))

    def forward(self, x: Tensor) -> Tensor:
        return F.amplitude_to_DB(x, self.multiplier, self.amin, self.db_multiplier, self.top_db)


class MelScale(torch.nn.Module):
    r"""STFT bins -> mel bins with triangular filters (reference _transforms.py:349-415)."""

    __constants__ = ["n_mels", "sample_rate", "f_min", "f_max"]

    def __init__(
        self,
        n_mels: int = 128,
        sample_rate: int = 16000,
        f_min: float = 0.0,
        f_max: Optional[float] = None,
        n_stft: int = 201,
        norm: Optional[str] = None,
        mel_scale: str = "htk",
    ) -> None:
        super().__init__()
        self.n_mels = n_mels
        self.sample_rate = sample_rate
        self.f_max = f_max if f_max is not None else float(sample_rate // 2)
        self.f_min = f_min
        self.norm = norm
        self.mel_scale = mel_scale
        if f_min > self.f_max:
            raise ValueError("Require f_min: {} <= f_max: {}".format(f_min, self.f_max))
        fb = F.melscale_fbanks(n_stft, self.f_min, self.f_max, self.n_mels, self.sample_rate, self.norm, self.mel_scale)
        self.register_buffer("fb", fb)

    def forward(self, specgram: Tensor) -> Tensor:
        return F._apply_fbank(specgram, self.fb)


class InverseMelScale(torch.nn.Module):
    r"""Estimate a linear-frequency spectrogram from a mel spectrogram (reference _transforms.py:418-503):
    ``(..., n_mels, time) -> (..., n_stft, time)``; buffer ``fb``.

    The reference returns ``relu(lstsq(fb^T, melspec, driver).solution)``.  For ``n_mels <= n_stft`` and a nonsingular
    Gram matrix ``G = fb^T fb`` every driver gives the minimum-norm solution ``relu(fb G^-1 m)``; ``G`` of a mel bank is
    banded (tridiagonal), so each frame is one banded solve (factored once per ``fb`` version, in double precision on
    the host) and a <= 2-tap expansion, in one kernel.  The output is a transposed view of a frame-major tensor, the
    strides the reference returns.  A singular ``G`` raises ``torch.linalg.LinAlgError`` with ``driver="gels"``, as the
    reference does, and a "not supported" error with the rank-revealing drivers; so do ``n_mels > n_stft`` banks except
    where gels fails.  Inside ``audio_b200.differentiable(features=True)`` the mel spectrogram gets its gradient.
    """

    __constants__ = ["n_stft", "n_mels", "sample_rate", "f_min", "f_max"]

    def __init__(
        self,
        n_stft: int,
        n_mels: int = 128,
        sample_rate: int = 16000,
        f_min: float = 0.0,
        f_max: Optional[float] = None,
        norm: Optional[str] = None,
        mel_scale: str = "htk",
        driver: str = "gels",
    ) -> None:
        super().__init__()
        self.n_mels = n_mels
        self.sample_rate = sample_rate
        self.f_max = f_max or float(sample_rate // 2)
        self.f_min = f_min
        self.driver = driver
        if f_min > self.f_max:
            raise ValueError("Require f_min: {} <= f_max: {}".format(f_min, self.f_max))
        if driver not in ["gels", "gelsy", "gelsd", "gelss"]:
            raise ValueError(f'driver must be one of ["gels", "gelsy", "gelsd", "gelss"]. Found {driver}.')
        fb = F.melscale_fbanks(n_stft, self.f_min, self.f_max, self.n_mels, self.sample_rate, norm, mel_scale)
        self.register_buffer("fb", fb)
        self._plan = InverseMelPlan(driver)

    def forward(self, melspec: Tensor) -> Tensor:
        shape = melspec.size()
        n_mels, time = shape[-2], shape[-1]
        if self.n_mels != n_mels:
            raise ValueError("Expected an input with {} mel bins. Found: {}".format(self.n_mels, n_mels))
        _require_cuda_f32(melspec, "melspec")
        _require_cuda_f32(self.fb, "fb")
        grad = _wants_grad(melspec, (("fb", self.fb),), is_feature_differentiable, "mel spectrogram")
        if not grad:
            _no_autograd(melspec)
        n_stft = self.fb.shape[0]
        plan = self._plan.plan(self.fb)
        m3 = melspec.reshape(-1, n_mels, time)
        out = _InverseMelFunction.apply(m3, plan, n_stft) if grad else _ops.inverse_mel(m3, plan, n_stft)
        return out.reshape(shape[:-2] + (time, n_stft)).transpose(-1, -2)


class MelSpectrogram(torch.nn.Module):
    r"""MelSpectrogram for a raw audio signal, as ONE fused kernel.

    Composes ``self.spectrogram`` and ``self.mel_scale`` exactly like the reference
    (_transforms.py:557-610) so buffers are named ``spectrogram.window`` / ``mel_scale.fb``.
    """

    __constants__ = ["sample_rate", "n_fft", "win_length", "hop_length", "pad", "n_mels", "f_min"]

    def __init__(
        self,
        sample_rate: int = 16000,
        n_fft: int = 400,
        win_length: Optional[int] = None,
        hop_length: Optional[int] = None,
        f_min: float = 0.0,
        f_max: Optional[float] = None,
        pad: int = 0,
        n_mels: int = 128,
        window_fn: Callable[..., Tensor] = torch.hann_window,
        power: float = 2.0,
        normalized: bool = False,
        wkwargs: Optional[dict] = None,
        center: bool = True,
        pad_mode: str = "reflect",
        onesided: Optional[bool] = None,
        norm: Optional[str] = None,
        mel_scale: str = "htk",
    ) -> None:
        super().__init__()
        if onesided is not None:
            warnings.warn(
                "Argument 'onesided' has been deprecated and has no influence on the behavior of this module."
            )
        self.sample_rate = sample_rate
        _setup_framing(self, n_fft, win_length, hop_length)
        self.pad = pad
        self.power = power
        self.normalized = normalized
        self.n_mels = n_mels
        self.f_max = f_max
        self.f_min = f_min
        self.spectrogram = Spectrogram(
            n_fft=self.n_fft,
            win_length=self.win_length,
            hop_length=self.hop_length,
            pad=self.pad,
            window_fn=window_fn,
            power=self.power,
            normalized=self.normalized,
            wkwargs=wkwargs,
            center=center,
            pad_mode=pad_mode,
            onesided=True,
        )
        self.mel_scale = MelScale(
            self.n_mels, self.sample_rate, self.f_min, self.f_max, self.n_fft // 2 + 1, norm, mel_scale
        )
        self._plan: Optional[FrontendPlan] = None

    def _fused_plan(self, n_mfcc: int = 0, log_mels: bool = False, db=None) -> FrontendPlan:
        if self.spectrogram.power is None:
            raise RuntimeError("MelSpectrogram needs a real power spectrogram (power must not be None)")
        plan = self.spectrogram._frontend_plan(self.mel_scale.fb.shape[1], n_mfcc, log_mels)
        if db is not None:
            plan.desc.db_multiplier, plan.desc.db_amin, plan.desc.db_offset = db
        if self._plan is None or self._plan.desc.key() != plan.desc.key():
            self._plan = plan
        return self._plan

    def forward(self, waveform: Tensor) -> Tensor:
        plan = self._fused_plan()
        return F.mel_spectrogram(plan, self.spectrogram.window, self.mel_scale.fb, waveform)


class MFCC(torch.nn.Module):
    r"""Mel-frequency cepstrum coefficients (reference _transforms.py:625-709).

    ``process_group``: optional ``torch.distributed`` group.  When the batch of a 2-D
    ``(batch, time)`` input is sharded across ranks, the reference's batch-global ``top_db``
    clamp needs the maximum over ALL shards; setting the group makes ``forward`` all-reduce that
    one scalar (MAX) between the two kernels.
    """

    __constants__ = ["sample_rate", "n_mfcc", "dct_type", "top_db", "log_mels"]

    def __init__(
        self,
        sample_rate: int = 16000,
        n_mfcc: int = 40,
        dct_type: int = 2,
        norm: str = "ortho",
        log_mels: bool = False,
        melkwargs: Optional[dict] = None,
    ) -> None:
        super().__init__()
        supported_dct_types = [2]
        if dct_type not in supported_dct_types:
            raise ValueError("DCT type not supported: {}".format(dct_type))
        self.sample_rate = sample_rate
        self.n_mfcc = n_mfcc
        self.dct_type = dct_type
        self.norm = norm
        self.top_db = 80.0
        self.amplitude_to_DB = AmplitudeToDB("power", self.top_db)
        melkwargs = melkwargs or {}
        self.MelSpectrogram = MelSpectrogram(sample_rate=self.sample_rate, **melkwargs)
        if self.n_mfcc > self.MelSpectrogram.n_mels:
            raise ValueError("Cannot select more MFCC coefficients than # mel bins")
        dct_mat = F.create_dct(self.n_mfcc, self.MelSpectrogram.n_mels, self.norm)
        self.register_buffer("dct_mat", dct_mat)
        self.log_mels = log_mels
        self.process_group = None

    def forward(self, waveform: Tensor) -> Tensor:
        mel = self.MelSpectrogram
        db = self.amplitude_to_DB
        plan = mel._fused_plan(
            self.dct_mat.shape[1], self.log_mels,
            (float(db.multiplier), float(db.amin), float(db.multiplier * db.db_multiplier)),
        )
        return F.mfcc(
            plan, mel.spectrogram.window, mel.mel_scale.fb, self.dct_mat, waveform,
            db.top_db, self.log_mels, self.process_group,
        )


class LFCC(torch.nn.Module):
    r"""Linear-frequency cepstral coefficients (reference _transforms.py:712-819): the MFCC pipeline with
    ``F.linear_fbanks`` instead of the mel bank -- same fused kernels, buffers ``filter_mat`` / ``dct_mat``."""

    __constants__ = ["sample_rate", "n_filter", "n_lfcc", "dct_type", "top_db", "log_lf"]

    def __init__(
        self,
        sample_rate: int = 16000,
        n_filter: int = 128,
        f_min: float = 0.0,
        f_max: Optional[float] = None,
        n_lfcc: int = 40,
        dct_type: int = 2,
        norm: str = "ortho",
        log_lf: bool = False,
        speckwargs: Optional[dict] = None,
    ) -> None:
        super().__init__()
        supported_dct_types = [2]
        if dct_type not in supported_dct_types:
            raise ValueError("DCT type not supported: {}".format(dct_type))
        self.sample_rate = sample_rate
        self.f_min = f_min
        self.f_max = f_max if f_max is not None else float(sample_rate // 2)
        self.n_filter = n_filter
        self.n_lfcc = n_lfcc
        self.dct_type = dct_type
        self.norm = norm
        self.top_db = 80.0
        self.amplitude_to_DB = AmplitudeToDB("power", self.top_db)
        speckwargs = speckwargs or {}
        self.Spectrogram = Spectrogram(**speckwargs)
        if self.n_lfcc > self.Spectrogram.n_fft:
            raise ValueError("Cannot select more LFCC coefficients than # fft bins")
        filter_mat = F.linear_fbanks(
            n_freqs=self.Spectrogram.n_fft // 2 + 1,
            f_min=self.f_min,
            f_max=self.f_max,
            n_filter=self.n_filter,
            sample_rate=self.sample_rate,
        )
        self.register_buffer("filter_mat", filter_mat)
        dct_mat = F.create_dct(self.n_lfcc, self.n_filter, self.norm)
        self.register_buffer("dct_mat", dct_mat)
        self.log_lf = log_lf
        self.process_group = None
        self._plan: Optional[FrontendPlan] = None

    def forward(self, waveform: Tensor) -> Tensor:
        spec = self.Spectrogram
        if spec.power is None or not spec.onesided:
            raise RuntimeError("LFCC needs a one-sided real (power) spectrogram")
        db = self.amplitude_to_DB
        plan = spec._frontend_plan(self.filter_mat.shape[1], self.dct_mat.shape[1], self.log_lf)
        plan.desc.db_multiplier, plan.desc.db_amin = float(db.multiplier), float(db.amin)
        plan.desc.db_offset = float(db.multiplier * db.db_multiplier)
        if self._plan is None or self._plan.desc.key() != plan.desc.key():
            self._plan = plan
        return F.mfcc(
            self._plan, spec.window, self.filter_mat, self.dct_mat, waveform, db.top_db, self.log_lf, self.process_group,
            fb_name="filter_mat",
        )


class SpectralCentroid(torch.nn.Module):
    r"""Spectral centroid per frame (reference _transforms.py:1612-1671)."""

    __constants__ = ["sample_rate", "n_fft", "win_length", "hop_length", "pad"]

    def __init__(
        self,
        sample_rate: int,
        n_fft: int = 400,
        win_length: Optional[int] = None,
        hop_length: Optional[int] = None,
        pad: int = 0,
        window_fn: Callable[..., Tensor] = torch.hann_window,
        wkwargs: Optional[dict] = None,
    ) -> None:
        super().__init__()
        self.sample_rate = sample_rate
        _setup_framing(self, n_fft, win_length, hop_length, window_fn, wkwargs)
        self.pad = pad

    def forward(self, waveform: Tensor) -> Tensor:
        return F.spectral_centroid(
            waveform, self.sample_rate, self.pad, self.window, self.n_fft, self.hop_length, self.win_length
        )


class Resample(torch.nn.Module):
    r"""Resample a signal from one frequency to another (reference _transforms.py:899-980)."""

    def __init__(
        self,
        orig_freq: int = 16000,
        new_freq: int = 16000,
        resampling_method: str = "sinc_interp_hann",
        lowpass_filter_width: int = 6,
        rolloff: float = 0.99,
        beta: Optional[float] = None,
        *,
        dtype: Optional[torch.dtype] = None,
    ) -> None:
        super().__init__()
        self.orig_freq = orig_freq
        self.new_freq = new_freq
        self.gcd = math.gcd(int(self.orig_freq), int(self.new_freq))
        self.resampling_method = resampling_method
        self.lowpass_filter_width = lowpass_filter_width
        self.rolloff = rolloff
        self.beta = beta
        self._plan: Optional[ResamplePlan] = None
        if self.orig_freq != self.new_freq:
            kernel, self.width = F._get_sinc_resample_kernel(
                self.orig_freq,
                self.new_freq,
                self.gcd,
                self.lowpass_filter_width,
                self.rolloff,
                self.resampling_method,
                beta,
                dtype=dtype,
            )
            self.register_buffer("kernel", kernel)

    def forward(self, waveform: Tensor) -> Tensor:
        if self.orig_freq == self.new_freq:
            return waveform
        if self._plan is None:
            self._plan = ResamplePlan(int(self.orig_freq) // self.gcd, int(self.new_freq) // self.gcd, self.width)
        return F._apply_sinc_resample_kernel(
            waveform, self.orig_freq, self.new_freq, self.gcd, self.kernel, self.width, self._plan
        )


def _source_target_sample_rate(orig_freq: int, speed: float):
    """Reduced integer rates whose ratio is the speed factor (reference _transforms.py:1951-1955)."""
    source, target = int(speed * orig_freq), int(orig_freq)
    g = math.gcd(source, target)
    return source // g, target // g


class Speed(torch.nn.Module):
    r"""Adjusts waveform speed by resampling (reference _transforms.py:1958-2001): the waveform is treated as if
    sampled at ``factor * orig_freq`` and brought back to ``orig_freq`` by the polyphase tensor-pipe resampler.

    ``forward(waveform, lengths=None) -> (waveform', lengths')`` with ``lengths' = ceil(lengths * target / source)``.
    """

    def __init__(self, orig_freq, factor) -> None:
        super().__init__()
        self.orig_freq = orig_freq
        self.factor = factor
        self.source_sample_rate, self.target_sample_rate = _source_target_sample_rate(orig_freq, factor)
        self.resampler = Resample(orig_freq=self.source_sample_rate, new_freq=self.target_sample_rate)

    def forward(self, waveform: Tensor, lengths: Optional[Tensor] = None):
        if lengths is None:
            out_lengths = None
        else:  # a handful of integers: bookkeeping, not signal processing
            out_lengths = torch.ceil(lengths * self.target_sample_rate / self.source_sample_rate).to(lengths.dtype)
        return self.resampler(waveform), out_lengths


class SpeedPerturbation(torch.nn.Module):
    r"""Speed perturbation augmentation (reference _transforms.py:2004-2055): each call draws one of ``factors``
    uniformly (``torch.randint``, so ``torch.manual_seed`` reproduces the reference's choices) and applies ``Speed``."""

    def __init__(self, orig_freq: int, factors) -> None:
        super().__init__()
        self.speeders = torch.nn.ModuleList([Speed(orig_freq=orig_freq, factor=factor) for factor in factors])

    def forward(self, waveform: Tensor, lengths: Optional[Tensor] = None):
        idx = int(torch.randint(len(self.speeders), ()))
        return self.speeders[idx](waveform, lengths)


class TimeStretch(torch.nn.Module):
    r"""Stretch a complex spectrogram in time without modifying pitch (reference _transforms.py:1001-1083):
    ``(..., freq, num_frame) -> (..., freq, ceil(num_frame / rate))``; buffer ``phase_advance``."""

    __constants__ = ["fixed_rate"]

    def __init__(self, hop_length: Optional[int] = None, n_freq: int = 201, fixed_rate: Optional[float] = None) -> None:
        super().__init__()
        self.fixed_rate = fixed_rate
        n_fft = (n_freq - 1) * 2
        hop_length = hop_length if hop_length is not None else n_fft // 2
        self.register_buffer("phase_advance", torch.linspace(0, math.pi * hop_length, n_freq)[..., None])

    def forward(self, complex_specgrams: Tensor, overriding_rate: Optional[float] = None) -> Tensor:
        if not torch.is_complex(complex_specgrams):
            warnings.warn(
                "The input to TimeStretch must be complex type. "
                "Providing non-complex tensor produces invalid results.",
                stacklevel=4,
            )
        if overriding_rate is None:
            if self.fixed_rate is None:
                raise ValueError("If no fixed_rate is specified, must pass a valid rate to the forward method.")
            rate = self.fixed_rate
        else:
            rate = overriding_rate
        return F.phase_vocoder(complex_specgrams, rate, self.phase_advance)


class PitchShift(torch.nn.Module):
    r"""Shift the pitch of a waveform by ``n_steps`` steps (reference _transforms.py:1674-1780): STFT -> phase vocoder ->
    inverse STFT -> resample -> crop / pad to the input length.  Buffer ``window``; the resampling taps are built on the
    first call in the input's dtype on its device, like the reference's lazily materialised ``kernel``."""

    __constants__ = ["sample_rate", "n_steps", "bins_per_octave", "n_fft", "win_length", "hop_length"]

    def __init__(
        self,
        sample_rate: int,
        n_steps: int,
        bins_per_octave: int = 12,
        n_fft: int = 512,
        win_length: Optional[int] = None,
        hop_length: Optional[int] = None,
        window_fn: Callable[..., Tensor] = torch.hann_window,
        wkwargs: Optional[dict] = None,
    ) -> None:
        super().__init__()
        self.n_steps = n_steps
        self.bins_per_octave = bins_per_octave
        self.sample_rate = sample_rate
        _setup_framing(self, n_fft, win_length, hop_length, window_fn, wkwargs, hop_div=4)
        rate = 2.0 ** (-float(n_steps) / bins_per_octave)
        self.orig_freq = int(sample_rate / rate)
        self.gcd = math.gcd(int(self.orig_freq), int(sample_rate))
        self.width = -1
        self.kernel = None
        self._plan = None

    # The reference keeps ``kernel`` as a lazily materialised parameter, so its state_dict carries a "kernel" entry
    # once the module has run (_transforms.py:1731-1757).  Mirror that: emit the taps when they exist, accept them on load.
    def _save_to_state_dict(self, destination, prefix, keep_vars):
        super()._save_to_state_dict(destination, prefix, keep_vars)
        if self.kernel is not None:
            destination[prefix + "kernel"] = self.kernel if keep_vars else self.kernel.detach()

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        k = state_dict.pop(prefix + "kernel", None)
        if isinstance(k, Tensor) and k.numel() > 0:
            orig_r = self.orig_freq // self.gcd
            taps = k.shape[-1]
            if k.dim() == 3 and k.shape[0] == self.sample_rate // self.gcd and taps > orig_r and (taps - orig_r) % 2 == 0:
                self.kernel, self.width, self._plan = k.detach().clone(), (taps - orig_r) // 2, None
            else:
                error_msgs.append(f"size mismatch for {prefix}kernel: {tuple(k.shape)} does not fit this PitchShift")
        super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs)

    def forward(self, waveform: Tensor) -> Tensor:
        with vocoder_chain(waveform):
            return self._shift(waveform)

    def _shift(self, waveform: Tensor) -> Tensor:
        shape = waveform.size()
        flat = waveform.reshape(-1, shape[-1])
        ori_len = shape[-1]
        rate = 2.0 ** (-float(self.n_steps) / self.bins_per_octave)
        spec_f = F.spectrogram(flat, 0, self.window, self.n_fft, self.hop_length, self.win_length, None, False)
        phase_advance = torch.linspace(0, math.pi * self.hop_length, spec_f.shape[-2], device=spec_f.device)[..., None]
        spec_stretch = F.phase_vocoder(spec_f, rate, phase_advance)
        stretched = F.inverse_spectrogram(spec_stretch, int(round(ori_len / rate)), 0, self.window, self.n_fft,
                                          self.hop_length, self.win_length, False)
        if self.orig_freq != self.sample_rate:
            if self.kernel is None:
                self.kernel, self.width = F._get_sinc_resample_kernel(
                    self.orig_freq, self.sample_rate, self.gcd, dtype=waveform.dtype, device=waveform.device)
                self._plan = None
            elif self.kernel.device != waveform.device or self.kernel.dtype != waveform.dtype:  # loaded / moved
                self.kernel, self._plan = self.kernel.to(device=waveform.device, dtype=waveform.dtype), None
            if self._plan is None:
                self._plan = ResamplePlan(self.orig_freq // self.gcd, self.sample_rate // self.gcd, self.width)
            shifted = F._apply_sinc_resample_kernel(stretched, self.orig_freq, self.sample_rate, self.gcd, self.kernel,
                                                    self.width, self._plan)
        else:
            shifted = stretched
        shift_len = shifted.size()[-1]
        if shift_len > ori_len:
            shifted = shifted[..., :ori_len]
        else:
            shifted = torch.nn.functional.pad(shifted, [0, ori_len - shift_len])
        return shifted.reshape(shape[:-1] + shifted.shape[-1:])


class Preemphasis(torch.nn.Module):
    """y[i] = x[i] - coeff * x[i - 1] along the last dimension (reference _transforms.py:2086-2112)."""

    def __init__(self, coeff: float = 0.97) -> None:
        super().__init__()
        self.coeff = coeff

    def forward(self, waveform: Tensor) -> Tensor:
        return F.preemphasis(waveform, coeff=self.coeff)


class Deemphasis(torch.nn.Module):
    """y[i] = x[i] + coeff * y[i - 1], clamped to [-1, 1] as the reference's is (reference _transforms.py:2115-2140)."""

    def __init__(self, coeff: float = 0.97) -> None:
        super().__init__()
        self.coeff = coeff

    def forward(self, waveform: Tensor) -> Tensor:
        return F.deemphasis(waveform, coeff=self.coeff)


class FFTConvolve(torch.nn.Module):
    """Convolves inputs along their last dimension (reference _transforms.py:1906-1948): ``F.fftconvolve(x, y, mode)``,
    uniformly partitioned overlap-save on the GPU."""

    def __init__(self, mode: str = "full") -> None:
        F._check_convolve_mode(mode)
        super().__init__()
        self.mode = mode

    def forward(self, x: Tensor, y: Tensor) -> Tensor:
        return F.fftconvolve(x, y, mode=self.mode)


class Convolve(torch.nn.Module):
    """Convolves inputs along their last dimension using the direct method (reference _transforms.py:1863-1903):
    ``F.convolve(x, y, mode)``, a banded TF32 x 3 tensor-core product on the GPU, for filters up to 4096 taps."""

    def __init__(self, mode: str = "full") -> None:
        F._check_convolve_mode(mode)
        super().__init__()
        self.mode = mode

    def forward(self, x: Tensor, y: Tensor) -> Tensor:
        return F.convolve(x, y, mode=self.mode)


class Vad(torch.nn.Module):
    """Voice-activity trim from the front of the audio, as SoX's vad (reference _transforms.py:1478-1612):
    ``F.vad(waveform, sample_rate, ...)`` with the module's parameters.  The host constants, windows and front-end
    workspaces are built at the first ``forward`` and kept."""

    def __init__(self, sample_rate: int, trigger_level: float = 7.0, trigger_time: float = 0.25,
                 search_time: float = 1.0, allowed_gap: float = 0.25, pre_trigger_time: float = 0.0,
                 boot_time: float = 0.35, noise_up_time: float = 0.1, noise_down_time: float = 0.01,
                 noise_reduction_amount: float = 1.35, measure_freq: float = 20.0,
                 measure_duration: Optional[float] = None, measure_smooth_time: float = 0.4,
                 hp_filter_freq: float = 50.0, lp_filter_freq: float = 6000.0, hp_lifter_freq: float = 150.0,
                 lp_lifter_freq: float = 2000.0) -> None:
        super().__init__()
        self.sample_rate = sample_rate
        self.trigger_level = trigger_level
        self.trigger_time = trigger_time
        self.search_time = search_time
        self.allowed_gap = allowed_gap
        self.pre_trigger_time = pre_trigger_time
        self.boot_time = boot_time
        self.noise_up_time = noise_up_time
        self.noise_down_time = noise_down_time
        self.noise_reduction_amount = noise_reduction_amount
        self.measure_freq = measure_freq
        self.measure_duration = measure_duration
        self.measure_smooth_time = measure_smooth_time
        self.hp_filter_freq = hp_filter_freq
        self.lp_filter_freq = lp_filter_freq
        self.hp_lifter_freq = hp_lifter_freq
        self.lp_lifter_freq = lp_lifter_freq
        self._plan = None

    def _params(self):
        return (self.sample_rate, self.trigger_level, self.trigger_time, self.search_time, self.allowed_gap,
                self.pre_trigger_time, self.boot_time, self.noise_up_time, self.noise_down_time,
                self.noise_reduction_amount, self.measure_freq, self.measure_duration, self.measure_smooth_time,
                self.hp_filter_freq, self.lp_filter_freq, self.hp_lifter_freq, self.lp_lifter_freq)

    def forward(self, waveform: Tensor) -> Tensor:
        _filtering._warn_batch(waveform)
        params = self._params()
        if self._plan is None or self._plan[0] != params:  # rebuilt only when an attribute was changed
            self._plan = (params, _filtering.VadPlan(*params))
        return _filtering._vad_trim(waveform, self._plan[1])


class RNNTLoss(torch.nn.Module):
    """The RNN Transducer loss (reference _transforms.py:1783-1850): ``forward(logits, targets, logit_lengths,
    target_lengths)`` is :func:`audio_b200.functional.rnnt_loss` with this module's ``blank``, ``clamp``, ``reduction``
    and ``fused_log_softmax``."""

    def __init__(self, blank: int = -1, clamp: float = -1.0, reduction: str = "mean", fused_log_softmax: bool = True):
        super().__init__()
        self.blank = blank
        self.clamp = clamp
        self.reduction = reduction
        self.fused_log_softmax = fused_log_softmax

    def forward(self, logits: Tensor, targets: Tensor, logit_lengths: Tensor, target_lengths: Tensor):
        return F.rnnt_loss(logits, targets, logit_lengths, target_lengths, self.blank, self.clamp, self.reduction,
                           self.fused_log_softmax)


class _AxisMasking(torch.nn.Module):
    """Masking along one axis (reference _transforms.py:1167-1206); ``axis`` counts as if the input were 3-D (1: freq,
    2: time).  With ``iid_masks`` each example gets its own mask (:func:`audio_b200.functional.mask_along_axis_iid`),
    otherwise one mask for all (:func:`audio_b200.functional.mask_along_axis`, a tensor ``mask_value`` read as a
    float)."""

    __constants__ = ["mask_param", "axis", "iid_masks", "p"]

    def __init__(self, mask_param: int, axis: int, iid_masks: bool, p: float = 1.0) -> None:
        super().__init__()
        self.mask_param = mask_param
        self.axis = axis
        self.iid_masks = iid_masks
        self.p = p

    def forward(self, specgram: Tensor, mask_value: Union[float, torch.Tensor] = 0.0) -> Tensor:
        axis = self.axis + specgram.dim() - 3
        if self.iid_masks:
            return F.mask_along_axis_iid(specgram, self.mask_param, mask_value, axis, p=self.p)
        mask_value_ = float(mask_value) if isinstance(mask_value, Tensor) else mask_value
        return F.mask_along_axis(specgram, self.mask_param, mask_value_, axis, p=self.p)


class FrequencyMasking(_AxisMasking):
    """SpecAugment frequency masking (reference _transforms.py:1209-1240)."""

    def __init__(self, freq_mask_param: int, iid_masks: bool = False) -> None:
        super().__init__(freq_mask_param, 1, iid_masks)


class TimeMasking(_AxisMasking):
    """SpecAugment time masking (reference _transforms.py:1243-1278)."""

    def __init__(self, time_mask_param: int, iid_masks: bool = False, p: float = 1.0) -> None:
        if not 0.0 <= p <= 1.0:
            raise ValueError(f"The value of p must be between 0.0 and 1.0 ({p} given).")
        super().__init__(time_mask_param, 2, iid_masks, p=p)


class SpecAugment(torch.nn.Module):
    """Time and frequency masking (reference _transforms.py:1281-1349): the reference's ``mean()`` fill (or 0 with
    ``zero_masking``) and its draws in its order -- every time mask, then every frequency mask, per example when the
    input has more than 2 dimensions and ``iid_masks`` -- then one launch for all of them.  Exact: every mask shares
    the fill fixed before the first, so their union is the reference's sequential result."""

    __constants__ = ["n_time_masks", "time_mask_param", "n_freq_masks", "freq_mask_param", "iid_masks", "p",
                     "zero_masking"]

    def __init__(self, n_time_masks: int, time_mask_param: int, n_freq_masks: int, freq_mask_param: int,
                 iid_masks: bool = True, p: float = 1.0, zero_masking: bool = False) -> None:
        super().__init__()
        self.n_time_masks = n_time_masks
        self.time_mask_param = time_mask_param
        self.n_freq_masks = n_freq_masks
        self.freq_mask_param = freq_mask_param
        self.iid_masks = iid_masks
        self.p = p
        self.zero_masking = zero_masking

    def forward(self, specgram: Tensor) -> Tensor:
        return _masking.spec_augment(specgram, self.n_time_masks, self.time_mask_param, self.n_freq_masks,
                                     self.freq_mask_param, self.iid_masks, self.p, self.zero_masking)


# ---- B200A_REFERENCE=1: A/B switch to the reference implementation (debugging only, never silent) -----------------
# SURVEY.md 8(b): "an explicit env override to run the reference for A/B".  With the variable set when this module is
# imported, every transform above keeps its constructor, attributes and buffers but `forward` runs the importable
# `torchaudio.transforms` class of the same name with the same constructor arguments and THIS module's buffers (on
# whatever device the input lives, CPU included).  A warning is issued at import; nothing is switched implicitly.
def _install_reference_switch() -> None:
    import os

    if os.environ.get("B200A_REFERENCE", "0") != "1":
        return
    try:
        import torchaudio.transforms as ref_T
    except Exception as exc:  # noqa: BLE001
        raise ImportError("B200A_REFERENCE=1 needs an importable torchaudio to route the transforms to") from exc
    warnings.warn(
        "B200A_REFERENCE=1: audio_b200.transforms modules run torchaudio's reference implementation "
        f"(torchaudio {getattr(__import__('torchaudio'), '__version__', '?')}); the CUDA kernels are bypassed",
        stacklevel=2,
    )

    def patch(cls, ref_cls):
        orig_init = cls.__init__

        def __init__(self, *args, **kwargs):
            orig_init(self, *args, **kwargs)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                self.__dict__["_reference_module"] = ref_cls(*args, **kwargs)  # not a registered sub-module

        def forward(self, *args, **kwargs):
            ref = self.__dict__["_reference_module"]
            dev = next((a.device for a in args if isinstance(a, Tensor)), None)
            if dev is not None:
                ref.to(dev)
            own = {k: v.to(dev) if dev is not None else v for k, v in self.state_dict().items()}
            ref.load_state_dict(own, strict=False)  # the buffers the user sees / edits are the ones used
            return ref(*args, **kwargs)

        cls.__init__ = __init__
        cls.forward = forward

    for name in __all__:
        if hasattr(ref_T, name):
            patch(globals()[name], getattr(ref_T, name))


_install_reference_switch()
