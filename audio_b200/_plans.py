"""Device-side plans: a descriptor + the caller-owned workspace libb200audio fills once.

PyTorch is used here only for what the C ABI deliberately leaves to the caller: device
memory (``torch.empty``), the current stream, and the device guard.
"""
from __future__ import annotations

import contextlib
import math
import threading
from typing import Optional, Tuple

import torch
from torch.autograd.function import once_differentiable

from . import _lib, _ops
from ._bookkeeping import resample_len


def _require_cuda_f32(t: torch.Tensor, what: str) -> None:
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{what} must be a torch.Tensor")
    if not t.is_cuda:
        raise RuntimeError(
            f"audio_b200: {what} is on '{t.device}'. This package runs only hand-written sm_90a CUDA "
            "kernels; there is no CPU or ATen fallback -- move the tensor (and the module) to a CUDA device."
        )
    if t.dtype != torch.float32:
        raise TypeError(f"audio_b200: {what} must be float32 (got {t.dtype}); other dtypes are not implemented")


_GRAD_STATE = threading.local()


def is_differentiable() -> bool:
    """Whether Spectrogram, MelSpectrogram and F.spectrogram accept inputs that require grad (in this thread)."""
    return getattr(_GRAD_STATE, "on", False)


def is_inverse_differentiable() -> bool:
    """Whether InverseSpectrogram and F.inverse_spectrogram accept spectrograms that require grad (in this thread)."""
    return getattr(_GRAD_STATE, "inverse", False)


def is_resample_differentiable() -> bool:
    """Whether Resample, F.resample, Speed and SpeedPerturbation accept waveforms that require grad (in this thread)."""
    return getattr(_GRAD_STATE, "resample", False)


def is_feature_differentiable() -> bool:
    """Whether MFCC, LFCC, AmplitudeToDB, MelScale, InverseMelScale, SpectralCentroid and pipelines.RNNTFeatureExtractor
    accept inputs that require grad (in this thread)."""
    return getattr(_GRAD_STATE, "features", False)


def is_kaldi_differentiable() -> bool:
    """Whether compliance.kaldi spectrogram, fbank and mfcc (and their ``_batch`` forms) accept waveforms that require
    grad (in this thread)."""
    return getattr(_GRAD_STATE, "kaldi", False)


def is_vocoder_differentiable() -> bool:
    """Whether F.phase_vocoder and TimeStretch accept spectrograms, and F.pitch_shift and PitchShift waveforms, that
    require grad (in this thread)."""
    return getattr(_GRAD_STATE, "vocoder", False)


def is_filtering_differentiable() -> bool:
    """Whether F.lfilter, F.filtfilt, the ``*_biquad`` filters, F.deemphasis, F.preemphasis, Preemphasis and
    Deemphasis accept waveforms and coefficients, and F.convolve, Convolve, F.fftconvolve and FFTConvolve operands, that
    require grad (in this thread)."""
    return getattr(_GRAD_STATE, "filtering", False)


def set_differentiable(mode: bool, *, inverse: bool = False, resample: bool = False, features: bool = False,
                       kaldi: bool = False, vocoder: bool = False, filtering: bool = False) -> None:
    """Turn waveform gradients on or off for the calling thread (off by default, like a fresh thread's grad mode).
    ``inverse=True`` (with ``mode``) also turns on the spectrogram gradients of the inverse STFT, ``resample=True``
    (with ``mode``) the waveform gradients of the resampler, ``features=True`` (with ``mode``) the input gradients of
    MFCC, LFCC, AmplitudeToDB, MelScale, InverseMelScale, SpectralCentroid and the RNN-T feature extractor,
    ``kaldi=True`` (with ``mode``) the waveform gradients of the Kaldi spectrogram, fbank and mfcc, ``vocoder=True`` (with ``mode``) the spectrogram gradients of the phase
    vocoder and TimeStretch and the waveform gradients of PitchShift, ``filtering=True`` (with ``mode``) the waveform
    and coefficient gradients of lfilter, filtfilt, the biquads and pre-/de-emphasis and the input gradients of
    F.convolve, Convolve, F.fftconvolve and FFTConvolve (convolution is FIR filtering).  They are separate switches so
    that vocoder inference, augmentation code (Speed, SpeedPerturbation, TimeStretch, PitchShift) and Kaldi feature preprocessing in
    data pipelines do not build graphs when loss gradients are on, and so that the top_db clamp's gradient -- every
    clamped element's share goes to the group maximum -- is opted into knowingly."""
    _GRAD_STATE.on = bool(mode)
    _GRAD_STATE.inverse = bool(mode) and bool(inverse)
    _GRAD_STATE.resample = bool(mode) and bool(resample)
    _GRAD_STATE.features = bool(mode) and bool(features)
    _GRAD_STATE.kaldi = bool(mode) and bool(kaldi)
    _GRAD_STATE.vocoder = bool(mode) and bool(vocoder)
    _GRAD_STATE.filtering = bool(mode) and bool(filtering)


def _switches():
    return (is_differentiable(), is_inverse_differentiable(), is_resample_differentiable(), is_feature_differentiable(),
            is_kaldi_differentiable(), is_vocoder_differentiable(), is_filtering_differentiable())


def _restore(prev) -> None:
    set_differentiable(prev[0], inverse=prev[1], resample=prev[2], features=prev[3], kaldi=prev[4], vocoder=prev[5],
                       filtering=prev[6])


@contextlib.contextmanager
def differentiable(mode: bool = True, *, inverse: bool = False, resample: bool = False, features: bool = False,
                   kaldi: bool = False, vocoder: bool = False, filtering: bool = False):
    """Context manager form of :func:`set_differentiable`; restores the previous settings on exit."""
    prev = _switches()
    set_differentiable(mode, inverse=inverse, resample=resample, features=features, kaldi=kaldi, vocoder=vocoder,
                       filtering=filtering)
    try:
        yield
    finally:
        _restore(prev)


@contextlib.contextmanager
def vocoder_chain(waveform: torch.Tensor):
    """PitchShift's stages (STFT, phase vocoder, inverse STFT, resampler) for one call: with ``vocoder=True`` on and a
    waveform that requires grad, the front-end, inverse and resampler gradients are on too for the duration of the call,
    and the caller's switches are restored on exit.  Otherwise the switches stay as they are."""
    if not (is_vocoder_differentiable() and torch.is_grad_enabled() and waveform.requires_grad):
        yield
        return
    prev = _switches()
    set_differentiable(True, inverse=True, resample=True, features=prev[3], kaldi=prev[4], vocoder=True,
                       filtering=prev[6])
    try:
        yield
    finally:
        _restore(prev)


def _no_autograd(t: torch.Tensor) -> None:
    if t.requires_grad and torch.is_grad_enabled():
        raise RuntimeError(
            "audio_b200 kernels are forward-only: the input requires grad. Call under torch.no_grad() / "
            "torch.inference_mode(), or detach() the input. (Spectrogram, MelSpectrogram and F.spectrogram compute "
            "waveform gradients inside audio_b200.differentiable(); InverseSpectrogram and F.inverse_spectrogram "
            "compute spectrogram gradients inside audio_b200.differentiable(inverse=True); Resample, F.resample, Speed "
            "and SpeedPerturbation compute waveform gradients inside audio_b200.differentiable(resample=True); MFCC, LFCC, "
            "AmplitudeToDB, MelScale, InverseMelScale, SpectralCentroid and pipelines.RNNTFeatureExtractor compute input "
            "gradients inside audio_b200.differentiable(features=True); compliance.kaldi spectrogram, fbank and mfcc compute waveform "
            "gradients inside audio_b200.differentiable(kaldi=True); F.phase_vocoder and TimeStretch compute spectrogram "
            "gradients, F.pitch_shift and PitchShift waveform gradients, inside audio_b200.differentiable(vocoder=True); F.lfilter, "
            "F.filtfilt, the *_biquad filters, F.preemphasis, F.deemphasis, Preemphasis and Deemphasis compute waveform and "
            "coefficient gradients, and F.convolve, Convolve, F.fftconvolve and FFTConvolve the gradients of both operands, "
            "inside "
            "audio_b200.differentiable(filtering=True).)"
        )


def _wants_grad(waveform: torch.Tensor, constants, switch=is_differentiable, input_name: str = "waveform") -> bool:
    """True when the output must carry a gradient of the input ``waveform`` and ``switch()`` is on; raises for
    constant buffers that require grad, whose gradients are not computed."""
    if not (switch() and torch.is_grad_enabled()):
        return False
    for name, t in constants:
        if t is not None and t.requires_grad:
            raise RuntimeError(
                f"audio_b200: {name} requires grad, but only the {input_name} gradient is implemented; detach() it "
                "or register it as a buffer"
            )
    return waveform.requires_grad


class _FrontendFunction(torch.autograd.Function):
    """b200audio::frontend_run on the packed (rows, L) waveform, with b200audio::frontend_backward as its backward.
    The workspace of the forward is kept, so a window or filterbank changed before backward does not change the
    gradient; the waveform goes through save_for_backward, so in-place edits of it are detected."""

    @staticmethod
    def forward(ctx, flat, ws, desc_i, desc_f, stage, frames, width, stride):
        out = _ops.frontend_run(flat, ws, desc_i, desc_f, stage, frames, width, stride, None, 1)
        ctx.save_for_backward(flat)
        ctx.ws, ctx.desc_i, ctx.desc_f, ctx.stage, ctx.stride = ws, desc_i, desc_f, stage, stride
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        (flat,) = ctx.saved_tensors
        grad = _ops.frontend_backward(flat, ctx.ws, ctx.desc_i, ctx.desc_f, ctx.stage, ctx.stride, grad_out)
        return grad, None, None, None, None, None, None, None


class _MfccFunction(torch.autograd.Function):
    """MFCC / LFCC from the packed (rows, L) waveform: the same STAGE_FEAT + mfcc_finish launches as the no-grad path, so
    the cepstra are bit-identical to it.  Saved: the waveform (save_for_backward), the pre-clamp features, the group
    maxima and the forward's workspace -- a window, filterbank or DCT edited before backward does not change the
    gradient.  Backward: the mel stage recomputed, the feature adjoint (b200audio::mfcc_backward), the mel-stage
    waveform gradient (b200audio::frontend_backward)."""

    @staticmethod
    def forward(ctx, flat, ws, desc_i, desc_f, frames, stride, groups, rows_per_group, top_db):
        n_mels = desc_i[_ops.field_index(_lib.FrontendDesc, "n_mels")]
        gmax = new_group_max(groups, flat.device) if groups > 0 else None
        feat = _ops.frontend_run(flat, ws, desc_i, desc_f, _lib.STAGE_FEAT, frames, n_mels, stride, gmax, rows_per_group)
        out = _ops.mfcc_finish(feat, ws, desc_i, desc_f, gmax, rows_per_group, top_db)
        ctx.save_for_backward(flat)
        ctx.feat, ctx.gmax, ctx.ws = feat, gmax, ws
        ctx.args = desc_i, desc_f, frames, stride, rows_per_group, top_db
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        (flat,) = ctx.saved_tensors
        desc_i, desc_f, frames, stride, rows_per_group, top_db = ctx.args
        n_mels = desc_i[_ops.field_index(_lib.FrontendDesc, "n_mels")]
        mel = _ops.frontend_run(flat, ctx.ws, desc_i, desc_f, _lib.STAGE_MEL, frames, n_mels, stride, None, 1)
        g_mel = _ops.mfcc_backward(grad_out, ctx.feat, mel, ctx.gmax, ctx.ws, desc_i, desc_f, rows_per_group, top_db)
        grad = _ops.frontend_backward(flat, ctx.ws, desc_i, desc_f, _lib.STAGE_MEL, stride, g_mel)
        return grad, None, None, None, None, None, None, None, None


class _RNNTFunction(torch.autograd.Function):
    """The RNN-T features of the packed (rows, L) waveform: the same b200audio::rnnt_features launch as the no-grad path
    plus the mel values before the chain, so the features are bit-identical to it.  Saved: the waveform and the
    statistics buffers ``mean`` / ``invstddev`` (save_for_backward: an in-place edit of either raises in backward), the
    mel values, the packed statistics the forward read and its workspace.  Backward: the chain's VJP
    (b200audio::rnnt_features_backward) on the first ``frames`` rows, then the mel-stage waveform gradient
    (b200audio::frontend_backward)."""

    @staticmethod
    def forward(ctx, flat, ws, desc_i, desc_f, stats, mean, invstd, gain, frames, pad_frames, stride):
        out, mel = _ops.rnnt_features(flat, ws, desc_i, desc_f, None, stats, gain, frames, pad_frames, stride, True)
        ctx.save_for_backward(flat, mean, invstd)
        ctx.mel, ctx.stats, ctx.ws = mel, stats, ws
        ctx.args = desc_i, desc_f, gain, frames, stride
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        flat, _, _ = ctx.saved_tensors
        desc_i, desc_f, gain, frames, stride = ctx.args
        g_mel = _ops.rnnt_features_backward(ctx.stats, gain, ctx.mel, grad_out[:, :frames])
        grad = _ops.frontend_backward(flat, ctx.ws, desc_i, desc_f, _lib.STAGE_MEL, stride, g_mel)
        return grad, None, None, None, None, None, None, None, None, None, None


class StampCache:
    """A value built from constant tensors, rebuilt when any of them changes.  A tensor's stamp is its (data_ptr,
    in-place edit counter, device); inference tensors (created under torch.inference_mode) keep no edit counter.  The
    tensors behind the stamp are held, so their storage cannot be recycled and an equal stamp can only mean the same,
    unmodified tensors."""

    def __init__(self):
        self.value = None
        self._stamp = None
        self._held = None

    def get(self, tensors: tuple, build):
        """The cached value while the stamp of ``tensors`` (``None`` entries allowed) is unchanged, else
        ``build(*tensors)``."""
        stamp = tuple(None if t is None else (t.data_ptr(), -1 if t.is_inference() else t._version, str(t.device))
                      for t in tensors)
        if stamp != self._stamp:
            self.value = build(*tensors)
            self._stamp, self._held = stamp, tensors
        return self.value


def _stream_ptr(device: torch.device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def pack_rows(waveform: torch.Tensor) -> Tuple[torch.Tensor, int]:
    """(..., time) -> (rows, time) view with unit inner stride; returns it and the row stride."""
    length = waveform.shape[-1]
    flat = waveform.reshape(-1, length)
    if flat.shape[0] > 0 and length > 0 and (flat.stride(1) != 1 or (flat.shape[0] > 1 and flat.stride(0) < length)):
        flat = flat.contiguous()
    stride = flat.stride(0) if flat.shape[0] > 1 else max(length, 1)
    return flat, stride


class FrontendPlan:
    """Workspace for one (descriptor, window, fb, dct) combination on one device."""

    def __init__(self, desc: "_lib.FrontendDesc"):
        self.desc = desc
        self._ws = StampCache()  # keyed on the (window, fb, dct) the workspace is built from
        self._desc_lists = None  # the descriptor as (ints, floats) for the torch.library ops

    @staticmethod
    def make_desc(
        n_fft: int,
        win_length: int,
        hop: int,
        pad: int,
        center: bool,
        pad_mode: str,
        onesided: bool,
        frame_length_norm: bool,
        window_norm: bool,
        power: Optional[float],
        n_mels: int = 0,
        n_mfcc: int = 0,
        log_mels: bool = False,
    ) -> "_lib.FrontendDesc":
        if pad_mode not in _lib.PAD_MODE:
            raise ValueError(f"Unsupported pad_mode: {pad_mode!r} (expected one of {sorted(_lib.PAD_MODE)})")
        d = _lib.FrontendDesc()
        d.n_fft, d.win_length, d.hop, d.pad = int(n_fft), int(win_length), int(hop), int(pad)
        d.center, d.pad_mode, d.onesided = int(bool(center)), _lib.PAD_MODE[pad_mode], int(bool(onesided))
        d.frame_length_norm, d.window_norm = int(bool(frame_length_norm)), int(bool(window_norm))
        d.power = float("nan") if power is None else float(power)
        d.n_mels, d.n_mfcc, d.log_mels = int(n_mels), int(n_mfcc), int(bool(log_mels))
        d.db_multiplier, d.db_amin = 10.0, 1e-10
        d.db_offset = 10.0 * math.log10(max(1e-10, 1.0))
        return d

    def workspace(self, window: torch.Tensor, fb: Optional[torch.Tensor], dct: Optional[torch.Tensor]) -> torch.Tensor:
        """Return a prepared workspace, rebuilding it if any constant buffer changed."""
        return self._ws.get((window, fb, dct), self._prepare)

    def _prepare(self, window: torch.Tensor, fb: Optional[torch.Tensor], dct: Optional[torch.Tensor]) -> torch.Tensor:
        lib = _lib.lib()
        _require_cuda_f32(window, "window")
        dev = window.device
        for name, t in (("fb", fb), ("dct_mat", dct)):
            if t is not None:
                _require_cuda_f32(t, name)
                if t.device != dev:
                    raise RuntimeError(f"audio_b200: {name} is on {t.device} but window is on {dev}")
        if window.numel() != self.desc.win_length:
            raise RuntimeError(
                f"expected a 1D window tensor of size equal to win_length={self.desc.win_length}, "
                f"but got: window size={window.numel()}"
            )
        nbytes = lib.b200a_frontend_workspace_bytes(self.desc)
        if nbytes == 0:
            raise _lib.B200AudioError(_lib.EUNSUPPORTED, "frontend_workspace_bytes (descriptor rejected)")
        window_c = window.contiguous()
        fb_c = None if fb is None else fb.contiguous()
        dct_c = None if dct is None else dct.contiguous()
        with torch.cuda.device(dev):
            ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            rc = lib.b200a_frontend_prepare(
                self.desc,
                window_c.data_ptr(),
                None if fb_c is None else fb_c.data_ptr(),
                None if dct_c is None else dct_c.data_ptr(),
                ws.data_ptr(),
                nbytes,
                _stream_ptr(dev),
            )
        _lib.check(rc, "frontend_prepare")
        return ws

    def frames(self, length: int) -> int:
        return _lib.lib().b200a_num_frames(length, self.desc.n_fft, self.desc.hop, self.desc.center, self.desc.pad)

    def run(
        self,
        ws: torch.Tensor,
        stage: int,
        waveform: torch.Tensor,
        group_max: Optional[torch.Tensor] = None,
        rows_per_group: int = 1,
        constants=None,
        switch=is_differentiable,
    ) -> torch.Tensor:
        """Launch the fused kernel; returns the FRAME-MAJOR result (rows, T, width[, 2]).

        ``constants``: ``(name, tensor)`` pairs of the module buffers the workspace was built from, given by the entry
        points that support waveform gradients (COMPLEX / POWER / MEL stages) when ``switch()`` is on; ``None`` keeps
        the call forward-only.
        """
        _require_cuda_f32(waveform, "waveform")
        grad = constants is not None and _wants_grad(waveform, constants, switch)
        if not grad:
            _no_autograd(waveform)
        flat, stride, frames = self._pack(ws, waveform)
        n_bins = _lib.lib().b200a_num_bins(self.desc.n_fft, self.desc.onesided)
        width = self.desc.n_mels if stage >= _lib.STAGE_MEL else n_bins
        # through the dispatcher (b200audio::frontend_run, audio_b200/_ops.py): allocates `out`, launches on the
        # current stream of the waveform's device, raises on a negative status
        desc_i, desc_f = self._packed_desc()
        if grad:
            return _FrontendFunction.apply(flat, ws, desc_i, desc_f, stage, frames, width, stride)
        return _ops.frontend_run(flat, ws, desc_i, desc_f, stage, frames, width, stride, group_max, rows_per_group)

    def _pack(self, ws: torch.Tensor, waveform: torch.Tensor):
        """The packed (rows, L) waveform, its row stride and its frame count."""
        if waveform.device != ws.device:
            raise RuntimeError(f"audio_b200: waveform is on {waveform.device} but the module buffers are on {ws.device}")
        d = self.desc
        flat, stride = pack_rows(waveform)
        length = flat.shape[1]
        frames = self.frames(length)
        if frames < 1:
            raise RuntimeError(
                f"audio_b200: waveform of {length} samples is too short for n_fft={d.n_fft} "
                f"(center={bool(d.center)}, pad={d.pad})"
            )
        return flat, stride, frames

    def mfcc_grad(self, ws: torch.Tensor, waveform: torch.Tensor, groups: int, rows_per_group: int,
                  top_db: Optional[float]) -> torch.Tensor:
        """The FEAT stage + mfcc_finish of an input that requires grad (the caller checked the feature switch and the
        constant buffers): the frame-major (rows, T, n_mfcc) cepstra of ``_MfccFunction``.  ``groups`` > 0 clamps."""
        flat, stride, frames = self._pack(ws, waveform)
        desc_i, desc_f = self._packed_desc()
        return _MfccFunction.apply(flat, ws, desc_i, desc_f, frames, stride, groups, rows_per_group,
                                   -1.0 if top_db is None else float(top_db))

    def mfcc_finish(self, ws, feat, group_max, rows_per_group: int, top_db: Optional[float]) -> torch.Tensor:
        desc_i, desc_f = self._packed_desc()
        return _ops.mfcc_finish(feat, ws, desc_i, desc_f, group_max, rows_per_group, -1.0 if top_db is None else float(top_db))

    def _packed_desc(self):
        if self._desc_lists is None:
            self._desc_lists = _ops.pack(self.desc)
        return self._desc_lists


_RANK_MESSAGE = ("torch.linalg.lstsq: The least squares solution could not be computed because the input matrix does not "
                 "have full rank (error code: {}).")


class InverseMelPlan:
    """InverseMelScale's banded L D L^T factorisation of G = fb^T fb (b200a_inverse_mel_plan) on fb's device.  Built on
    the host from one device-to-host copy of ``fb`` and uploaded once; rebuilt only when ``fb`` changes (a
    :class:`StampCache`).  The errors of the reference's ``lstsq`` are raised here, at ``forward``."""

    def __init__(self, driver: str):
        self.driver = driver
        self._cache = StampCache()

    @property
    def _plan(self) -> Optional[torch.Tensor]:
        """The uploaded blob of the last build (None before the first)."""
        return self._cache.value

    def plan(self, fb: torch.Tensor) -> torch.Tensor:
        return self._cache.get((fb,), self._build)

    def _build(self, fb: torch.Tensor) -> torch.Tensor:
        import ctypes

        lib = _lib.lib()
        n_stft, n_mels = fb.shape
        nbytes = lib.b200a_inverse_mel_plan_bytes(n_stft, n_mels)
        blob = torch.zeros(nbytes, dtype=torch.uint8)
        fb_host = fb.detach().to("cpu").contiguous()
        bw, pivot = ctypes.c_int32(), ctypes.c_int32()
        rc = lib.b200a_inverse_mel_plan(fb_host.data_ptr(), n_stft, n_mels, _lib.LSTSQ_DRIVER[self.driver], blob.data_ptr(),
                                        nbytes, ctypes.byref(bw), ctypes.byref(pivot))
        if rc == _lib.ESINGULAR and self.driver == "gels":
            raise torch.linalg.LinAlgError(_RANK_MESSAGE.format(pivot.value + 1))
        if rc == _lib.ESINGULAR:
            raise RuntimeError(
                f"audio_b200: InverseMelScale(driver={self.driver!r}) on a rank-deficient filterbank (first zero pivot at "
                f"filter {pivot.value} of fb{tuple(fb.shape)}) is not supported: the rank-revealing drivers return "
                "different answers there; drop the empty filters or use driver='gels', which raises as the reference does")
        if rc == _lib.EUNSUPPORTED:
            raise RuntimeError(
                f"audio_b200: InverseMelScale with fb{tuple(fb.shape)} is not supported: it needs n_mels <= n_stft "
                f"(an underdetermined system), n_mels <= {_lib.INVERSE_MEL_MAX_MELS} and a Gram bandwidth <= "
                f"{_lib.INVERSE_MEL_MAX_BANDWIDTH} (this bank: {bw.value})")
        _lib.check(rc, "inverse_mel_plan")
        return blob.to(fb.device)


class _InverseMelFunction(torch.autograd.Function):
    """b200audio::inverse_mel on the packed (rows, n_mels, T) mel spectrogram, with b200audio::inverse_mel_backward as its
    backward.  The mel input goes through save_for_backward (in-place edits are detected); the forward's plan is kept,
    so an fb changed before backward does not change the gradient."""

    @staticmethod
    def forward(ctx, m3, plan, n_stft):
        ctx.save_for_backward(m3)
        ctx.plan, ctx.n_stft = plan, n_stft
        return _ops.inverse_mel(m3, plan, n_stft)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        (m3,) = ctx.saved_tensors
        return _ops.inverse_mel_backward(g, m3, ctx.plan, ctx.n_stft).transpose(1, 2), None, None


def new_group_max(groups: int, device: torch.device) -> torch.Tensor:
    """[groups] running maxima initialised to -inf by the library's fill kernel."""
    with torch.cuda.device(device):
        g = torch.empty(groups, dtype=torch.float32, device=device)
        _lib.check(_lib.lib().b200a_fill_f32(g.data_ptr(), groups, float("-inf"), _stream_ptr(device)), "fill_f32")
    return g


class _ResampleFunction(torch.autograd.Function):
    """b200audio::resample_run on the packed (rows, L) waveform, sliced to out_len inside (so autograd adds no
    slice_backward fill), with b200audio::resample_backward as its backward.  The map is linear: only the backward
    workspace built from the forward's kernel is kept, so a kernel edited after the forward does not change the
    gradient."""

    @staticmethod
    def forward(ctx, flat, ws, k, bws, orig_r, new_r, width, stride, out_len, pitch):
        buf = _ops.resample_run(flat, ws, k, orig_r, new_r, width, stride, out_len, pitch)
        ctx.bws, ctx.ratio, ctx.length = bws, (orig_r, new_r, width), flat.shape[1]
        return buf[:, :out_len]

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        grad = _ops.resample_backward(grad_out, ctx.bws, *ctx.ratio, ctx.length)
        return grad, None, None, None, None, None, None, None, None, None


class ResamplePlan:
    """Per-phase tap supports of a cached sinc kernel, kept next to the kernel buffer; the adjoint tables are built
    from the same kernel on the first forward that wants a gradient."""

    def __init__(self, orig_r: int, new_r: int, width: int):
        self.orig_r, self.new_r, self.width = int(orig_r), int(new_r), int(width)
        self.taps = 2 * self.width + self.orig_r
        self._forward = StampCache()  # (workspace, contiguous kernel) keyed on the kernel buffer
        self._backward = StampCache()  # adjoint tables keyed on the contiguous kernel the forward was built from

    def workspace(self, kernel: torch.Tensor):
        """The prepared workspace and the contiguous (new_r, taps) kernel it was built from."""
        return self._forward.get((kernel,), self._prepare)

    def _prepare(self, kernel: torch.Tensor):
        _require_cuda_f32(kernel, "kernel")
        if kernel.numel() != self.new_r * self.taps:
            raise RuntimeError(
                f"audio_b200: resample kernel has {kernel.numel()} elements, expected {self.new_r}x{self.taps}"
            )
        lib = _lib.lib()
        dev = kernel.device
        k = kernel.reshape(self.new_r, self.taps).contiguous()
        nbytes = lib.b200a_resample_workspace_bytes(self.new_r, self.taps)
        with torch.cuda.device(dev):
            ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            rc = lib.b200a_resample_prepare(k.data_ptr(), self.orig_r, self.new_r, self.width, ws.data_ptr(), nbytes, _stream_ptr(dev))
        _lib.check(rc, "resample_prepare")
        return ws, k

    def backward_workspace(self) -> torch.Tensor:
        """The adjoint tables of the kernel the forward workspace was last built from (call after ``workspace``)."""
        return self._backward.get((self._forward.value[1],), self._prepare_backward)

    def _prepare_backward(self, k: torch.Tensor) -> torch.Tensor:
        lib = _lib.lib()
        dev = k.device
        nbytes = lib.b200a_resample_backward_workspace_bytes(self.orig_r, self.new_r, self.width)
        with torch.cuda.device(dev):
            bws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            rc = lib.b200a_resample_backward_prepare(k.data_ptr(), self.orig_r, self.new_r, self.width, bws.data_ptr(),
                                                     nbytes, _stream_ptr(dev))
        _lib.check(rc, "resample_backward_prepare")
        return bws

    def run(self, kernel: torch.Tensor, waveform: torch.Tensor) -> torch.Tensor:
        _require_cuda_f32(waveform, "waveform")
        grad = _wants_grad(waveform, (("kernel", kernel),), is_resample_differentiable)
        if not grad:
            _no_autograd(waveform)
        ws, k = self.workspace(kernel)
        if waveform.device != ws.device:
            raise RuntimeError(f"audio_b200: waveform is on {waveform.device} but the kernel buffer is on {ws.device}")
        flat, stride = pack_rows(waveform)
        rows, length = flat.shape
        out_len = resample_len(length, self.orig_r, self.new_r)
        # the reference returns a view into (rows, frames*new') memory: keep that row pitch
        pitch = (length // self.orig_r + 1) * self.new_r
        if grad:
            out = _ResampleFunction.apply(flat, ws, k, self.backward_workspace(), self.orig_r, self.new_r, self.width,
                                          stride, out_len, pitch)
        else:
            buf = _ops.resample_run(flat, ws, k, self.orig_r, self.new_r, self.width, stride, out_len, pitch)
            out = buf[:, :out_len]
        return out.view(waveform.shape[:-1] + (out_len,)) if rows > 0 else out.reshape(waveform.shape[:-1] + (out_len,))
