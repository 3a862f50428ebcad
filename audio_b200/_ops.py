"""``torch.library`` registration of the hot-path ops, so the dispatcher, ``torch.profiler`` and CUDA-graph
capture tooling see them as ``b200audio::<name>``.  Each op is defined by one ``_op`` call next to its two
implementations.

Same shape as the reference's native ops -- ``STABLE_TORCH_LIBRARY_FRAGMENT(torchaudio, m){ m.def(...) }`` with a
per-backend ``..._IMPL(torchaudio, CUDA, m)`` (pytorch/audio/src/libtorchaudio/lfilter.cpp:118-138) bound on the
Python side as ``torch.ops.torchaudio.X`` (pytorch/audio/src/torchaudio/functional/filtering.py:935-938): here the
schema is defined from Python (the library itself has no torch headers), the CUDA implementation forwards to the
C ABI of libb200audio.so on the current stream, and a Meta implementation gives shapes for fake tensors.  There is
deliberately NO CPU implementation: a CPU tensor fails in the dispatcher ("no kernel for CPU"), never falls back.

A descriptor structure (``b200a_frontend_desc``, ``b200a_kaldi_desc``, ``b200a_vad_desc``: plain old data) travels as
an ``int[]`` and a ``float[]`` list: ``pack`` and ``unpack`` derive both from the structure's ``_fields_``.
"""
from __future__ import annotations

import ctypes
import functools

import torch

from . import _lib


@functools.cache
def _layout(cls):
    """(int field names, float field names, position in ints + floats of each field in struct order) of a descriptor
    structure.  Integer fields go to the int[] list and floating-point fields to the float[] list, in struct order."""
    ints = tuple(name for name, ctype in cls._fields_ if ctype in (ctypes.c_int32, ctypes.c_int64))
    floats = tuple(name for name, ctype in cls._fields_ if ctype in (ctypes.c_float, ctypes.c_double))
    names = ints + floats
    if len(names) != len(cls._fields_):
        raise TypeError(f"{cls.__name__} has fields that are neither integers nor floats; it cannot be packed")
    return ints, floats, tuple(names.index(name) for name, _ in cls._fields_)


def pack(d: ctypes.Structure):
    """The (ints, floats) lists of a descriptor structure, as the ops' ``int[]`` / ``float[]`` arguments take it."""
    ints, floats, _ = _layout(type(d))
    return [getattr(d, name) for name in ints], [getattr(d, name) for name in floats]


def unpack(cls, ints, floats):
    """The ``cls`` descriptor that ``pack`` turned into ``ints`` and ``floats``."""
    int_names, float_names, order = _layout(cls)
    if len(ints) != len(int_names) or len(floats) != len(float_names):
        raise ValueError(f"audio_b200: a packed {cls.__name__} has {len(int_names)} ints and {len(float_names)} floats, "
                         f"got {len(ints)} and {len(floats)}")
    values = [*ints, *floats]
    return cls(*[values[i] for i in order])  # positional construction: the fastest way to fill every field


def field_index(cls, name: str) -> int:
    """Where field ``name`` of ``cls`` sits in the list ``pack`` puts it in."""
    ints, floats, _ = _layout(cls)
    return ints.index(name) if name in ints else floats.index(name)


_LIB = torch.library.Library("b200audio", "DEF")


def _op(schema: str, cuda, meta):
    """Define ``b200audio::<name>`` from ``schema`` with its CUDA and Meta implementations; returns the op."""
    name = _LIB.define(schema)
    _LIB.impl(name, cuda, "CUDA")
    _LIB.impl(name, meta, "Meta")
    return getattr(torch.ops.b200audio, name)


def _stream(dev: torch.device) -> int:
    return torch.cuda.current_stream(dev).cuda_stream


def _out_shape(wave, stage, frames, width):
    rows = wave.shape[0]
    return (rows, frames, width, 2) if stage == _lib.STAGE_COMPLEX else (rows, frames, width)


# ---- frontend_run ------------------------------------------------------------------------------------------------
def _frontend_run_cuda(wave, workspace, desc_i, desc_f, stage, frames, width, row_stride, group_max, rows_per_group):
    d = unpack(_lib.FrontendDesc, desc_i, desc_f)
    dev = wave.device
    with torch.cuda.device(dev):
        out = torch.empty(_out_shape(wave, stage, frames, width), dtype=torch.float32, device=dev)
        rc = _lib.lib().b200a_frontend_run(
            d, workspace.data_ptr(), stage, wave.data_ptr(), wave.shape[0], wave.shape[1], row_stride, out.data_ptr(),
            None if group_max is None else group_max.data_ptr(), rows_per_group, _stream(dev))
    if rc == _lib.ESHORT:
        raise RuntimeError(
            f"audio_b200: padding size n_fft//2={d.n_fft // 2} should be less than the input length "
            f"{wave.shape[1] + 2 * d.pad} for pad_mode reflect/circular (torch.stft raises the same way)")
    _lib.check(rc, "frontend_run")
    return out


def _frontend_run_meta(wave, workspace, desc_i, desc_f, stage, frames, width, row_stride, group_max, rows_per_group):
    return wave.new_empty(_out_shape(wave, stage, frames, width), dtype=torch.float32)


frontend_run = _op(
    "frontend_run(Tensor wave, Tensor workspace, int[] desc_i, float[] desc_f, int stage, int frames, int width, "
    "int row_stride, Tensor(a!)? group_max, int rows_per_group) -> Tensor", _frontend_run_cuda, _frontend_run_meta)


# ---- frontend_backward -------------------------------------------------------------------------------------------
def _complex_strides(grad_out):
    """Element strides of a (rows, T, bins, 2) float gradient in complex elements, copying it when the pairs are not
    adjacent, 8-byte aligned floats."""
    st = grad_out.stride()
    if st[3] != 1 or any(s % 2 for s in st[:3]) or grad_out.data_ptr() % 8:
        grad_out = grad_out.contiguous()
        st = grad_out.stride()
    return grad_out, (st[0] // 2, st[1] // 2, st[2] // 2)


def _frontend_backward_cuda(wave, workspace, desc_i, desc_f, stage, row_stride, grad_out):
    d = unpack(_lib.FrontendDesc, desc_i, desc_f)
    rows, length = wave.shape
    dev = wave.device
    if stage == _lib.STAGE_COMPLEX:
        grad_out, gs = _complex_strides(grad_out)
    else:
        gs = grad_out.stride()
    lib = _lib.lib()
    with torch.cuda.device(dev):
        grad = torch.empty((rows, length), dtype=torch.float32, device=dev)
        nbytes = lib.b200a_frontend_backward_scratch_bytes(d, stage, rows, length)
        scratch = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        rc = lib.b200a_frontend_backward(
            d, workspace.data_ptr(), stage, wave.data_ptr(), rows, length, row_stride, grad_out.data_ptr(), gs[0], gs[1],
            gs[2], scratch.data_ptr(), grad.data_ptr(), length, _stream(dev))
    _lib.check(rc, "frontend_backward")
    return grad


def _frontend_backward_meta(wave, workspace, desc_i, desc_f, stage, row_stride, grad_out):
    return wave.new_empty(wave.shape, dtype=torch.float32)


frontend_backward = _op(
    "frontend_backward(Tensor wave, Tensor workspace, int[] desc_i, float[] desc_f, int stage, int row_stride, "
    "Tensor grad_out) -> Tensor", _frontend_backward_cuda, _frontend_backward_meta)


# ---- istft_backward ----------------------------------------------------------------------------------------------
def _istft_backward_cuda(grad, workspace, desc_i, desc_f, start, frames):
    """(rows, L) upstream gradient -> (rows, frames, n_fft//2+1, 2) frame-major spectrogram gradient."""
    d = unpack(_lib.FrontendDesc, desc_i, desc_f)
    if grad.shape[0] > 0 and grad.shape[1] > 0 and grad.stride(1) != 1:
        grad = grad.contiguous()
    rows, g_len = grad.shape
    dev = grad.device
    lib = _lib.lib()
    with torch.cuda.device(dev):
        out = torch.empty((rows, frames, d.n_fft // 2 + 1, 2), dtype=torch.float32, device=dev)
        nbytes = lib.b200a_istft_backward_scratch_bytes(d, rows, frames)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev) if nbytes else None
        rc = lib.b200a_istft_backward(
            d, workspace.data_ptr(), grad.data_ptr(), rows, grad.stride(0) if rows > 1 else g_len, start, g_len, frames,
            None if scratch is None else scratch.data_ptr(), out.data_ptr(), _stream(dev))
    _lib.check(rc, "istft_backward")
    return out


def _istft_backward_meta(grad, workspace, desc_i, desc_f, start, frames):
    n_fft = int(desc_i[field_index(_lib.FrontendDesc, "n_fft")])
    return grad.new_empty((grad.shape[0], frames, n_fft // 2 + 1, 2))


istft_backward = _op(
    "istft_backward(Tensor grad, Tensor workspace, int[] desc_i, float[] desc_f, int start, int frames) -> Tensor",
    _istft_backward_cuda, _istft_backward_meta)


# ---- mfcc_finish -------------------------------------------------------------------------------------------------
def _mfcc_finish_cuda(feat, workspace, desc_i, desc_f, group_max, rows_per_group, top_db):
    d = unpack(_lib.FrontendDesc, desc_i, desc_f)
    rows, frames, _ = feat.shape
    dev = feat.device
    with torch.cuda.device(dev):
        out = torch.empty((rows, frames, d.n_mfcc), dtype=torch.float32, device=dev)
        rc = _lib.lib().b200a_mfcc_finish(
            d, workspace.data_ptr(), feat.data_ptr(), rows, frames, None if group_max is None else group_max.data_ptr(),
            rows_per_group, float(top_db), out.data_ptr(), _stream(dev))
    _lib.check(rc, "mfcc_finish")
    return out


def _mfcc_finish_meta(feat, workspace, desc_i, desc_f, group_max, rows_per_group, top_db):
    return feat.new_empty((feat.shape[0], feat.shape[1], int(desc_i[field_index(_lib.FrontendDesc, "n_mfcc")])))


mfcc_finish = _op(
    "mfcc_finish(Tensor feat, Tensor workspace, int[] desc_i, float[] desc_f, Tensor? group_max, int rows_per_group, "
    "float top_db) -> Tensor", _mfcc_finish_cuda, _mfcc_finish_meta)


# ---- mfcc_backward -----------------------------------------------------------------------------------------------
def _mfcc_backward_cuda(grad, feat, mel, group_max, workspace, desc_i, desc_f, rows_per_group, top_db):
    """(rows, T, n_mfcc) cepstral gradient at any element strides -> (rows, T, n_mels) mel-stage gradient."""
    d = unpack(_lib.FrontendDesc, desc_i, desc_f)
    rows, frames, n_mels = mel.shape
    dev = mel.device
    gs = grad.stride()
    lib = _lib.lib()
    clamp = group_max is not None and top_db >= 0 and not d.log_mels
    with torch.cuda.device(dev):
        out = torch.empty((rows, frames, n_mels), dtype=torch.float32, device=dev)
        nbytes = lib.b200a_mfcc_backward_scratch_bytes(d, rows, frames, rows_per_group) if clamp else 0
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev) if nbytes else None
        rc = lib.b200a_mfcc_backward(
            d, workspace.data_ptr(), grad.data_ptr(), gs[0], gs[1], gs[2], feat.data_ptr(), mel.data_ptr(),
            None if group_max is None else group_max.data_ptr(), rows, frames, rows_per_group, float(top_db),
            None if scratch is None else scratch.data_ptr(), out.data_ptr(), _stream(dev))
    _lib.check(rc, "mfcc_backward")
    return out


def _mfcc_backward_meta(grad, feat, mel, group_max, workspace, desc_i, desc_f, rows_per_group, top_db):
    return mel.new_empty(mel.shape)


mfcc_backward = _op(
    "mfcc_backward(Tensor grad, Tensor feat, Tensor mel, Tensor? group_max, Tensor workspace, int[] desc_i, "
    "float[] desc_f, int rows_per_group, float top_db) -> Tensor", _mfcc_backward_cuda, _mfcc_backward_meta)


# ---- amplitude_to_db_backward ------------------------------------------------------------------------------------
def _amplitude_to_db_backward_cuda(grad, x, group_max, groups, multiplier, amin, offset, top_db):
    """Gradient of amplitude_to_DB on the contiguous input x; ``grad`` is read contiguous or as an expanded scalar
    (all strides 0) and copied otherwise."""
    expanded = all(s == 0 for s in grad.stride())
    if not expanded and not grad.is_contiguous():
        grad = grad.contiguous()
    dev = x.device
    lib = _lib.lib()
    group_elems = x.numel() // groups if groups > 0 else 0
    clamp = group_max is not None and top_db >= 0
    with torch.cuda.device(dev):
        out = torch.empty(x.shape, dtype=torch.float32, device=dev)
        nbytes = lib.b200a_amplitude_to_db_backward_scratch_bytes(groups, group_elems) if clamp else 0
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev) if nbytes else None
        rc = lib.b200a_amplitude_to_db_backward(
            x.data_ptr(), grad.data_ptr(), 0 if expanded else 1, groups, group_elems, float(multiplier), float(amin), float(offset),
            float(top_db), None if group_max is None else group_max.data_ptr(),
            None if scratch is None else scratch.data_ptr(), out.data_ptr(), _stream(dev))
    _lib.check(rc, "amplitude_to_db_backward")
    return out


def _amplitude_to_db_backward_meta(grad, x, group_max, groups, multiplier, amin, offset, top_db):
    return x.new_empty(x.shape)


amplitude_to_db_backward = _op(
    "amplitude_to_db_backward(Tensor grad, Tensor x, Tensor? group_max, int groups, float multiplier, float amin, "
    "float offset, float top_db) -> Tensor", _amplitude_to_db_backward_cuda, _amplitude_to_db_backward_meta)


# ---- apply_fbank_backward ----------------------------------------------------------------------------------------
def _apply_fbank_backward_cuda(grad, fb):
    """(rows, T, n_filters) MelScale output gradient at any element strides -> (rows, T, n_bins) frame-major."""
    rows, frames, n_filters = grad.shape
    n_bins = fb.shape[0]
    dev = grad.device
    gs = grad.stride()
    with torch.cuda.device(dev):
        out = torch.empty((rows, frames, n_bins), dtype=torch.float32, device=dev)
        rc = _lib.lib().b200a_apply_fbank_backward(grad.data_ptr(), rows, n_filters, frames, gs[0], gs[2], gs[1],
                                                   fb.data_ptr(), n_bins, out.data_ptr(), _stream(dev))
    _lib.check(rc, "apply_fbank_backward")
    return out


def _apply_fbank_backward_meta(grad, fb):
    return grad.new_empty((grad.shape[0], grad.shape[1], fb.shape[0]))


apply_fbank_backward = _op("apply_fbank_backward(Tensor grad, Tensor fb) -> Tensor", _apply_fbank_backward_cuda,
                           _apply_fbank_backward_meta)


# ---- ratio_backward ----------------------------------------------------------------------------------------------
def _ratio_backward_cuda(grad, pairs):
    """(rows, T) SpectralCentroid gradient at any element strides -> (rows, T, 2) gradient of the (N, D) pairs."""
    rows, frames = grad.shape
    dev = grad.device
    with torch.cuda.device(dev):
        out = torch.empty((rows, frames, 2), dtype=torch.float32, device=dev)
        rc = _lib.lib().b200a_ratio_backward(pairs.data_ptr(), grad.data_ptr(), rows, frames, grad.stride(0),
                                             grad.stride(1), out.data_ptr(), _stream(dev))
    _lib.check(rc, "ratio_backward")
    return out


def _ratio_backward_meta(grad, pairs):
    return pairs.new_empty(pairs.shape)


ratio_backward = _op("ratio_backward(Tensor grad, Tensor pairs) -> Tensor", _ratio_backward_cuda, _ratio_backward_meta)


# ---- resample_run ------------------------------------------------------------------------------------------------
def _resample_run_cuda(wave, workspace, kernel, orig_r, new_r, width, row_stride, out_len, pitch):
    rows, length = wave.shape
    dev = wave.device
    with torch.cuda.device(dev):
        buf = torch.empty((rows, pitch), dtype=torch.float32, device=dev)
        rc = _lib.lib().b200a_resample_run(
            workspace.data_ptr(), kernel.data_ptr(), orig_r, new_r, width, wave.data_ptr(), rows, length, row_stride,
            buf.data_ptr(), pitch, out_len, _stream(dev))
    _lib.check(rc, "resample_run")
    return buf


def _resample_run_meta(wave, workspace, kernel, orig_r, new_r, width, row_stride, out_len, pitch):
    return wave.new_empty((wave.shape[0], pitch))


resample_run = _op(
    "resample_run(Tensor wave, Tensor workspace, Tensor kernel, int orig_r, int new_r, int width, int row_stride, "
    "int out_len, int pitch) -> Tensor", _resample_run_cuda, _resample_run_meta)


# ---- resample_backward -------------------------------------------------------------------------------------------
def _resample_backward_cuda(grad, workspace, orig_r, new_r, width, length):
    """(rows, out_len) upstream gradient -> (rows, length) waveform gradient."""
    if grad.shape[0] > 0 and grad.shape[1] > 0 and grad.stride(1) != 1:
        grad = grad.contiguous()
    rows, out_len = grad.shape
    dev = grad.device
    with torch.cuda.device(dev):
        out = torch.empty((rows, length), dtype=torch.float32, device=dev)
        rc = _lib.lib().b200a_resample_backward(
            workspace.data_ptr(), orig_r, new_r, width, grad.data_ptr(), rows, grad.stride(0) if rows > 1 else out_len,
            out_len, out.data_ptr(), length, length, _stream(dev))
    _lib.check(rc, "resample_backward")
    return out


def _resample_backward_meta(grad, workspace, orig_r, new_r, width, length):
    return grad.new_empty((grad.shape[0], length))


resample_backward = _op(
    "resample_backward(Tensor grad, Tensor workspace, int orig_r, int new_r, int width, int length) -> Tensor",
    _resample_backward_cuda, _resample_backward_meta)


# ---- kaldi_run / kaldi_backward ---------------------------------------------------------------------------------
def _kaldi_run_cuda(wave, workspace, desc_i, desc_f, kaldi_i, kaldi_f, stage, frames, width, row_stride):
    """(rows, L) waveform -> (rows, frames, width) Kaldi feature rows (b200a_kaldi_run)."""
    d, k = unpack(_lib.FrontendDesc, desc_i, desc_f), unpack(_lib.KaldiDesc, kaldi_i, kaldi_f)
    rows, length = wave.shape
    dev = wave.device
    with torch.cuda.device(dev):
        out = torch.empty((rows, frames, width), dtype=torch.float32, device=dev)
        rc = _lib.lib().b200a_kaldi_run(k, d, workspace.data_ptr(), stage, wave.data_ptr(), rows, length, row_stride,
                                        out.data_ptr(), _stream(dev))
    _lib.check(rc, "kaldi_run")
    return out


def _kaldi_run_meta(wave, workspace, desc_i, desc_f, kaldi_i, kaldi_f, stage, frames, width, row_stride):
    return wave.new_empty((wave.shape[0], frames, width), dtype=torch.float32)


kaldi_run = _op(
    "kaldi_run(Tensor wave, Tensor workspace, int[] desc_i, float[] desc_f, int[] kaldi_i, float[] kaldi_f, int stage, "
    "int frames, int width, int row_stride) -> Tensor", _kaldi_run_cuda, _kaldi_run_meta)


def _kaldi_backward_cuda(wave, workspace, desc_i, desc_f, kaldi_i, kaldi_f, stage, row_stride, grad_out):
    """(rows, frames, width) feature-row gradient at any element strides -> (rows, L) waveform gradient."""
    d, k = unpack(_lib.FrontendDesc, desc_i, desc_f), unpack(_lib.KaldiDesc, kaldi_i, kaldi_f)
    rows, length = wave.shape
    dev = wave.device
    gs = grad_out.stride()
    lib = _lib.lib()
    with torch.cuda.device(dev):
        grad = torch.empty((rows, length), dtype=torch.float32, device=dev)
        nbytes = lib.b200a_kaldi_backward_scratch_bytes(k, d, stage, rows, length)
        scratch = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        rc = lib.b200a_kaldi_backward(k, d, workspace.data_ptr(), stage, wave.data_ptr(), rows, length, row_stride,
                                      grad_out.data_ptr(), gs[0], gs[1], gs[2], scratch.data_ptr(), grad.data_ptr(), length,
                                      _stream(dev))
    _lib.check(rc, "kaldi_backward")
    return grad


def _kaldi_backward_meta(wave, workspace, desc_i, desc_f, kaldi_i, kaldi_f, stage, row_stride, grad_out):
    return wave.new_empty(wave.shape, dtype=torch.float32)


kaldi_backward = _op(
    "kaldi_backward(Tensor wave, Tensor workspace, int[] desc_i, float[] desc_f, int[] kaldi_i, float[] kaldi_f, "
    "int stage, int row_stride, Tensor grad_out) -> Tensor", _kaldi_backward_cuda, _kaldi_backward_meta)


# ---- phase_vocoder_backward --------------------------------------------------------------------------------------
def _phase_vocoder_backward_cuda(spec, out, grad, rate):
    """(rows, bins, frames_in) complex64 input of the forward, its (rows, frames_out, bins, 2) frame-major output and
    the (rows, bins, frames_out) complex upstream gradient at any strides (0 included) -> (rows, frames_in, bins, 2)
    frame-major spectrogram gradient."""
    rows, bins, frames_in = spec.shape
    frames_out = out.shape[1]
    spec_r, ss = _complex_strides(torch.view_as_real(spec.resolve_conj()))
    grad_r, gs = _complex_strides(torch.view_as_real(grad.resolve_conj()))
    dev = spec.device
    with torch.cuda.device(dev):
        gx = torch.empty((rows, frames_in, bins, 2), dtype=torch.float32, device=dev)
        rc = _lib.lib().b200a_phase_vocoder_backward(
            spec_r.data_ptr(), ss[0], ss[1], ss[2], rows, bins, frames_in, float(rate), out.data_ptr(), grad_r.data_ptr(),
            gs[0], gs[1], gs[2], gx.data_ptr(), frames_out, _stream(dev))
    _lib.check(rc, "phase_vocoder_backward")
    return gx


def _phase_vocoder_backward_meta(spec, out, grad, rate):
    return spec.new_empty((spec.shape[0], spec.shape[2], spec.shape[1], 2), dtype=torch.float32)


phase_vocoder_backward = _op("phase_vocoder_backward(Tensor spec, Tensor out, Tensor grad, float rate) -> Tensor",
                             _phase_vocoder_backward_cuda, _phase_vocoder_backward_meta)


# ---- rnnt_features / rnnt_features_backward ----------------------------------------------------------------------
def _rnnt_shapes(wave, desc_i, out_frames, pad_frames):
    n_mels = int(desc_i[field_index(_lib.FrontendDesc, "n_mels")])
    return (wave.shape[0], out_frames + pad_frames, n_mels), (wave.shape[0], out_frames, n_mels)


def _rnnt_features_cuda(wave, workspace, desc_i, desc_f, lengths, stats, gain, out_frames, pad_frames, row_stride, with_mel):
    """(rows, L) waveform -> ((rows, out_frames + pad_frames, n_mels) features, (rows, out_frames, n_mels) mel values
    or an empty tensor).  ``pad_frames`` zero rows after the features (one row only) are written by b200a_fill_f32."""
    d = unpack(_lib.FrontendDesc, desc_i, desc_f)
    rows, length = wave.shape
    if pad_frames > 0 and rows != 1:
        raise RuntimeError("audio_b200: rnnt_features pads a single row only")
    out_shape, mel_shape = _rnnt_shapes(wave, desc_i, out_frames, pad_frames)
    dev = wave.device
    lib = _lib.lib()
    with torch.cuda.device(dev):
        out = torch.empty(out_shape, dtype=torch.float32, device=dev)
        mel = torch.empty(mel_shape if with_mel else (0,), dtype=torch.float32, device=dev)
        rc = lib.b200a_rnnt_features_run(
            d, workspace.data_ptr(), wave.data_ptr(), rows, length, row_stride,
            None if lengths is None else lengths.data_ptr(), stats.data_ptr(), float(gain), out_frames, out.data_ptr(),
            mel.data_ptr() if with_mel else None, _stream(dev))
        if rc == _lib.OK and pad_frames > 0:
            n = pad_frames * d.n_mels
            rc = lib.b200a_fill_f32(out.data_ptr() + 4 * out_frames * d.n_mels, n, 0.0, _stream(dev))
    if rc == _lib.ESHORT:
        raise RuntimeError(
            f"audio_b200: padding size n_fft//2={d.n_fft // 2} should be less than the input length "
            f"{length + 2 * d.pad} for pad_mode reflect/circular (torch.stft raises the same way)")
    _lib.check(rc, "rnnt_features")
    return out, mel


def _rnnt_features_meta(wave, workspace, desc_i, desc_f, lengths, stats, gain, out_frames, pad_frames, row_stride, with_mel):
    out_shape, mel_shape = _rnnt_shapes(wave, desc_i, out_frames, pad_frames)
    return wave.new_empty(out_shape, dtype=torch.float32), wave.new_empty(mel_shape if with_mel else (0,),
                                                                           dtype=torch.float32)


rnnt_features = _op(
    "rnnt_features(Tensor wave, Tensor workspace, int[] desc_i, float[] desc_f, Tensor? lengths, Tensor stats, float gain, "
    "int out_frames, int pad_frames, int row_stride, bool with_mel) -> (Tensor, Tensor)",
    _rnnt_features_cuda, _rnnt_features_meta)


def _rnnt_features_backward_cuda(stats, gain, mel, grad):
    """(rows, T, n_mels) feature gradient at any element strides (0 included) -> (rows, T, n_mels) mel gradient."""
    rows, frames, n_mels = mel.shape
    dev = mel.device
    gs = grad.stride()
    with torch.cuda.device(dev):
        out = torch.empty((rows, frames, n_mels), dtype=torch.float32, device=dev)
        rc = _lib.lib().b200a_rnnt_features_backward(stats.data_ptr(), float(gain), mel.data_ptr(), grad.data_ptr(), gs[0],
                                                     gs[1], gs[2], rows, frames, n_mels, out.data_ptr(), _stream(dev))
    _lib.check(rc, "rnnt_features_backward")
    return out


def _rnnt_features_backward_meta(stats, gain, mel, grad):
    return mel.new_empty(mel.shape)


rnnt_features_backward = _op("rnnt_features_backward(Tensor stats, float gain, Tensor mel, Tensor grad) -> Tensor",
                             _rnnt_features_backward_cuda, _rnnt_features_backward_meta)


# ---- inverse_mel / inverse_mel_backward ----------------------------------------------------------------------------
def _inverse_mel_cuda(mel, plan, n_stft):
    """(rows, n_mels, T) mel spectrogram at any element strides -> (rows, T, n_stft) frame-major linear spectrogram."""
    rows, n_mels, frames = mel.shape
    dev = mel.device
    ms = mel.stride()
    with torch.cuda.device(dev):
        out = torch.empty((rows, frames, n_stft), dtype=torch.float32, device=dev)
        rc = _lib.lib().b200a_inverse_mel_run(plan.data_ptr(), n_stft, n_mels, mel.data_ptr(), rows, frames, ms[0], ms[1],
                                              ms[2], out.data_ptr(), _stream(dev))
    _lib.check(rc, "inverse_mel")
    return out


def _inverse_mel_meta(mel, plan, n_stft):
    return mel.new_empty((mel.shape[0], mel.shape[2], n_stft))


inverse_mel = _op("inverse_mel(Tensor mel, Tensor plan, int n_stft) -> Tensor", _inverse_mel_cuda, _inverse_mel_meta)


def _inverse_mel_backward_cuda(grad, mel, plan, n_stft):
    """(rows, T, n_stft) output gradient at any element strides (0 included) -> (rows, T, n_mels) frame-major."""
    rows, n_mels, frames = mel.shape
    dev = mel.device
    ms, gs = mel.stride(), grad.stride()
    with torch.cuda.device(dev):
        out = torch.empty((rows, frames, n_mels), dtype=torch.float32, device=dev)
        rc = _lib.lib().b200a_inverse_mel_backward(plan.data_ptr(), n_stft, n_mels, mel.data_ptr(), rows, frames, ms[0],
                                                   ms[1], ms[2], grad.data_ptr(), gs[0], gs[1], gs[2], out.data_ptr(),
                                                   _stream(dev))
    _lib.check(rc, "inverse_mel_backward")
    return out


def _inverse_mel_backward_meta(grad, mel, plan, n_stft):
    return mel.new_empty((mel.shape[0], mel.shape[2], mel.shape[1]))


inverse_mel_backward = _op("inverse_mel_backward(Tensor grad, Tensor mel, Tensor plan, int n_stft) -> Tensor",
                           _inverse_mel_backward_cuda, _inverse_mel_backward_meta)


# ---- lfilter / lfilter_backward ---------------------------------------------------------------------------------
def _lfilter_strides(x):
    """Batch and filter element strides of a (batch, n_filters, T) input with a unit (or irrelevant) time stride."""
    return x.stride(0), x.stride(1)


def _lfilter_cuda(x, a, b, clamp, reverse, with_raw):
    """(batch, n_filters, T) waveform rows at any batch / filter strides (0 included), unit time stride, and
    (n_filters, n_order) contiguous coefficients -> (y, unclamped y or an empty tensor), both contiguous."""
    batch, n_filters, length = x.shape
    n_order = a.shape[1]
    dev = x.device
    lib = _lib.lib()
    sb, sf = _lfilter_strides(x)
    with torch.cuda.device(dev):
        y = torch.empty((batch, n_filters, length), dtype=torch.float32, device=dev)
        raw = torch.empty((batch, n_filters, length) if with_raw else (0,), dtype=torch.float32, device=dev)
        nbytes = lib.b200a_lfilter_workspace_bytes(batch * n_filters, length, n_order, n_filters)
        ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        rc = lib.b200a_lfilter_run(a.data_ptr(), b.data_ptr(), n_filters, n_order, x.data_ptr(), batch, length, sb, sf,
                                   int(clamp), int(reverse), y.data_ptr(), raw.data_ptr() if with_raw else None,
                                   ws.data_ptr(), nbytes, _stream(dev))
    _lib.check(rc, "lfilter")
    return y, raw


def _lfilter_meta(x, a, b, clamp, reverse, with_raw):
    return x.new_empty(x.shape), x.new_empty(x.shape if with_raw else (0,))


lfilter = _op("lfilter(Tensor x, Tensor a, Tensor b, bool clamp, bool reverse, bool with_raw) -> (Tensor, Tensor)",
              _lfilter_cuda, _lfilter_meta)


def _lfilter_backward_cuda(grad, x, y_raw, a, b, clamp, reverse):
    """Upstream gradient of the (batch, n_filters, T) output -> (grad_x (batch, n_filters, T), grad_a, grad_b)."""
    batch, n_filters, length = x.shape
    n_order = a.shape[1]
    grad = grad.contiguous()
    dev = x.device
    lib = _lib.lib()
    sb, sf = _lfilter_strides(x)
    with torch.cuda.device(dev):
        gx = torch.empty((batch, n_filters, length), dtype=torch.float32, device=dev)
        ga = torch.empty((n_filters, n_order), dtype=torch.float32, device=dev)
        gb = torch.empty((n_filters, n_order), dtype=torch.float32, device=dev)
        nbytes = lib.b200a_lfilter_backward_workspace_bytes(batch * n_filters, length, n_order, n_filters)
        ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        rc = lib.b200a_lfilter_backward(a.data_ptr(), b.data_ptr(), n_filters, n_order, x.data_ptr(), batch, length, sb,
                                        sf, y_raw.data_ptr(), grad.data_ptr(), int(clamp), int(reverse), gx.data_ptr(),
                                        ga.data_ptr(), gb.data_ptr(), ws.data_ptr(), nbytes, _stream(dev))
    _lib.check(rc, "lfilter_backward")
    return gx, ga, gb


def _lfilter_backward_meta(grad, x, y_raw, a, b, clamp, reverse):
    return x.new_empty(x.shape), a.new_empty(a.shape), b.new_empty(b.shape)


lfilter_backward = _op(
    "lfilter_backward(Tensor grad, Tensor x, Tensor y_raw, Tensor a, Tensor b, bool clamp, bool reverse) "
    "-> (Tensor, Tensor, Tensor)", _lfilter_backward_cuda, _lfilter_backward_meta)


# ---- fftconvolve / fftconvolve_backward -------------------------------------------------------------------------
def _fftconvolve_desc(x, y, x_index, y_index, start, out_len):
    if not (x_index.is_contiguous() and y_index.is_contiguous() and x_index.dtype == y_index.dtype == torch.int64):
        raise ValueError("fftconvolve: the row index vectors must be contiguous int64")
    return _lib.FftconvolveDesc(n=x.shape[1], m=y.shape[1], out_len=out_len, start=start, rows=x_index.shape[0],
                                x_rows=x.shape[0], y_rows=y.shape[0], x_index=x_index.data_ptr(),
                                y_index=y_index.data_ptr(), x_stride=x.stride(0), y_stride=y.stride(0))


def _conv_run(kind, x, y, x_index, y_index, start, out_len):
    """(x_rows, N) and (y_rows, M) operand rows with a unit time stride, and int64 (rows,) index vectors naming each
    output row's operand rows -> the (rows, out_len) slice [start, start + out_len) of the full convolution, by
    b200a_{kind}_run."""
    dev = x.device
    lib = _lib.lib()
    d = _fftconvolve_desc(x, y, x_index, y_index, start, out_len)
    with torch.cuda.device(dev):
        out = torch.empty((x_index.shape[0], out_len), dtype=torch.float32, device=dev)
        nbytes = getattr(lib, f"b200a_{kind}_workspace_bytes")(ctypes.byref(d))
        ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        rc = getattr(lib, f"b200a_{kind}_run")(ctypes.byref(d), x.data_ptr(), y.data_ptr(), out.data_ptr(),
                                               ws.data_ptr(), nbytes, _stream(dev))
    _lib.check(rc, kind)
    return out


def _conv_backward(kind, grad, x, y, x_index, y_index, start):
    """Upstream gradient of the (rows, L) output -> per-output-row (grad_x (rows, N), grad_y (rows, M)), by
    b200a_{kind}_backward."""
    dev = x.device
    lib = _lib.lib()
    grad = grad.contiguous()
    d = _fftconvolve_desc(x, y, x_index, y_index, start, grad.shape[1])
    rows = x_index.shape[0]
    with torch.cuda.device(dev):
        gx = torch.empty((rows, x.shape[1]), dtype=torch.float32, device=dev)
        gy = torch.empty((rows, y.shape[1]), dtype=torch.float32, device=dev)
        nbytes = getattr(lib, f"b200a_{kind}_backward_workspace_bytes")(ctypes.byref(d))
        ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        rc = getattr(lib, f"b200a_{kind}_backward")(ctypes.byref(d), x.data_ptr(), y.data_ptr(), grad.data_ptr(),
                                                    gx.data_ptr(), gy.data_ptr(), ws.data_ptr(), nbytes, _stream(dev))
    _lib.check(rc, f"{kind}_backward")
    return gx, gy


def _fftconvolve_cuda(x, y, x_index, y_index, start, out_len):
    return _conv_run("fftconvolve", x, y, x_index, y_index, start, out_len)


def _fftconvolve_meta(x, y, x_index, y_index, start, out_len):
    return x.new_empty((x_index.shape[0], out_len))


fftconvolve = _op("fftconvolve(Tensor x, Tensor y, Tensor x_index, Tensor y_index, int start, int out_len) -> Tensor",
                  _fftconvolve_cuda, _fftconvolve_meta)


def _fftconvolve_backward_cuda(grad, x, y, x_index, y_index, start):
    return _conv_backward("fftconvolve", grad, x, y, x_index, y_index, start)


def _fftconvolve_backward_meta(grad, x, y, x_index, y_index, start):
    rows = x_index.shape[0]
    return x.new_empty((rows, x.shape[1])), y.new_empty((rows, y.shape[1]))


fftconvolve_backward = _op(
    "fftconvolve_backward(Tensor grad, Tensor x, Tensor y, Tensor x_index, Tensor y_index, int start) -> (Tensor, Tensor)",
    _fftconvolve_backward_cuda, _fftconvolve_backward_meta)


# ---- convolve / convolve_backward: the direct method on the same descriptor -----------------------------------------
def _convolve_cuda(x, y, x_index, y_index, start, out_len):
    return _conv_run("convolve", x, y, x_index, y_index, start, out_len)


def _convolve_backward_cuda(grad, x, y, x_index, y_index, start):
    return _conv_backward("convolve", grad, x, y, x_index, y_index, start)


convolve = _op("convolve(Tensor x, Tensor y, Tensor x_index, Tensor y_index, int start, int out_len) -> Tensor",
               _convolve_cuda, _fftconvolve_meta)
convolve_backward = _op(
    "convolve_backward(Tensor grad, Tensor x, Tensor y, Tensor x_index, Tensor y_index, int start) -> (Tensor, Tensor)",
    _convolve_backward_cuda, _fftconvolve_backward_meta)


# ---- vad_walk / vad_trigger ----------------------------------------------------------------------------------------
def _vad_walk_cuda(spectrum, cepstrum_window, rows, workspace, desc_i, desc_f, chunk, frame0):
    """(C, frames, dft/2+1) |X| of a chunk -> bins [s0, s1) of the first `frames` rows of the (C, chunk, dft/2) cepstrum
    rows, carrying the smoothed spectrum and the noise estimate in ``workspace`` (b200a_vad_walk)."""
    d = unpack(_lib.VadDesc, desc_i, desc_f)
    dev = spectrum.device
    with torch.cuda.device(dev):
        rc = _lib.lib().b200a_vad_walk(d, chunk, frame0, spectrum.shape[1], spectrum.data_ptr(), cepstrum_window.data_ptr(),
                                       rows.data_ptr(), workspace.data_ptr(), workspace.numel(), _stream(dev))
    _lib.check(rc, "vad_walk")


def _vad_walk_meta(spectrum, cepstrum_window, rows, workspace, desc_i, desc_f, chunk, frame0):
    return None


vad_walk = _op(
    "vad_walk(Tensor spectrum, Tensor cepstrum_window, Tensor(a!) rows, Tensor(b!) workspace, int[] desc_i, "
    "float[] desc_f, int chunk, int frame0) -> ()", _vad_walk_cuda, _vad_walk_meta)


def _vad_trigger_cuda(power, workspace, desc_i, desc_f, chunk, frame0):
    """(C, frames) cepstral band powers of a chunk -> (C, frames) float32 measures; the trigger status goes to the first
    16 bytes of ``workspace`` (b200a_vad_trigger)."""
    d = unpack(_lib.VadDesc, desc_i, desc_f)
    dev = power.device
    with torch.cuda.device(dev):
        measures = torch.empty(power.shape, dtype=torch.float32, device=dev)
        rc = _lib.lib().b200a_vad_trigger(d, chunk, frame0, power.shape[1], power.data_ptr(), measures.data_ptr(),
                                          workspace.data_ptr(), workspace.numel(), _stream(dev))
    _lib.check(rc, "vad_trigger")
    return measures


def _vad_trigger_meta(power, workspace, desc_i, desc_f, chunk, frame0):
    return power.new_empty(power.shape)


vad_trigger = _op(
    "vad_trigger(Tensor power, Tensor(a!) workspace, int[] desc_i, float[] desc_f, int chunk, int frame0) -> Tensor",
    _vad_trigger_cuda, _vad_trigger_meta)
