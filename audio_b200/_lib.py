"""ctypes binding of libb200audio.so (the C ABI in include/b200audio.h).

This is the stub a pytorch/audio maintainer would add next to
``src/torchaudio/_extension/utils.py:_load_lib``: load the shared object, declare the
argument types, turn negative status codes into exceptions.  There is NO fallback: if the
library is missing the import of any op raises, and ops refuse non-CUDA tensors.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_double, c_float, c_int32, c_int64, c_size_t, c_void_p

_PKG = os.path.dirname(os.path.abspath(__file__))
# B200A_LIB: load another build of the same ABI (A/B timing of kernel changes); the default is the in-tree build
LIB_PATH = os.environ.get("B200A_LIB") or os.path.join(_PKG, "lib", "libb200audio.so")

OK, EINVAL, EUNSUPPORTED, ESHORT, EWORKSPACE, ECUDA, ESINGULAR = 0, -1, -2, -3, -4, -5, -6
PAD_MODE = {"reflect": 0, "constant": 1, "replicate": 2, "circular": 3}
STAGE_COMPLEX, STAGE_POWER, STAGE_MEL, STAGE_FEAT = 0, 1, 2, 3
LSTSQ_DRIVER = {"gels": 0, "gelsy": 1, "gelsd": 2, "gelss": 3}
INVERSE_MEL_MAX_BANDWIDTH, INVERSE_MEL_MAX_MELS = 4, 512  # B200A_INVERSE_MEL_MAX_BANDWIDTH / _MAX_MELS
LFILTER_MAX_ORDER = 16  # B200A_LFILTER_MAX_ORDER
FFTCONVOLVE_MAX_PARTITIONS, FFTCONVOLVE_MAX_BLOCK = 128, 2048  # B200A_FFTCONVOLVE_MAX_PARTITIONS; the largest block
CONVOLVE_MAX_TAPS = 4096  # B200A_CONVOLVE_MAX_TAPS
VAD_MAX_DFT = 8192  # the largest dft_len of b200a_vad_desc
DTYPE_F32, DTYPE_F16, DTYPE_F64 = 0, 1, 2  # B200A_DTYPE_*
RNNT_MAX_U = 8192  # B200A_RNNT_MAX_U
INDEX_I32, INDEX_I64 = 0, 1  # B200A_INDEX_*
FORCED_ALIGN_MAX_L = 8191  # B200A_FORCED_ALIGN_MAX_L
CTC_DECODER_MAX_BEAM, CTC_DECODER_MAX_VOCAB = 128, 1 << 24  # B200A_CTC_DECODER_MAX_BEAM / _MAX_VOCAB
MASK_AXIS_FREQ, MASK_AXIS_TIME = 0, 1  # B200A_MASK_AXIS_*


class FrontendDesc(ctypes.Structure):
    """Mirror of ``b200a_frontend_desc``."""

    _fields_ = [
        ("n_fft", c_int32),
        ("win_length", c_int32),
        ("hop", c_int32),
        ("pad", c_int32),
        ("center", c_int32),
        ("pad_mode", c_int32),
        ("onesided", c_int32),
        ("frame_length_norm", c_int32),
        ("window_norm", c_int32),
        ("power", c_float),
        ("n_mels", c_int32),
        ("n_mfcc", c_int32),
        ("log_mels", c_int32),
        ("db_multiplier", c_float),
        ("db_amin", c_float),
        ("db_offset", c_float),
    ]

    def key(self):
        return tuple(getattr(self, f) for f, _ in self._fields_)


class KaldiDesc(ctypes.Structure):
    """Mirror of ``b200a_kaldi_desc``."""

    _fields_ = [
        ("window_size", c_int32),
        ("window_shift", c_int32),
        ("padded_size", c_int32),
        ("snip_edges", c_int32),
        ("remove_dc_offset", c_int32),
        ("preemphasis", c_float),
        ("energy_mode", c_int32),
        ("energy_floor", c_float),
        ("energy_col", c_int32),
        ("out_width", c_int32),
        ("out_col0", c_int32),
        ("use_log", c_int32),
    ]


class FftconvolveDesc(ctypes.Structure):
    """Mirror of ``b200a_fftconvolve_desc`` (also ``b200a_convolve_desc``)."""

    _fields_ = [
        ("n", c_int64),
        ("m", c_int64),
        ("out_len", c_int64),
        ("start", c_int64),
        ("rows", c_int64),
        ("x_rows", c_int64),
        ("y_rows", c_int64),
        ("x_index", c_void_p),
        ("y_index", c_void_p),
        ("x_stride", c_int64),
        ("y_stride", c_int64),
    ]


class VadDesc(ctypes.Structure):
    """Mirror of ``b200a_vad_desc``."""

    _fields_ = [
        ("channels", c_int32),
        ("dft_len", c_int32),
        ("spectrum_start", c_int32),
        ("spectrum_end", c_int32),
        ("cepstrum_start", c_int32),
        ("cepstrum_end", c_int32),
        ("measures_len", c_int32),
        ("gap_len", c_int32),
        ("boot_count_max", c_int32),
        ("period", c_int32),
        ("fixed_pre_trigger", c_int64),
        ("noise_up_mult", c_double),
        ("noise_down_mult", c_double),
        ("noise_reduction_amount", c_double),
        ("measure_smooth_mult", c_double),
        ("trigger_mult", c_double),
        ("trigger_level", c_double),
    ]


class RnntLossDesc(ctypes.Structure):
    """Mirror of ``b200a_rnnt_loss_desc``."""

    _fields_ = [
        ("batch", c_int32),
        ("max_t", c_int32),
        ("max_u", c_int32),
        ("classes", c_int32),
        ("blank", c_int32),
        ("dtype", c_int32),
        ("fused", c_int32),
        ("clamp", c_float),
    ]


class ForcedAlignDesc(ctypes.Structure):
    """Mirror of ``b200a_forced_align_desc``."""

    _fields_ = [
        ("batch", c_int32),
        ("max_t", c_int32),
        ("max_l", c_int32),
        ("classes", c_int32),
        ("blank", c_int32),
        ("dtype", c_int32),
        ("target_dtype", c_int32),
        ("length_dtype", c_int32),
    ]


class CtcDecoderDesc(ctypes.Structure):
    """Mirror of ``b200a_ctc_decoder_desc``."""

    _fields_ = [
        ("batch", c_int32),
        ("max_t", c_int32),
        ("vocab", c_int32),
        ("beam", c_int32),
        ("threshold", c_float),
    ]


class MaskSpec(ctypes.Structure):
    """Mirror of ``b200a_mask_spec``."""

    _fields_ = [
        ("axis", c_int32),
        ("mask_param", c_int32),
        ("start", c_int64),
        ("end", c_int64),
        ("value_draws", c_void_p),
        ("start_draws", c_void_p),
    ]


class MaskDesc(ctypes.Structure):
    """Mirror of ``b200a_mask_desc``."""

    _fields_ = [
        ("rows0", c_int64),
        ("rows1", c_int64),
        ("freq", c_int64),
        ("time", c_int64),
        ("in_stride", c_int64 * 4),
        ("out_stride", c_int64 * 4),
        ("n_masks", c_int32),
        ("fill", c_float),
    ]


_SIGNATURES = {
    "b200a_version": (ctypes.c_int, []),
    "b200a_strerror": (c_char_p, [ctypes.c_int]),
    "b200a_num_frames": (c_int64, [c_int64, c_int32, c_int32, c_int32, c_int32]),
    "b200a_pad_index": (c_int64, [c_int64, c_int64, c_int32]),
    "b200a_num_bins": (c_int32, [c_int32, c_int32]),
    "b200a_resample_width": (c_int32, [c_int32, c_int32, c_int32, c_double]),
    "b200a_resample_len": (c_int64, [c_int64, c_int32, c_int32]),
    "b200a_resample_support": (ctypes.c_int, [c_int32, c_int32, c_int32, c_double, c_int32, POINTER(c_int32), POINTER(c_int32)]),
    "b200a_frontend_workspace_bytes": (c_size_t, [POINTER(FrontendDesc)]),
    "b200a_frontend_prepare": (
        ctypes.c_int,
        [POINTER(FrontendDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p],
    ),
    "b200a_frontend_run": (
        ctypes.c_int,
        [POINTER(FrontendDesc), c_void_p, c_int32, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_int64, c_void_p],
    ),
    "b200a_frontend_backward": (
        ctypes.c_int,
        [POINTER(FrontendDesc), c_void_p, c_int32, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_int64, c_int64, c_int64,
         c_void_p, c_void_p, c_int64, c_void_p],
    ),
    "b200a_frontend_backward_scratch_bytes": (c_size_t, [POINTER(FrontendDesc), c_int32, c_int64, c_int64]),
    "b200a_rnnt_features_run": (
        ctypes.c_int,
        [POINTER(FrontendDesc), c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_float, c_int64,
         c_void_p, c_void_p, c_void_p],
    ),
    "b200a_rnnt_features_backward": (
        ctypes.c_int,
        [c_void_p, c_float, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_int32, c_void_p, c_void_p],
    ),
    "b200a_mfcc_finish": (
        ctypes.c_int,
        [POINTER(FrontendDesc), c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_int64, c_float, c_void_p, c_void_p],
    ),
    "b200a_apply_fbank": (
        ctypes.c_int,
        [c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_int64, c_void_p, c_int32, c_void_p, c_void_p],
    ),
    "b200a_amplitude_to_db": (
        ctypes.c_int,
        [c_void_p, c_int64, c_int64, c_float, c_float, c_float, c_float, c_void_p, c_void_p, c_void_p],
    ),
    "b200a_mfcc_backward_scratch_bytes": (c_size_t, [POINTER(FrontendDesc), c_int64, c_int64, c_int64]),
    "b200a_mfcc_backward": (
        ctypes.c_int,
        [POINTER(FrontendDesc), c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_int64, c_int64,
         c_int64, c_float, c_void_p, c_void_p, c_void_p],
    ),
    "b200a_amplitude_to_db_backward_scratch_bytes": (c_size_t, [c_int64, c_int64]),
    "b200a_amplitude_to_db_backward": (
        ctypes.c_int,
        [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_float, c_float, c_float, c_float, c_void_p, c_void_p, c_void_p,
         c_void_p],
    ),
    "b200a_apply_fbank_backward": (
        ctypes.c_int,
        [c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_int64, c_void_p, c_int64, c_void_p, c_void_p],
    ),
    "b200a_ratio_backward": (ctypes.c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_void_p, c_void_p]),
    "b200a_istft_run": (
        ctypes.c_int,
        [POINTER(FrontendDesc), c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_int64,
         c_int64, c_int64, c_void_p],
    ),
    "b200a_istft_backward": (
        ctypes.c_int,
        [POINTER(FrontendDesc), c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_void_p],
    ),
    "b200a_istft_backward_scratch_bytes": (c_size_t, [POINTER(FrontendDesc), c_int64, c_int64]),
    "b200a_griffinlim_update": (
        ctypes.c_int,
        [c_void_p, c_int64, c_int64, c_int64, c_float, c_void_p, c_void_p, c_float, c_int32, c_void_p, c_int64, c_int64, c_int64,
         c_void_p],
    ),
    "b200a_phase_vocoder": (
        ctypes.c_int,
        [c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_int64, c_double, c_void_p, c_void_p, c_int64, c_void_p],
    ),
    "b200a_phase_vocoder_backward": (
        ctypes.c_int,
        [c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_int64, c_double, c_void_p, c_void_p, c_int64, c_int64,
         c_int64, c_void_p, c_int64, c_void_p],
    ),
    "b200a_kaldi_num_frames": (c_int64, [c_int64, c_int32, c_int32, c_int32]),
    "b200a_kaldi_run": (
        ctypes.c_int,
        [POINTER(KaldiDesc), POINTER(FrontendDesc), c_void_p, c_int32, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_void_p],
    ),
    "b200a_kaldi_backward": (
        ctypes.c_int,
        [POINTER(KaldiDesc), POINTER(FrontendDesc), c_void_p, c_int32, c_void_p, c_int64, c_int64, c_int64, c_void_p,
         c_int64, c_int64, c_int64, c_void_p, c_void_p, c_int64, c_void_p],
    ),
    "b200a_kaldi_backward_scratch_bytes": (
        c_size_t, [POINTER(KaldiDesc), POINTER(FrontendDesc), c_int32, c_int64, c_int64]),
    "b200a_subtract_column_mean": (ctypes.c_int, [c_void_p, c_int64, c_int64, c_int64, c_void_p]),
    "b200a_fill_f32": (ctypes.c_int, [c_void_p, c_int64, c_float, c_void_p]),
    "b200a_ratio_f32": (ctypes.c_int, [c_void_p, c_int64, c_void_p, c_void_p]),
    "b200a_resample_workspace_bytes": (c_size_t, [c_int32, c_int32]),
    "b200a_resample_prepare": (ctypes.c_int, [c_void_p, c_int32, c_int32, c_int32, c_void_p, c_size_t, c_void_p]),
    "b200a_resample_run": (
        ctypes.c_int,
        [c_void_p, c_void_p, c_int32, c_int32, c_int32, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_int64, c_int64, c_void_p],
    ),
    "b200a_resample_backward_workspace_bytes": (c_size_t, [c_int32, c_int32, c_int32]),
    "b200a_resample_backward_prepare": (ctypes.c_int, [c_void_p, c_int32, c_int32, c_int32, c_void_p, c_size_t, c_void_p]),
    "b200a_resample_backward": (
        ctypes.c_int,
        [c_void_p, c_int32, c_int32, c_int32, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_int64, c_int64, c_void_p],
    ),
    "b200a_inverse_mel_plan_bytes": (c_size_t, [c_int32, c_int32]),
    "b200a_inverse_mel_plan": (
        ctypes.c_int, [c_void_p, c_int32, c_int32, c_int32, c_void_p, c_size_t, POINTER(c_int32), POINTER(c_int32)]),
    "b200a_inverse_mel_run": (
        ctypes.c_int,
        [c_void_p, c_int32, c_int32, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_void_p, c_void_p],
    ),
    "b200a_inverse_mel_backward": (
        ctypes.c_int,
        [c_void_p, c_int32, c_int32, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_void_p, c_int64, c_int64,
         c_int64, c_void_p, c_void_p],
    ),
    "b200a_lfilter_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int32, c_int32]),
    "b200a_lfilter_backward_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int32, c_int32]),
    "b200a_lfilter_run": (
        ctypes.c_int,
        [c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int32, c_int32, c_void_p,
         c_void_p, c_void_p, c_size_t, c_void_p],
    ),
    "b200a_lfilter_backward": (
        ctypes.c_int,
        [c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_int64, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_int32,
         c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p],
    ),
    "b200a_fftconvolve_workspace_bytes": (c_size_t, [POINTER(FftconvolveDesc)]),
    "b200a_fftconvolve_backward_workspace_bytes": (c_size_t, [POINTER(FftconvolveDesc)]),
    "b200a_fftconvolve_run": (
        ctypes.c_int,
        [POINTER(FftconvolveDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p],
    ),
    "b200a_fftconvolve_backward": (
        ctypes.c_int,
        [POINTER(FftconvolveDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p],
    ),
    "b200a_convolve_workspace_bytes": (c_size_t, [POINTER(FftconvolveDesc)]),
    "b200a_convolve_backward_workspace_bytes": (c_size_t, [POINTER(FftconvolveDesc)]),
    "b200a_convolve_run": (
        ctypes.c_int,
        [POINTER(FftconvolveDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p],
    ),
    "b200a_convolve_backward": (
        ctypes.c_int,
        [POINTER(FftconvolveDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p],
    ),
    "b200a_vad_workspace_bytes": (c_size_t, [POINTER(VadDesc), c_int64]),
    "b200a_vad_walk": (
        ctypes.c_int,
        [POINTER(VadDesc), c_int64, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p],
    ),
    "b200a_vad_trigger": (
        ctypes.c_int,
        [POINTER(VadDesc), c_int64, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p],
    ),
    "b200a_rnnt_loss_check": (
        ctypes.c_int, [c_int32, c_int32, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200a_rnnt_loss_workspace_bytes": (c_size_t, [POINTER(RnntLossDesc)]),
    "b200a_rnnt_loss_forward": (
        ctypes.c_int,
        [POINTER(RnntLossDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
         c_size_t, c_void_p],
    ),
    "b200a_rnnt_loss_backward": (
        ctypes.c_int,
        [POINTER(RnntLossDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64,
         c_void_p, c_void_p],
    ),
    "b200a_forced_align_check": (
        ctypes.c_int,
        [POINTER(ForcedAlignDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "b200a_forced_align_workspace_bytes": (c_size_t, [POINTER(ForcedAlignDesc)]),
    "b200a_forced_align_run": (
        ctypes.c_int,
        [POINTER(ForcedAlignDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t,
         c_void_p]),
    "b200a_ctc_decoder_workspace_bytes": (c_size_t, [POINTER(CtcDecoderDesc)]),
    "b200a_ctc_decoder_run": (
        ctypes.c_int,
        [POINTER(CtcDecoderDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t,
         c_void_p]),
    "b200a_mask_workspace_bytes": (c_size_t, [POINTER(MaskDesc)]),
    "b200a_mask_run": (
        ctypes.c_int, [POINTER(MaskDesc), POINTER(MaskSpec), c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "b200a_mask_backward": (
        ctypes.c_int, [POINTER(MaskDesc), POINTER(MaskSpec), c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)

_lib = None


class B200AudioError(RuntimeError):
    def __init__(self, status: int, where: str):
        self.status = status
        msg = lib().b200a_strerror(status).decode()
        super().__init__(f"libb200audio: {where}: {msg} (status {status})")


def lib() -> ctypes.CDLL:
    """Load (once) and return the shared library; raises if it is not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing. Build it with `python -m audio_b200._build` "
                "(nvcc, sm_90a). audio_b200 has no CPU or ATen fallback."
            )
        handle = ctypes.CDLL(LIB_PATH)
        for name, (restype, argtypes) in _SIGNATURES.items():
            fn = getattr(handle, name)  # AttributeError here == header/library mismatch
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = handle
    return _lib


def check(status: int, where: str) -> None:
    if status != OK:
        raise B200AudioError(status, where)
