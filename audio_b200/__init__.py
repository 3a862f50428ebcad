"""audio_b200 -- H100-native (sm_90a) implementation of torchaudio's DSP front-end hot path.

    import audio_b200.transforms as T          # Spectrogram, MelSpectrogram, MFCC, LFCC, Resample, InverseSpectrogram,
                                               # GriffinLim, TimeStretch, PitchShift, Speed, ...
    import audio_b200.functional as F          # spectrogram, resample, melscale_fbanks, griffinlim, phase_vocoder,
                                               # lfilter, filtfilt, the *_biquad filters, deemphasis,
                                               # fftconvolve, convolve, ...
    import audio_b200.compliance.kaldi as K    # spectrogram, fbank, mfcc (Kaldi-compatible)

Everything computes in hand-written CUDA kernels reached through the C ABI of
``audio_b200/lib/libb200audio.so`` (``include/b200audio.h``).  There is no CPU fallback and no
dispatch to ``aten::stft`` / cuFFT / cuBLAS / cuDNN.
"""
from . import _lib  # noqa: F401  (does not load the .so until first use)
from . import compliance, functional, models, transforms  # noqa: F401
from ._plans import (differentiable, is_differentiable, is_feature_differentiable,  # noqa: F401
                     is_filtering_differentiable, is_inverse_differentiable, is_kaldi_differentiable,
                     is_resample_differentiable, is_vocoder_differentiable, set_differentiable)

__version__ = "0.1.0"


def library_path() -> str:
    return _lib.LIB_PATH
