"""Parameter tables shared by the CPU (oracle) and GPU (product) golden tests.

They restate the parameterisations of the reference's own tests:
transforms/librosa_compatibility_test_impl.py:17-134 and
functional/librosa_compatibility_test_impl.py:56-94 (paths under
pytorch/audio/test/torchaudio_unittest).
"""
import itertools

# test_Spectrogram (impl.py:17-44): whitenoise input, atol=rtol=1e-4
SPECTROGRAM = [
    dict(n_fft=400, hop_length=200, power=2.0),
    dict(n_fft=600, hop_length=100, power=2.0),
    dict(n_fft=400, hop_length=200, power=3.0),
    dict(n_fft=200, hop_length=50, power=2.0),
]

# test_MelSpectrogram (impl.py:64-100): sinusoid input, atol=5e-4 rtol=1e-5;
# nested_params order = product(configs, norm, mel_scale)
MELSPECTROGRAM = [
    dict(cfg, norm=norm, mel_scale=ms)
    for cfg, norm, ms in itertools.product(
        [dict(n_fft=400, hop_length=200, n_mels=64), dict(n_fft=600, hop_length=100, n_mels=128), dict(n_fft=200, hop_length=50, n_mels=32)],
        [None, "slaney"],
        ["htk", "slaney"],
    )
]

# test_mfcc (impl.py:114-134): whitenoise input, atol=5e-4 rtol=1e-5
MFCC = [
    dict(n_fft=400, hop_length=200, n_mels=64, n_mfcc=40),
    dict(n_fft=600, hop_length=100, n_mels=128, n_mfcc=20),
    dict(n_fft=200, hop_length=50, n_mels=32, n_mfcc=25),
]

# test_create_mel_fb (functional impl.py:56-94): atol=7e-5 rtol=1.3e-6
_FB_DEFAULT = dict(n_mels=40, sample_rate=22050, n_fft=2048, fmin=0.0, fmax=8000.0)
MEL_FB = [
    dict(_FB_DEFAULT, **cfg, norm=norm, mel_scale=ms)
    for cfg, norm, ms in itertools.product(
        [
            dict(),
            dict(n_mels=128, sample_rate=44100),
            dict(n_mels=128, fmin=2000.0, fmax=5000.0),
            dict(n_mels=56, fmin=100.0, fmax=9000.0),
            dict(n_mels=56, fmin=800.0, fmax=900.0),
            dict(n_mels=56, fmin=1900.0, fmax=900.0),
            dict(n_mels=10, fmin=1900.0, fmax=900.0),
        ],
        [None, "slaney"],
        ["htk", "slaney"],
    )
]

# Spectrogram option variants stored in ref_cases.npz (see tests/golden/make_golden.py)
SPEC_VARIANTS = {
    "default400": dict(),
    "n512_h128": dict(n_fft=512, hop_length=128),
    "n1024_h256": dict(n_fft=1024, hop_length=256),
    "n256_h64_p1": dict(n_fft=256, hop_length=64, power=1.0),
    "n2048_h512": dict(n_fft=2048, hop_length=512),
    "n400_win300": dict(n_fft=400, win_length=300, hop_length=100),
    "n512_win400_h160": dict(n_fft=512, win_length=400, hop_length=160),
    "n400_p3": dict(n_fft=400, hop_length=200, power=3.0),
    "n400_normwin": dict(n_fft=400, normalized=True),
    "n400_normfl": dict(n_fft=400, normalized="frame_length"),
    "n512_nocenter": dict(n_fft=512, hop_length=100, center=False),
    "n512_pad37": dict(n_fft=512, hop_length=128, pad=37),
    "n512_constant": dict(n_fft=512, hop_length=128, pad_mode="constant"),
    "n512_replicate": dict(n_fft=512, hop_length=128, pad_mode="replicate"),
    "n512_circular": dict(n_fft=512, hop_length=128, pad_mode="circular"),
    "n512_twosided": dict(n_fft=512, hop_length=128, onesided=False),
    "n600_h100": dict(n_fft=600, hop_length=100),
    "n200_h50": dict(n_fft=200, hop_length=50),
    "n77_h13": dict(n_fft=77, hop_length=13),
    "n1024_hamming": dict(n_fft=1024, hop_length=256, window="hamming"),
}

# Resample cases stored in ref_cases.npz: key -> (input slice, ctor kwargs)
RESAMPLE = {
    "rs_kaiser_out": (None, dict(orig_freq=44100, new_freq=16000, resampling_method="sinc_interp_kaiser")),
    "rs_hann_out": (None, dict(orig_freq=44100, new_freq=16000)),
    "rs_16k_8k": (None, dict(orig_freq=16000, new_freq=8000)),
    "rs_8k_16k": (None, dict(orig_freq=8000, new_freq=16000)),
    "rs_48k_44k1": (2400, dict(orig_freq=48000, new_freq=44100)),
    "rs_16k_44k1": (1000, dict(orig_freq=16000, new_freq=44100, resampling_method="sinc_interp_kaiser")),
    "rs_lpw16": (None, dict(orig_freq=16000, new_freq=12000, lowpass_filter_width=16, rolloff=0.9)),
    "rs_short": (7, dict(orig_freq=44100, new_freq=16000)),
}

# librosa_transforms.npz keeps every second frame of each expected output (tests/golden/make_golden.py); the tests
# compare the same frames of what they compute
LIBROSA_FRAMES = slice(None, None, 2)
