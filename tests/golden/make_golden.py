#!/usr/bin/env python
"""Generate the committed golden fixtures under tests/golden/.

Run ONCE (needs a pytorch/audio checkout named by AUDIO_REFERENCE, which does not exist on the
GPU box):   python tests/golden/make_golden.py

Two kinds of fixture are written:

1. ``librosa_*.npz`` -- the golden vectors the reference's own test-suite pins the
   hot path with (test/torchaudio_unittest/assets/librosa_expected_results/...,
   consumed by transforms/librosa_compatibility_test_impl.py:17-134 and
   functional/librosa_compatibility_test_impl.py:56-94), converted from torch-pickled
   float64 numpy arrays to float32 npz so they are small and load without torch.
   The matching *inputs* are regenerated with the reference's own generators
   (common_utils/data_utils.py:37-118 -- get_whitenoise / get_sinusoid) and stored too.

2. ``ref_*.npz`` -- outputs of the reference itself (imported from
   the reference's src/, CPU, float32) on seeded inputs stored next to them.  These
   pin the paths no librosa golden covers (resample values, STFT option variants,
   MFCC batch coupling) and the integer bookkeeping.
"""
import importlib.util
import itertools
import math
import os
import sys

import numpy as np
import torch

REF = os.environ["AUDIO_REFERENCE"]  # a pytorch/audio checkout at the pinned version
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(REF, "src"))
import torchaudio  # noqa: E402  (the reference, pure python on this path)
import torchaudio.functional as F  # noqa: E402
import torchaudio.transforms as T  # noqa: E402
from torchaudio.functional import functional as FF  # noqa: E402  (private kernel builders)

assert torchaudio.__file__.startswith(REF), torchaudio.__file__

spec = importlib.util.spec_from_file_location(
    "ref_data_utils", os.path.join(REF, "test/torchaudio_unittest/common_utils/data_utils.py")
)
data_utils = importlib.util.module_from_spec(spec)
spec.loader.exec_module(data_utils)

ASSETS = os.path.join(REF, "test/torchaudio_unittest/assets/librosa_expected_results/test/torchaudio_unittest")


def load_pt(sub, name):
    return torch.load(os.path.join(ASSETS, sub, name), weights_only=False)


def save(name, **arrays):
    path = os.path.join(HERE, name)
    np.savez_compressed(path, **arrays)
    print(f"{name}: {os.path.getsize(path) / 1024:.0f} KiB, keys={len(arrays)}")


def f32(a):
    return np.ascontiguousarray(np.asarray(a), dtype=np.float32)


LIBROSA_FRAMES = slice(None, None, 2)


def librosa_goldens():
    noise = data_utils.get_whitenoise(sample_rate=16000, n_channels=1)  # (1,16000) fp32, seed 0
    sine = data_utils.get_sinusoid(sample_rate=16000, n_channels=1)
    out = {"whitenoise": f32(noise), "sinusoid": f32(sine)}
    tr = "transforms"
    # the expected outputs keep every second frame (LIBROSA_FRAMES) so that the file stays under 1 MB; the tests
    # compare the same frames of what they compute
    pre = "librosa_compatibility_test.py__TestTransforms__test_"
    for i in range(4):
        out[f"spectrogram_{i}"] = f32(load_pt(tr, f"{pre}Spectrogram_{i}.pt")[0])
    out["spectrogram_complex"] = f32(load_pt(tr, f"{pre}Spectrogram_complex.pt")[0])
    for i in range(12):
        out[f"melspectrogram_{i:02d}"] = f32(load_pt(tr, f"{pre}MelSpectrogram_{i:02d}.pt"))
    for i in range(3):
        out[f"mfcc_{i}"] = f32(load_pt(tr, f"{pre}mfcc_{i}.pt"))
    out["power_to_db"] = f32(load_pt(tr, f"{pre}power_to_db.pt"))
    out["magnitude_to_db"] = f32(load_pt(tr, f"{pre}magnitude_to_db.pt"))
    for i in range(3):  # test_spectral_centroid (impl.py:136-158): n_fft/hop = 400/200, 600/100, 200/50
        out[f"spectral_centroid_{i}"] = f32(load_pt(tr, f"{pre}spectral_centroid_{i}.pt"))
    for k in list(out):
        if k not in ("whitenoise", "sinusoid"):
            out[k] = np.ascontiguousarray(out[k][..., LIBROSA_FRAMES])
    save("librosa_transforms.npz", **out)

    fb = {}
    pre = "librosa_compatibility_test.py__TestFunctionalCPU__test_create_mel_fb_"
    for i in range(28):
        # librosa returns (n_mels, n_freqs); the reference test transposes (impl.py:84)
        fb[f"fb_{i:02d}"] = np.asarray(load_pt("functional", f"{pre}{i:02d}.pt"), dtype=np.float64).T.copy()
    save("librosa_melfb.npz", **fb)


def seeded(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g) * scale


def reference_cases():
    out = {}
    with torch.inference_mode():
        # ---- BASELINE config 1: Spectrogram n_fft=512 hop=256 on 1x16000 --------------
        x = seeded((1, 16000), 11).clamp(-1, 1) * 0.5
        out["c1_in"] = f32(x)
        out["c1_out"] = f32(T.Spectrogram(n_fft=512, hop_length=256)(x))

        # ---- Spectrogram option variants (each key documents its kwargs) -------------
        x = seeded((1, 1600), 12)
        out["spec_in"] = f32(x)
        variants = {
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
            "n1024_hamming": dict(n_fft=1024, hop_length=256, window_fn=torch.hamming_window),
        }
        for k, kw in variants.items():
            out[f"spec_{k}"] = f32(T.Spectrogram(**kw)(x))
        c = T.Spectrogram(n_fft=400, hop_length=200, power=None)(x)
        out["spec_complex400"] = np.ascontiguousarray(torch.view_as_real(c).numpy(), dtype=np.float32)
        c = T.Spectrogram(n_fft=1024, hop_length=256, power=None)(x)
        out["spec_complex1024"] = np.ascontiguousarray(torch.view_as_real(c).numpy(), dtype=np.float32)

        # ---- MelSpectrogram: BASELINE config-2 parameters at a small batch ------------
        x = seeded((4, 2000), 13)
        out["mel_in"] = f32(x)
        m = T.MelSpectrogram(16000, n_fft=1024, hop_length=256, n_mels=80)
        out["mel_c2_out"] = f32(m(x))
        out["mel_c2_fb"] = f32(m.mel_scale.fb)
        out["mel_c2_window"] = f32(m.spectrogram.window)
        m = T.MelSpectrogram(16000)  # all defaults: n_fft=400 n_mels=128
        out["mel_default_out"] = f32(m(x))
        m = T.MelSpectrogram(16000, n_fft=400, hop_length=160, n_mels=80)  # rnnt_pipeline.py:316-343
        out["mel_rnnt_out"] = f32(m(x))
        m = T.MelSpectrogram(22050, n_fft=2048, hop_length=512, n_mels=128, norm="slaney", mel_scale="slaney", f_max=8000.0)
        out["mel_slaney2048_out"] = f32(m(x))
        out["mel_slaney2048_fb"] = f32(m.mel_scale.fb)
        m = T.MelSpectrogram(16000, n_fft=512, hop_length=128, n_mels=40, power=1.0)
        out["mel_512_p1_out"] = f32(m(x))
        m = T.MelSpectrogram(16000, n_fft=256, hop_length=64, n_mels=80)  # 2 all-zero filters (warns)
        out["mel_256_out"] = f32(m(x))
        # loud / quiet / silent rows
        xs = x.clone()
        xs[0] *= 1000.0
        xs[1] *= 1e-3
        xs[2] = 0.0
        out["mel_scaled_in"] = f32(xs)
        out["mel_scaled_out"] = f32(T.MelSpectrogram(16000, n_fft=1024, hop_length=256, n_mels=80)(xs))

        # ---- MFCC: 2-D input (one global top_db) and 3-D input (per item) -------------
        mf = T.MFCC(16000, n_mfcc=40, melkwargs=dict(n_fft=1024, hop_length=256, n_mels=80))
        out["mfcc_dct"] = f32(mf.dct_mat)
        out["mfcc_2d_out"] = f32(mf(xs))  # (4, 40, 8) -- batch-coupled clamp
        out["mfcc_3d_out"] = f32(mf(xs[:, None, :]))  # (4, 1, 40, 8) -- per item
        out["mfcc_1d_out"] = f32(mf(xs[0]))
        out["mfcc_x_out"] = f32(mf(x))
        mfl = T.MFCC(16000, n_mfcc=13, log_mels=True, melkwargs=dict(n_fft=400, hop_length=160, n_mels=23))
        out["mfcc_log_out"] = f32(mfl(x))
        mfn = T.MFCC(16000, n_mfcc=20, norm=None, melkwargs=dict(n_fft=512, hop_length=256, n_mels=64))
        out["mfcc_nonorm_out"] = f32(mfn(x))
        out["mfcc_default_out"] = f32(T.MFCC()(x))

        # ---- LFCC / SpectralCentroid (SURVEY 8f.2: same kernels, other filter matrix / epilogue) ----
        lf = T.LFCC(16000, n_filter=64, n_lfcc=20, speckwargs=dict(n_fft=512, hop_length=128))
        out["lfcc_filter_mat"] = f32(lf.filter_mat)
        out["lfcc_512_out"] = f32(lf(x))
        out["lfcc_default_out"] = f32(T.LFCC()(x[:, None]))
        out["lfcc_log_out"] = f32(T.LFCC(16000, n_filter=40, n_lfcc=13, log_lf=True, speckwargs=dict(n_fft=1024, hop_length=256))(x))
        out["centroid_1024_out"] = f32(T.SpectralCentroid(16000, n_fft=1024, hop_length=256)(x))
        out["centroid_default_out"] = f32(T.SpectralCentroid(16000)(x))

        # ---- AmplitudeToDB stand-alone -------------------------------------------------
        p = T.Spectrogram(n_fft=400)(xs)  # (4, 201, 11)
        out["db_in"] = f32(p)
        out["db_power_top80_3d"] = f32(T.AmplitudeToDB("power", 80.0)(p))
        out["db_power_top80_4d"] = f32(T.AmplitudeToDB("power", 80.0)(p[:, None]))
        out["db_mag_none"] = f32(T.AmplitudeToDB("magnitude")(p))

        # ---- Resample (config 3 parameters, short signals) ------------------------------
        x = seeded((1, 4410), 14)
        out["rs_in"] = f32(x)
        r = T.Resample(44100, 16000, resampling_method="sinc_interp_kaiser")
        out["rs_kaiser_kernel"] = f32(r.kernel)
        out["rs_kaiser_out"] = f32(r(x))
        r = T.Resample(44100, 16000)
        out["rs_hann_kernel"] = f32(r.kernel)
        out["rs_hann_out"] = f32(r(x))
        out["rs_16k_8k"] = f32(T.Resample(16000, 8000)(x))
        out["rs_8k_16k"] = f32(T.Resample(8000, 16000)(x))
        out["rs_48k_44k1"] = f32(T.Resample(48000, 44100)(x[:, :2400]))
        out["rs_16k_44k1"] = f32(T.Resample(16000, 44100, resampling_method="sinc_interp_kaiser")(x[:, :1000]))
        out["rs_lpw16"] = f32(T.Resample(16000, 12000, lowpass_filter_width=16, rolloff=0.9)(x))
        out["rs_short"] = f32(T.Resample(44100, 16000)(x[:, :7]))
        out["rs_func_kaiser"] = f32(F.resample(x, 44100, 16000, resampling_method="sinc_interp_kaiser"))
        out["rs_func_hann_3_2"] = f32(F.resample(x, 3, 2))
    save("ref_cases.npz", **out)


def integer_cases():
    rows = []
    for L, n_fft, hop, center, pad in itertools.product(
        [1, 7, 255, 256, 257, 1000, 16000, 160000], [16, 77, 256, 400, 1024], [1, 13, 160, 256], [0, 1], [0, 5]
    ):
        x = torch.zeros(1, L)
        try:
            t = torch.stft(
                torch.nn.functional.pad(x, (pad, pad)),
                n_fft,
                hop,
                window=torch.ones(n_fft),
                center=bool(center),
                pad_mode="constant",
                return_complex=True,
            ).shape[-1]
        except RuntimeError:
            t = -1
        rows.append((L, n_fft, hop, center, pad, t))
    frames = np.asarray(rows, dtype=np.int64)

    rows = []
    for (o, n), L in itertools.product(
        [(44100, 16000), (16000, 44100), (16000, 8000), (8000, 16000), (48000, 44100), (3, 2), (2, 3), (16000, 16001), (7, 5)],
        [1, 2, 7, 100, 441, 442, 4410, 22050, 220500, 160000],
    ):
        g = math.gcd(o, n)
        k, w = FF._get_sinc_resample_kernel(o, n, g)
        y = FF._apply_sinc_resample_kernel(torch.zeros(1, L), o, n, g, k, w)
        rows.append((o, n, L, w, k.shape[-1], y.shape[-1]))
    rs = np.asarray(rows, dtype=np.int64)
    save("ref_integers.npz", stft_frames=frames, resample=rs)


if __name__ == "__main__":
    torch.set_num_threads(1)  # run-to-run deterministic reductions
    librosa_goldens()
    reference_cases()
    integer_cases()
