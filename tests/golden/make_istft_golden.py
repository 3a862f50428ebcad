#!/usr/bin/env python
"""Generate tests/golden/istft_ref_cases.npz: outputs of the reference's F.inverse_spectrogram (over torch.istft, CPU,
float32) on generic complex spectrograms (a forward STFT of noise, perturbed so that it is NOT a consistent STFT),
with the inputs stored next to them.  Needs a pytorch/audio checkout named by AUDIO_REFERENCE; run once:

    python tests/golden/make_istft_golden.py
"""
import json
import os
import sys

import numpy as np
import torch

REF = os.environ["AUDIO_REFERENCE"]  # a pytorch/audio checkout at the pinned version
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(REF, "src"))
import torchaudio  # noqa: E402
import torchaudio.functional as F  # noqa: E402

assert torchaudio.__file__.startswith(REF), torchaudio.__file__

CASES = [
    dict(n_fft=512, hop=128, win=512, normalized=False, center=True, length=None, pad=0),
    dict(n_fft=400, hop=200, win=400, normalized=True, center=True, length=7900, pad=0),
    dict(n_fft=1024, hop=256, win=800, normalized="frame_length", center=True, length=7500, pad=30),
    dict(n_fft=256, hop=64, win=256, normalized=False, center=False, length=None, pad=0),
    dict(n_fft=100, hop=25, win=100, normalized="window", center=True, length=5100, pad=0),
    dict(n_fft=512, hop=256, win=512, normalized=False, center=True, length=8400, pad=0),  # longer than covered: zero tail
]


def main():
    g = torch.Generator().manual_seed(77)
    out = {"cases": np.array([json.dumps(c) for c in CASES])}
    for i, c in enumerate(CASES):
        x = torch.randn(1, 8000, generator=g)  # one row: rows are independent, and the file stays under 1 MB
        window = torch.hann_window(c["win"]) if c["center"] else torch.hamming_window(c["win"])
        spec = F.spectrogram(x, c["pad"], window, c["n_fft"], c["hop"], c["win"], None, c["normalized"], c["center"])
        spec = spec * (1 + 0.1 * torch.randn(spec.shape, generator=g))
        y = F.inverse_spectrogram(spec, c["length"], c["pad"], window, c["n_fft"], c["hop"], c["win"], c["normalized"],
                                  c["center"])
        out[f"spec_{i}"], out[f"window_{i}"], out[f"out_{i}"] = spec.numpy(), window.numpy(), y.numpy()
        print(i, tuple(spec.shape), "->", tuple(y.shape))
    np.savez_compressed(os.path.join(HERE, "istft_ref_cases.npz"), **out)


def griffinlim_goldens():
    """The two librosa.griffinlim outputs the reference's test holds (functional/librosa_compatibility_test_impl.py:16-54,
    float64, n_fft 400 / hop 100 / power 1 / 8 iterations, momentum 0 and 0.99, atol 5e-5) with the magnitude
    spectrogram they were computed from (get_whitenoise -> get_spectrogram, common_utils/data_utils.py)."""
    import importlib.util

    spec_ = importlib.util.spec_from_file_location(
        "ref_data_utils", os.path.join(REF, "test/torchaudio_unittest/common_utils/data_utils.py"))
    du = importlib.util.module_from_spec(spec_)
    spec_.loader.exec_module(du)
    assets = os.path.join(REF, "test/torchaudio_unittest/assets/librosa_expected_results/test/torchaudio_unittest/functional")
    wave = du.get_whitenoise(dtype=torch.float64)
    window = torch.hann_window(400)
    specgram = du.get_spectrogram(wave, n_fft=400, hop_length=100, power=1, win_length=400, window=window)
    out = {"waveform": wave.numpy(), "specgram": specgram.numpy()}
    for tag in ("0", "0_99"):
        t = torch.load(os.path.join(assets, f"librosa_compatibility_test.py__TestFunctionalCPU__test_griffinlim_{tag}.pt"),
                       weights_only=False)
        out[f"librosa_{tag}"] = np.asarray(t)
        res = F.griffinlim(specgram, window=window.double(), n_fft=400, hop_length=100, win_length=400, power=1, n_iter=8,
                           momentum=float(tag.replace("_", ".")), length=wave.size(1), rand_init=False)
        out[f"ref_{tag}"] = res.numpy()
    # a float32 run of the reference with the module defaults (power 2, 32 iterations, momentum 0.99)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 6000, generator=g)
    w = torch.hann_window(512)
    p2 = F.spectrogram(x, 0, w, 512, 128, 512, 2.0, False)
    out["power_spec_512"] = p2.numpy()
    out["ref_512"] = F.griffinlim(p2, w, 512, 128, 512, 2.0, 32, 0.99, 6000, False).numpy()
    np.savez_compressed(os.path.join(HERE, "griffinlim_goldens.npz"), **out)
    print("griffinlim_goldens.npz", {k: v.shape for k, v in out.items()})


def vocoder_goldens():
    """Reference outputs (CPU float32) of F.phase_vocoder and F.pitch_shift."""
    import math

    g = torch.Generator().manual_seed(11)
    x = torch.randn(2, 6000, generator=g)
    w = torch.hann_window(512)
    spec = F.spectrogram(x, 0, w, 512, 128, 512, None, False)
    pa = torch.linspace(0, math.pi * 128, 257)[..., None]
    out = {"wave": x.numpy(), "spec": spec.numpy()}
    for rate in (0.8, 1.3, 2.0):
        out[f"pv_{rate}"] = F.phase_vocoder(spec, rate, pa).numpy()
    for tag, (sr, steps) in {"up12": (16000, 12), "down12": (16000, -12), "up7_1k": (1000, 7), "down5_1k": (1000, -5)}.items():
        out[f"ps_{tag}"] = F.pitch_shift(x, sr, steps).numpy()
    np.savez_compressed(os.path.join(HERE, "vocoder_ref_cases.npz"), **out)
    print("vocoder_ref_cases.npz", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
    griffinlim_goldens()
    vocoder_goldens()
