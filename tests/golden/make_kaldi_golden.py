#!/usr/bin/env python
"""Generate the committed Kaldi fixtures under tests/golden/ (needs a pytorch/audio checkout named by AUDIO_REFERENCE; run once):

    python tests/golden/make_kaldi_golden.py

1. ``kaldi_goldens.npz`` -- the outputs of the Kaldi binaries (compute-{fbank,mfcc,spectrogram}-feats) that the
   reference's own tests hold under test/torchaudio_unittest/assets/kaldi_expected_results and compare with at
   rtol 1e-4 (compliance/kaldi/kaldi_compatibility_impl.py:20-48), the option sets they were produced with
   (assets/kaldi_test_{fbank,mfcc,spectrogram}_args.jsonl, kept as JSON strings) and the 20-sample input
   (assets/kaldi_file.wav, read un-normalised as load_wav(normalize=False) does).
2. ``kaldi_ref_cases.npz`` -- outputs of the reference itself (the reference's src/, CPU, float32) on seeded
   signals of realistic length, for option sets the tiny Kaldi cases do not reach (25 ms frames at 16 kHz =
   512-point FFT, 80 mel bins, snip_edges on/off, energy, HTK order, mean subtraction), plus the reference's
   constant tables (windows, mel banks, DCT, lifter) for the bit-identity checks of the host code.
"""
import glob
import json
import os
import re
import sys
import wave

import numpy as np
import torch

REF = os.environ["AUDIO_REFERENCE"]  # a pytorch/audio checkout at the pinned version
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(REF, "src"))
import torchaudio  # noqa: E402
import torchaudio.compliance.kaldi as K  # noqa: E402

assert torchaudio.__file__.startswith(REF), torchaudio.__file__
ASSETS = os.path.join(REF, "test/torchaudio_unittest/assets")
RESULTS = os.path.join(ASSETS, "kaldi_expected_results/test/torchaudio_unittest/compliance/kaldi")


def read_wav(path):
    with wave.open(path) as w:
        assert w.getsampwidth() == 2
        data = np.frombuffer(w.readframes(w.getnframes()), dtype="<i2").reshape(-1, w.getnchannels())
    return data.T.astype(np.float32)  # (channels, samples), un-normalised


def kaldi_goldens():
    out = {"wave": read_wav(os.path.join(ASSETS, "kaldi_file.wav"))}
    for kind in ("fbank", "mfcc", "spectrogram"):
        with open(os.path.join(ASSETS, f"kaldi_test_{kind}_args.jsonl")) as fh:
            args = [line.strip() for line in fh if line.strip()]
        files = glob.glob(os.path.join(RESULTS, f"kaldi_compatibility_test.py__TestKaldiFloat32__test_{kind}_*.pt"))
        files.sort(key=lambda f: int(re.search(r"_(\d+)\.pt$", f).group(1)))
        assert len(files) == len(args), (kind, len(files), len(args))
        out[f"{kind}_args"] = np.array(args)
        for i, f in enumerate(files):
            out[f"{kind}_{i}"] = torch.load(f).numpy().astype(np.float32)
    np.savez_compressed(os.path.join(HERE, "kaldi_goldens.npz"), **out)
    print("kaldi_goldens.npz:", {k: len(out[f"{k}_args"]) for k in ("fbank", "mfcc", "spectrogram")})


REF_CASES = {
    "fbank": [
        dict(),
        dict(num_mel_bins=80, dither=0.0),
        dict(num_mel_bins=40, snip_edges=False, use_energy=True),
        dict(num_mel_bins=40, use_energy=True, htk_compat=True, raw_energy=False, subtract_mean=True),
        dict(num_mel_bins=64, frame_length=20.0, frame_shift=8.0, window_type="hamming", use_power=False,
             remove_dc_offset=False, preemphasis_coefficient=0.0, round_to_power_of_two=False),
        dict(num_mel_bins=30, sample_frequency=8000.0, low_freq=60.0, high_freq=-200.0, vtln_warp=1.1, vtln_low=200.0,
             vtln_high=-600.0, use_log_fbank=False, window_type="blackman", energy_floor=0.0),
    ],
    "mfcc": [
        dict(),
        dict(num_ceps=20, num_mel_bins=40, use_energy=True),
        dict(htk_compat=True, cepstral_lifter=0.0, snip_edges=False),
        dict(htk_compat=True, use_energy=True, subtract_mean=True, window_type="hanning"),
    ],
    "spectrogram": [
        dict(),
        dict(snip_edges=False, raw_energy=False, subtract_mean=True, window_type="rectangular"),
        dict(frame_length=10.0, frame_shift=5.0, round_to_power_of_two=False, energy_floor=0.0, remove_dc_offset=False),
    ],
}


def ref_cases():
    g = torch.Generator().manual_seed(2024)
    # int16-scale speech-like input: noise with a slow envelope and a DC offset, two channels
    n = 19999
    env = 0.3 + 0.7 * torch.sin(torch.linspace(0, 9.0, n)) ** 2
    x = (torch.randn(2, n, generator=g) * 3000.0 * env + 150.0).round()
    out = {"wave": x.numpy().astype(np.float32)}
    for kind, cases in REF_CASES.items():
        out[f"{kind}_args"] = np.array([json.dumps(c) for c in cases])
        for i, kw in enumerate(cases):
            y = getattr(K, kind)(x[:1], **kw)
            out[f"{kind}_{i}"] = y.numpy().astype(np.float32)
    y = K.fbank(x, channel=1, num_mel_bins=23)
    out["fbank_channel1"] = y.numpy()
    # constant tables for bit-identity checks
    for wt in K.WINDOWS:
        out[f"window_{wt}"] = K._feature_window_function(wt, 400, 0.42, torch.device("cpu"), torch.float32).numpy()
    banks, centers = K.get_mel_banks(23, 512, 16000.0, 20.0, 0.0, 100.0, -500.0, 1.0)
    out["banks_23_512"], out["centers_23_512"] = banks.numpy(), centers.numpy()
    banks, centers = K.get_mel_banks(30, 256, 8000.0, 60.0, -200.0, 200.0, -600.0, 1.1)
    out["banks_vtln"], out["centers_vtln"] = banks.numpy(), centers.numpy()
    out["dct_13_23"] = K._get_dct_matrix(13, 23).numpy()
    out["lifter_13"] = K._get_lifter_coeffs(13, 22.0).numpy()
    np.savez_compressed(os.path.join(HERE, "kaldi_ref_cases.npz"), **out)
    print("kaldi_ref_cases.npz:", {k: len(v) for k, v in REF_CASES.items()})


if __name__ == "__main__":
    kaldi_goldens()
    ref_cases()
