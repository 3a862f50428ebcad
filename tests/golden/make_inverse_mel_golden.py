#!/usr/bin/env python
"""Generate tests/golden/inverse_mel_ref_cases.npz, the InverseMelScale fixture (needs a pytorch/audio checkout named by
AUDIO_REFERENCE; run once):

    python tests/golden/make_inverse_mel_golden.py

It holds, all float32 from the reference on the CPU, for each configuration ``c`` of ``CONFIGS``:
- ``{c}_fb``: the reference module's ``fb`` buffer;
- ``{c}_speech_in`` / ``{c}_speech_out``: MelSpectrogram(power=1) of a seeded speech-like signal, (2, n_mels, T), and
  InverseMelScale of it;
- ``{c}_rand_in`` / ``{c}_rand_out``: a seeded random positive (2, n_mels, 5) input and its InverseMelScale;
- ``{c}_grad_in`` / ``{c}_grad_up`` / ``{c}_grad``: an input redrawn until no float64 minimum-norm solution element lies
  within 1e-4 rms of zero outside the empty bins (the relu mask is unambiguous), a seeded upstream gradient and the reference's autograd input
  gradient;
and for the two rank-deficient banks of ``SINGULAR``, ``{s}_{driver}``: what the reference raises for each driver
(``"<exception type>: <message>"``, or ``"ok"`` when it returns).
"""
import os
import sys

import numpy as np
import torch

REF = os.environ["AUDIO_REFERENCE"]  # a pytorch/audio checkout at the pinned version
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(REF, "src"))
import torchaudio  # noqa: E402
import torchaudio.transforms as RT  # noqa: E402

assert torchaudio.__file__.startswith(REF), torchaudio.__file__

# name: (n_stft, n_mels, sample_rate, f_min, f_max, norm, mel_scale)
CONFIGS = {
    "c201_64_8k": (201, 64, 8000, 0.0, None, None, "htk"),
    "c513_128_16k": (513, 128, 16000, 0.0, None, None, "htk"),
    "c513_80_16k": (513, 80, 16000, 0.0, None, None, "htk"),
    "c1025_128_22k_slaney": (1025, 128, 22050, 0.0, None, "slaney", "slaney"),
    "c257_40_16k_band": (257, 40, 16000, 20.0, 7600.0, None, "htk"),
    "c201_40_16k": (201, 40, 16000, 0.0, None, None, "htk"),
}
SINGULAR = {"s201_128_16k": (201, 128, 16000), "s65_128_16k": (65, 128, 16000)}
DRIVERS = ("gels", "gelsy", "gelsd", "gelss")


def speech_like(n, sr, g):
    """Two harmonic stacks with a slow vibrato plus a little noise."""
    t = torch.arange(n, dtype=torch.float64) / sr
    x = torch.zeros(n, dtype=torch.float64)
    for f0, amp in ((140.0, 0.5), (215.0, 0.3)):
        phase = 2 * np.pi * f0 * t + 3.0 * torch.sin(2 * np.pi * 4.0 * t)
        for h in range(1, 12):
            x += amp / h * torch.sin(h * phase)
    x += 0.01 * torch.randn(n, generator=g, dtype=torch.float64)
    return x.to(torch.float32)


def min_norm(fb, m):
    fb = fb.double()
    return fb @ torch.linalg.solve(fb.T @ fb, m.double())


def main():
    out = {}
    g = torch.Generator().manual_seed(20261016)
    for name, (n_stft, n_mels, sr, f_min, f_max, norm, scale) in CONFIGS.items():
        n_fft = 2 * (n_stft - 1)
        mod = RT.InverseMelScale(n_stft, n_mels, sr, f_min, f_max, norm, scale)
        out[f"{name}_fb"] = mod.fb.numpy()
        spec = RT.MelSpectrogram(sr, n_fft=n_fft, hop_length=n_fft // 2, f_min=f_min, f_max=f_max, n_mels=n_mels,
                                 power=1.0, norm=norm, mel_scale=scale)
        wave = torch.stack([speech_like(3 * n_fft, sr, g), 0.1 * speech_like(3 * n_fft, sr, g)])
        with torch.no_grad():
            mel = spec(wave).contiguous()
            out[f"{name}_speech_in"], out[f"{name}_speech_out"] = mel.numpy(), mod(mel).numpy()
            r = torch.rand(2, n_mels, 5, generator=g)
            out[f"{name}_rand_in"], out[f"{name}_rand_out"] = r.numpy(), mod(r).numpy()
        live = mod.fb.abs().sum(1) > 0  # empty bins are exactly 0 in every solution
        for _ in range(1000):
            m = torch.rand(2, n_mels, 4, generator=g)
            x = min_norm(mod.fb, m)[:, live]
            if x.abs().min() > 1e-4 * x.pow(2).mean().sqrt():
                break
        else:
            raise RuntimeError(f"{name}: no input with an unambiguous relu mask")
        up = torch.randn(2, n_stft, 4, generator=g)
        m.requires_grad_()
        mod(m).backward(up)
        out[f"{name}_grad_in"], out[f"{name}_grad_up"], out[f"{name}_grad"] = m.detach().numpy(), up.numpy(), m.grad.numpy()
    for name, (n_stft, n_mels, sr) in SINGULAR.items():
        m = torch.rand(1, n_mels, 3, generator=g)
        for drv in DRIVERS:
            try:
                RT.InverseMelScale(n_stft, n_mels, sr, driver=drv)(m)
                out[f"{name}_{drv}"] = np.array("ok")
            except Exception as e:  # noqa: BLE001
                out[f"{name}_{drv}"] = np.array(f"{type(e).__name__}: {e}")
    path = os.path.join(HERE, "inverse_mel_ref_cases.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
