#!/usr/bin/env python
"""Generate tests/golden/rnnt_ref_cases.npz, the RNN-T feature-chain fixture (needs a pytorch/audio checkout named by
AUDIO_REFERENCE; run once):

    python tests/golden/make_rnnt_golden.py

It holds, all float32 from the reference itself on the CPU:
- ``stats_librispeech_{mean,invstddev}`` and ``stats_tedlium3_{mean,invstddev}``: the arrays of the recipes'
  global_stats.json files (examples/asr/librispeech_conformer_rnnt/global_stats.json, which the Emformer LibriSpeech
  recipe shares, and examples/asr/emformer_rnnt/tedlium3/global_stats.json);
- ``base_{n}``: seeded speech-like signals of n = 201 (T = 2), 3200 (0.2 s), 16000 (1 s) and 37920 (2.37 s) samples
  with a stretch of exact zeros; the inputs are ``fl32(base * level)`` for the levels in ``levels``;
- ``full_{n}_{i}`` / ``stream_{n}_{i}``: the non-streaming / streaming extractor of RNNTBundle
  (pipelines/rnnt_pipeline.py:310-343, the Emformer LibriSpeech bundle's parameters) on input (n, levels[i]), built by
  the reference's own get_feature_extractor() with the statistics file read locally;
- ``batch_lengths``, ``batch_levels``, ``batch_feats``: the recipes' _extract_features + _piecewise_linear_log +
  GlobalStatsNormalization (examples/asr/librispeech_conformer_rnnt/transforms.py:13-78, without SpecAugment) on six
  utterances ``fl32(base_37920[:L] * level)`` of different lengths, with the TED-LIUM 3 statistics.
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
import torchaudio.pipelines.rnnt_pipeline as RP  # noqa: E402

assert torchaudio.__file__.startswith(REF), torchaudio.__file__

LENGTHS = (201, 3200, 16000, 37920)
LEVELS = np.array([1.0, 1e-3, 1e-5], dtype=np.float32)
BATCH_LENGTHS = np.array([16000, 12345, 8000, 4321, 3200, 801], dtype=np.int64)
BATCH_LEVELS = np.array([1.0, 1e-3, 1e-5, 1.0, 1e-3, 1.0], dtype=np.float32)


def base_signal(n, g):
    """Noise with a slow envelope and a stretch of exact zeros over the middle fifth (silence frames)."""
    t = torch.linspace(0, 7.0, n)
    env = 0.2 + 0.8 * torch.sin(t) ** 2
    x = 0.3 * torch.randn(n, generator=g) * env
    x[2 * n // 5 : 3 * n // 5] = 0.0
    return x.to(torch.float32)


def read_stats(path):
    with open(path) as fh:
        blob = json.load(fh)
    return np.asarray(blob["mean"], dtype=np.float32), np.asarray(blob["invstddev"], dtype=np.float32)


def main():
    ex = os.path.join(REF, "examples", "asr")
    libri = os.path.join(ex, "librispeech_conformer_rnnt", "global_stats.json")
    ted = os.path.join(ex, "emformer_rnnt", "tedlium3", "global_stats.json")
    out = {}
    out["stats_librispeech_mean"], out["stats_librispeech_invstddev"] = read_stats(libri)
    out["stats_tedlium3_mean"], out["stats_tedlium3_invstddev"] = read_stats(ted)
    out["levels"] = LEVELS

    # the reference's own extractors; its asset download is replaced by the local statistics file
    bundle = torchaudio.pipelines.EMFORMER_RNNT_BASE_LIBRISPEECH
    RP.torchaudio.utils._download_asset = lambda key, *a, **k: libri
    full, stream = bundle.get_feature_extractor(), bundle.get_streaming_feature_extractor()

    g = torch.Generator().manual_seed(1234)
    for n in LENGTHS:
        base = base_signal(n, g)
        out[f"base_{n}"] = base.numpy()
        for i, level in enumerate(LEVELS):
            x = torch.from_numpy(base.numpy() * level)
            with torch.no_grad():
                f, lf = full(x)
                s, ls = stream(x)
            assert int(lf) == f.shape[0] == s.shape[0] + 4 and int(ls) == s.shape[0]
            out[f"full_{n}_{i}"] = f.numpy()
            out[f"stream_{n}_{i}"] = s.numpy()

    # the recipes' batched form (transforms.py:13-24, :35-49, :62-67)
    spec = torchaudio.transforms.MelSpectrogram(sample_rate=16000, n_fft=400, n_mels=80, hop_length=160)
    mean, invstd = (torch.from_numpy(a) for a in read_stats(ted))
    base = torch.from_numpy(out["base_37920"])
    utts = [base[:n] * lv for n, lv in zip(BATCH_LENGTHS.tolist(), BATCH_LEVELS.tolist())]
    with torch.no_grad():
        mel = [spec(u).transpose(1, 0) for u in utts]
        feats = torch.nn.utils.rnn.pad_sequence(mel, batch_first=True)
        feats = RP._piecewise_linear_log(feats * RP._gain)
        feats = (feats - mean) * invstd
    out["batch_lengths"], out["batch_levels"] = BATCH_LENGTHS, BATCH_LEVELS
    out["batch_frames"] = np.array([m.shape[0] for m in mel], dtype=np.int32)
    out["batch_feats"] = feats.numpy()
    path = os.path.join(HERE, "rnnt_ref_cases.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
