"""Timing of the RNN-T feature extractors (audio_b200.pipelines.RNNTFeatureExtractor) against the reference chain on
CUDA: torchaudio's MelSpectrogram (when it imports, else torch.stft + the mel matrix) followed by the reference's
piecewise log and normalisation as torch ops.

    python tools/rnnt_bench.py [--steps 20] [--warmup 3] [--rounds 3]

  (a) the 1-D non-streaming extractor on one 10 s utterance: call latency including the host return (host clock around
      the call and a device synchronise), per call;
  (b) 256 x 10 s uniform batch (forward_batch without lengths): the kernel time, CUDA events over --steps launches;
  (c) a seeded ragged batch of 256 utterances of 2-16 s: one forward_batch launch with lengths against the recipes'
      per-utterance MelSpectrogram loop + pad_sequence + chain, CUDA events (both arms include their host work);
  (d) forward + backward on 64 x 10 s: audio_b200.differentiable(features=True) against torch autograd through the
      reference chain on CUDA.
The arms alternate, --rounds times; the table gives medians and the ranges, next to the device name and power limit.
All statistics are the LibriSpeech recipe's shape (80 values); their values do not change the timing.
"""
import argparse
import json
import math
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import audio_b200  # noqa: E402
from audio_b200.pipelines import RNNTFeatureExtractor, _gain  # noqa: E402
from bench import device_info  # noqa: E402


def reference_chain(ours, dev):
    """(mel(x) -> (..., n_mels, T), chain(mel frames-major) ) of the reference on CUDA."""
    mel_mod = ours.pipeline["0"]
    try:
        import torchaudio.transforms as TA

        mel = TA.MelSpectrogram(sample_rate=16000, n_fft=400, n_mels=80, hop_length=160).to(dev)
        src = "torchaudio"
    except Exception:  # noqa: BLE001
        w, fb = mel_mod.spectrogram.window, mel_mod.mel_scale.fb

        def mel(x):
            s = torch.stft(x, 400, 160, 400, w, center=True, pad_mode="reflect", return_complex=True).abs().pow(2.0)
            return torch.matmul(s.transpose(-1, -2), fb).transpose(-1, -2)

        src = "torch.stft"
    mean, invstd = ours.pipeline["3"].mean, ours.pipeline["3"].invstddev

    def chain(x):  # rnnt_pipeline.py:20-23, :43-44 (the recipe's form multiplies by the gain inside)
        x = x * _gain
        x[x > math.e] = torch.log(x[x > math.e])
        x[x <= math.e] = x[x <= math.e] / math.e
        return (x - mean) * invstd

    return mel, chain, src


def events_ms(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def host_ms(fn, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
        torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / steps


def compare(name, ours, ref, timer, steps, warmup, rounds):
    for _ in range(warmup):
        ours()
        ref()
    torch.cuda.synchronize()
    t_o, t_r = [], []
    for _ in range(rounds):
        t_o.append(timer(ours, steps))
        t_r.append(timer(ref, steps))
    row = {"workload": name, "audio_b200_ms": statistics.median(t_o), "audio_b200_ms_range": [min(t_o), max(t_o)],
           "reference_ms": statistics.median(t_r), "reference_ms_range": [min(t_r), max(t_r)]}
    row["speedup"] = row["reference_ms"] / row["audio_b200_ms"]
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    print(json.dumps({"device": device_info(0)}), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "global_stats.json")
        g = torch.Generator().manual_seed(0)
        with open(path, "w") as fh:
            json.dump({"mean": (15 + torch.rand(80, generator=g)).tolist(),
                       "invstddev": (0.3 + 0.05 * torch.rand(80, generator=g)).tolist()}, fh)
        full = RNNTFeatureExtractor(path).to(dev)
        stream = RNNTFeatureExtractor(path, right_padding=0).to(dev)
    mel, chain, src = reference_chain(full, dev)
    print(json.dumps({"reference_arm": src}), flush=True)
    rows = []

    # (a) 1-D, 10 s, call latency
    x = (0.1 * torch.randn(160000, generator=g)).to(dev)

    def ref_1d():
        f = chain(mel(x).transpose(1, 0))
        f = torch.nn.functional.pad(f, (0, 0, 0, 4))
        return f, torch.tensor([f.shape[0]])

    with torch.no_grad():
        rows.append(compare("(a) 1-D extractor, 10 s, call latency incl. host return", lambda: full(x), ref_1d, host_ms,
                            a.steps, a.warmup, a.rounds))

        # (b) 256 x 10 s uniform batch, kernel time
        xb = (0.1 * torch.randn(256, 160000, generator=g)).to(dev)
        rows.append(compare("(b) 256 x 10 s uniform batch, device time", lambda: stream.forward_batch(xb),
                            lambda: chain(mel(xb).transpose(-1, -2)), events_ms, a.steps, a.warmup, a.rounds))
        del xb

        # (c) ragged 256 x 2-16 s: one launch vs the recipe's per-utterance loop + pad_sequence
        lens = torch.randint(32000, 256001, (256,), generator=g).tolist()
        xr = torch.zeros(256, max(lens))
        for r, n in enumerate(lens):
            xr[r, :n] = 0.1 * torch.randn(n, generator=g)
        xr = xr.to(dev)
        utts = [xr[r, :n] for r, n in enumerate(lens)]

        def recipe():
            feats = torch.nn.utils.rnn.pad_sequence([mel(u).transpose(1, 0) for u in utts], batch_first=True)
            return chain(feats), torch.tensor([1 + n // 160 for n in lens], dtype=torch.int32)

        out, _ = stream.forward_batch(xr, lens)
        ref, _ = recipe()
        print(json.dumps({"ragged_max_abs_diff": float((out - ref).abs().max())}), flush=True)
        rows.append(compare("(c) ragged 256 x 2-16 s, one launch vs per-utterance loop + pad_sequence",
                            lambda: stream.forward_batch(xr, lens), recipe, events_ms, a.steps, a.warmup, a.rounds))
        del xr, utts

    # (d) forward + backward on 64 x 10 s
    xg = (0.1 * torch.randn(64, 160000, generator=g)).to(dev).requires_grad_(True)
    gy = torch.randn(64, 1001, 80, generator=g).to(dev)

    def ours_fb():
        with audio_b200.differentiable(features=True):
            out, _ = stream.forward_batch(xg)
        (gx,) = torch.autograd.grad(out, xg, gy)
        return gx

    def ref_fb():
        out = chain(mel(xg).transpose(-1, -2))
        (gx,) = torch.autograd.grad(out, xg, gy)
        return gx

    d = (ours_fb() - ref_fb()).abs().max() / ref_fb().abs().max()
    print(json.dumps({"grad_max_diff_rel_to_max": float(d)}), flush=True)
    rows.append(compare("(d) forward + backward, 64 x 10 s", ours_fb, ref_fb, events_ms, max(1, a.steps // 4), a.warmup,
                        a.rounds))
    print(json.dumps({"summary": rows}))


if __name__ == "__main__":
    main()
