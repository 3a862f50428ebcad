#!/usr/bin/env python
"""Forward + backward of the Kaldi features with waveform gradients on one GPU: fbank_batch(num_mel_bins=80) and
mfcc_batch() on 256 x 160 000 samples at 16 kHz (the tools/kaldi_bench.py workload), against torch's CUDA autograd of the
same op sequence (tests/kaldi_grad_oracle.py:torch_kaldi, batched over the rows) and torchaudio.compliance.kaldi.fbank per row
where it is importable.  Medians of alternating rounds; the card and its power limit are read in the same run.  Also
the backward's compulsory HBM traffic against the data-sheet 3.35 TB/s.
    python tools/kaldi_grad_bench.py
"""
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

import audio_b200  # noqa: E402
import audio_b200.compliance.kaldi as K  # noqa: E402
from kaldi_grad_oracle import torch_kaldi  # noqa: E402

ROWS, LENGTH, PADDED, WIN = 256, 160000, 512, 400


def _time(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def main():
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print("card:", card)
    x = (torch.randn(ROWS, LENGTH, device="cuda") * 3000.0).round()
    frames = 1 + (LENGTH - WIN) // 160

    def ours(fn, kw):
        def run():
            with audio_b200.differentiable(kaldi=True):
                xt = x.detach().requires_grad_()
                fn(xt, **kw).sum().backward()
        return run

    def restated(kind, kw):  # all rows in one graph: the frame gather indexes (rows, T, win)
        def run():
            xt = x.detach().requires_grad_()
            torch_kaldi(kind, xt, **kw).sum().backward()
        return run

    cases = [("fbank 80 bins", ours(K.fbank_batch, dict(num_mel_bins=80)), restated("fbank", dict(num_mel_bins=80))),
             ("mfcc 13 of 23", ours(K.mfcc_batch, {}), restated("mfcc", {}))]
    try:
        import torchaudio.compliance.kaldi as TK

        def ta():
            xt = x.detach().requires_grad_()
            sum(TK.fbank(xt[r:r + 1], num_mel_bins=80).sum() for r in range(ROWS)).backward()
        cases[0] = cases[0] + (ta,)
    except Exception as e:  # noqa: BLE001
        print("torchaudio unavailable:", e)
    for name, *fns in cases:
        for f in fns:
            f()
        rounds = [[_time(f, 3 if i == 0 else 1) for i, f in enumerate(fns)] for _ in range(5)]
        med = [statistics.median(r[i] for r in rounds) for i in range(len(fns))]
        labels = ["audio_b200", "torch restatement, batched (CUDA autograd)", "torchaudio, one call per row (CUDA autograd)"]
        print(f"{name}: " + ", ".join(f"{labels[i]} {m:.2f} ms" for i, m in enumerate(med)), flush=True)

    # the backward alone (fbank, padded 512: the fused kernel): compulsory bytes = waveform read + gradient write +
    # pre-log rows (81 floats a frame) written and read + frame gradients (padded floats a frame) written and read
    with audio_b200.differentiable(kaldi=True):
        xt = x.detach().requires_grad_()
        y = K.fbank_batch(xt, num_mel_bins=80)
    g = torch.ones_like(y)
    bwd = lambda: torch.autograd.grad(y, xt, g, retain_graph=True)  # noqa: E731
    bwd()
    t = statistics.median(_time(bwd, 3) for _ in range(5))
    n = ROWS * frames
    nbytes = 4 * (2 * ROWS * LENGTH + 2 * n * PADDED + 2 * n * 81)
    print(f"fbank backward alone: {t:.3f} ms, compulsory {nbytes / 1e6:.1f} MB -> {nbytes / t / 1e9:.3f} TB/s "
          f"({100 * nbytes / t / 1e9 / 3.35:.1f}% of 3.35 TB/s)")


if __name__ == "__main__":
    main()
