#!/usr/bin/env python
"""Per-config throughput table for BASELINE.json configs 2-5 on ONE GPU (inputs resident in HBM).

Not the benchmark's JSON line (that is bench.py); a per-config table for kernel work.
    python tools/bench_configs.py [--quick] [--out configs.json]
For every config: kernel time (CUDA events, median of blocks of back-to-back launches), throughput,
algorithmic bytes (SURVEY.md 8d) / time vs the measured HBM peak, and the torchaudio CPU reference on a
bounded sample of the same workload.
"""
import argparse
import json
import os
import statistics
import sys
import time
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import audio_b200.transforms as T  # noqa: E402


def hbm_peak():
    try:
        with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as fh:
            return float(json.load(fh)["hbm_gbs"])
    except Exception:
        return 3350.0  # H100 SXM data-sheet HBM3 bandwidth, not measured


def time_gpu(fn, iters=20, blocks=5):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(blocks):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / iters)
    return statistics.median(times)


def time_cpu(make_module, x_cpu, threads=16):
    try:
        import torchaudio  # noqa: F401
    except Exception:
        return None
    torch.set_num_threads(min(threads, os.cpu_count() or 1))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        mod = make_module(__import__("torchaudio").transforms)
    with torch.inference_mode():
        mod(x_cpu)
        t0 = time.perf_counter()
        mod(x_cpu)
        return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-cpu", action="store_true", help="skip the torchaudio CPU reference timings")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    peak = hbm_peak()
    rows = []
    L = 160000

    def run(name, make, x, units, unit_name, algo_bytes, cpu_rows):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            mod = make(T).to(dev)
        with torch.inference_mode():
            ms = time_gpu(lambda: mod(x), iters=5 if args.quick else 20, blocks=3 if args.quick else 5)
        cpu_s = None if args.no_cpu else time_cpu(make, x[:cpu_rows].cpu())
        cpu_rate = None if cpu_s is None else units * cpu_rows / x.shape[0] / cpu_s
        rec = {"config": name, "ms": ms, "rate": units / (ms * 1e-3), "unit": unit_name,
               "algorithmic_MB": algo_bytes / 1e6, "achieved_GBs": algo_bytes / (ms * 1e-3) / 1e9,
               "frac_of_hbm_peak": algo_bytes / (ms * 1e-3) / 1e9 / peak, "cpu_reference_rate": cpu_rate,
               "cpu_sample_rows": cpu_rows}
        rows.append(rec)
        print(json.dumps(rec), flush=True)

    g = torch.Generator(device=dev).manual_seed(1234)
    x = torch.randn(256, L, device=dev, generator=g)
    # config 2
    fr = 1 + L // 256
    run("C2 MelSpectrogram n_fft=1024 hop=256 n_mels=80, 256x160000",
        lambda M: M.MelSpectrogram(16000, n_fft=1024, hop_length=256, n_mels=80), x, 256 * fr, "frames/s",
        4 * (256 * L + 256 * fr * 80) + 4 * (1024 + 513 * 80), 32)
    # Spectrogram alone (power output)
    run("Spectrogram n_fft=1024 hop=256, 256x160000",
        lambda M: M.Spectrogram(n_fft=1024, hop_length=256), x, 256 * fr, "frames/s",
        4 * (256 * L + 256 * fr * 513), 32)
    # config 4 (one GPU's shard of 256)
    run("C4 MFCC n_mfcc=40 over C2 mel, 256x160000 (2-D input: batch-global top_db)",
        lambda M: M.MFCC(16000, n_mfcc=40, melkwargs=dict(n_fft=1024, hop_length=256, n_mels=80)), x, 256 * fr,
        "frames/s", 4 * (256 * L + 256 * fr * 40), 32)
    # config 5 sweep
    for n_fft in (256, 512, 1024, 2048):
        hop = n_fft // 4
        fr5 = 1 + L // hop
        for batch in ((64, 256) if args.quick else (64, 128, 256, 512, 1024)):
            if n_fft == 256 and batch == 1024:
                xb = torch.randn(batch, L, device=dev, generator=g)
            else:
                xb = torch.randn(batch, L, device=dev, generator=g)
            run(f"C5 MelSpectrogram n_fft={n_fft} hop={hop} n_mels=80, {batch}x160000",
                lambda M, n=n_fft, h=hop: M.MelSpectrogram(16000, n_fft=n, hop_length=h, n_mels=80), xb, batch * fr5,
                "frames/s", 4 * (batch * L + batch * fr5 * 80) + 4 * (n_fft + (n_fft // 2 + 1) * 80), 16)
            del xb
    # config 3
    del x
    torch.cuda.empty_cache()
    xr = torch.randn(1024, 220500, device=dev, generator=g)
    run("C3 Resample 44.1k->16k sinc_interp_kaiser, 1024x220500",
        lambda M: M.Resample(44100, 16000, resampling_method="sinc_interp_kaiser"), xr, 1024 * 80000, "out-samples/s",
        4 * (1024 * 220500 + 1024 * 80000), 64)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump({"hbm_peak_GBs": peak, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
