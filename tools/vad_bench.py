#!/usr/bin/env python
"""Time F.vad on the GPU, and torchaudio's vad (CUDA and CPU) when torchaudio is importable.

Workloads: leading low-level noise, then a voiced signal (harmonics of a 140 Hz pitch contour), so the trigger lands where the voice
starts and the work done follows it:
  short  1 x 8 s at 16 kHz, voice at 3 s
  stereo 2 x 30 s at 44.1 kHz, voice at 20 s
  long   1 x 10 min at 16 kHz, voice at 9 min (many 1024-frame chunks)
  calls  64 sequential 4 s calls at 16 kHz, voice at 2 s (the per-call overhead)
Reports time per call (host clock around work that ends in a device synchronise), measurement frames per second,
kernel launches and status readbacks per call, and the card's name and power limit.

    python tools/vad_bench.py [--reps 20] [--out vad_bench.json]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import audio_b200.functional as F  # noqa: E402
from audio_b200 import _filtering  # noqa: E402


def signal(channels, seconds, sr, voice_at, seed=0):
    g = torch.Generator().manual_seed(seed)
    n = int(seconds * sr)
    x = torch.randn(channels, n, generator=g) * 1e-3
    t = torch.arange(n - int(voice_at * sr), dtype=torch.float64) / sr
    # 20 harmonics of a 140 Hz +-10% pitch contour under a 4 Hz syllable envelope: a steady tone would be learned by
    # the noise tracker and never trigger
    phase = 2 * math.pi * torch.cumsum(140 * (1 + 0.1 * torch.sin(2 * math.pi * 3 * t)), 0) / sr
    voice = sum(torch.sin(k * phase) / k for k in range(1, 21)) * 0.5 * (1 - torch.cos(2 * math.pi * 4 * t))
    x[:, int(voice_at * sr):] += (0.1 * voice).float()
    return x


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps


def launches(fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "vad_bench measures the GPU"
    try:
        import torchaudio.functional as RF
    except Exception:  # noqa: BLE001
        RF = None
    dev = torch.device("cuda")
    workloads = [("short", 1, 8, 16000, 3, 1), ("stereo", 2, 30, 44100, 20, 1), ("long", 1, 600, 16000, 540, 1),
                 ("calls", 1, 4, 16000, 2, 64)]
    rows = []
    for name, ch, sec, sr, at, calls in workloads:
        xs = [signal(ch, sec, sr, at, seed=i) for i in range(calls)]
        xd = [x.to(dev) for x in xs]
        plan = _filtering.VadPlan(sr)
        run = lambda: [F.vad(x, sr) for x in xd]  # noqa: E731
        t = timed(run, max(1, args.reps // calls))
        out = run()
        trig, _, _ = plan.run(xd[0].reshape(-1, xd[0].shape[-1]))
        chunks = trig // _filtering.VAD_CHUNK + 1 if trig >= 0 else math.ceil(plan.num_frames(sec * sr) / _filtering.VAD_CHUNK)
        row = dict(workload=name, channels=ch, seconds=sec, sample_rate=sr, calls=calls, out_len=out[0].shape[-1],
                   trigger_frame=trig, us_per_call=1e6 * t / calls,
                   frames_per_s=(trig + 1) * ch * calls / t if trig >= 0 else None,
                   launches_per_call=launches(lambda: F.vad(xd[0], sr)), readbacks_per_call=chunks)
        if RF is not None:
            ref_out = RF.vad(xd[0], sr)
            row["torchaudio_cuda_us_per_call"] = 1e6 * timed(lambda: RF.vad(xd[0], sr), 1)
            row["torchaudio_cpu_us_per_call"] = 1e6 * timed(lambda: RF.vad(xs[0], sr), 1)
            row["lengths_equal"] = ref_out.shape[-1] == out[0].shape[-1] == RF.vad(xs[0], sr).shape[-1]
        else:
            row["torchaudio"] = "not importable"
        rows.append(row)
        print(json.dumps(row))
    result = dict(card=card(), rows=rows)
    print(json.dumps(dict(card=result["card"])))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
