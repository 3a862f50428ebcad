#!/usr/bin/env python
"""Time F.forced_align on the GPU against torchaudio's forced_align on CUDA (row by row: it takes batch 1) and on
the CPU.

Workloads (log-softmax of N(0, 2) emissions, float32, int32 targets drawn from the non-blank classes):
  long       B 1,  T 30000, L 8000,             C 32:   one long utterance, the walk's per-frame latency
  batch      B 64, T 1000,  L_b ragged 150-300, C 32:   many utterances in one launch
  wordpiece  B 16, T 500,   L 100,              C 5000: wide vocabulary, gathered emissions
Per workload: a host clock around `reps` calls that end in a device synchronise, after warm-up, for ours, torchaudio
CUDA (the whole batch, one row after another) and torchaudio CPU (one pass); how many rows' paths and scores equal
torchaudio CPU's; the card's name and power limit.  --profile instead writes the check / walk kernel split from
torch.profiler.

    python tools/forced_align_bench.py [--reps 10] [--out forced_align_bench.json] [--profile] [--no-cpu]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import audio_b200.functional as F  # noqa: E402

WORKLOADS = {  # B, T, L_min, L_max, C
    "long": (1, 30000, 8000, 8000, 32),
    "batch": (64, 1000, 150, 300, 32),
    "wordpiece": (16, 500, 100, 100, 5000),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def inputs(B, T, lo, hi, C, seed=0):
    g = torch.Generator().manual_seed(seed)
    lp = torch.log_softmax(2 * torch.randn(B, T, C, generator=g), -1)
    ul = torch.randint(lo, hi + 1, (B,), generator=g)
    ul[0] = hi
    tg = torch.randint(1, C, (B, hi), generator=g, dtype=torch.int32)
    return lp, tg, torch.full((B,), T), ul


def timed(fn, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps


def rows(TF, lp, tg, tl, ul):
    return [TF.forced_align(lp[b: b + 1, : int(tl[b])], tg[b: b + 1, : int(ul[b])], blank=0)
            for b in range(lp.shape[0])]


def profile_split(args):
    from torch.profiler import ProfilerActivity, profile

    for _ in range(2):
        F.forced_align(*args)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            F.forced_align(*args)
        torch.cuda.synchronize()
    split = {"check": 0.0, "walk": 0.0, "other": 0.0}
    for e in prof.key_averages():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        key = "check" if "fa_check_kernel" in e.key else "walk" if "fa_walk_kernel" in e.key else "other"
        split[key] += e.device_time_total / 5
    return {k: round(v, 2) for k, v in split.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    a = ap.parse_args()
    try:
        import torchaudio.functional as TF
    except Exception:  # noqa: BLE001
        TF = None
    res = {"card": card(), "workloads": {}}
    for name in a.workloads.split(","):
        B, T, lo, hi, C = WORKLOADS[name]
        lp, tg, tl, ul = inputs(B, T, lo, hi, C)
        dev = (lp.cuda(), tg.cuda(), tl.cuda(), ul.cuda())
        r = {"shape": [B, T, hi, C]}
        if a.profile:
            r["kernel_us_per_call"] = profile_split(dev)
            res["workloads"][name] = r
            print(name, json.dumps(r), flush=True)
            continue
        r["ours_ms"] = timed(lambda: F.forced_align(*dev), a.reps) * 1e3
        if TF is not None:
            r["torchaudio_cuda_ms"] = timed(lambda: rows(TF, *dev), max(1, a.reps // 5)) * 1e3
            r["speedup_vs_torchaudio_cuda"] = r["torchaudio_cuda_ms"] / r["ours_ms"]
            if not a.no_cpu:
                t0 = time.perf_counter()
                ref = rows(TF, lp, tg, tl, ul)
                r["torchaudio_cpu_ms"] = (time.perf_counter() - t0) * 1e3
                r["speedup_vs_torchaudio_cpu"] = r["torchaudio_cpu_ms"] / r["ours_ms"]
                p, s = (x.cpu() for x in F.forced_align(*dev))
                r["rows_equal_to_cpu"] = sum(int(torch.equal(p[b], rp[0]) and torch.equal(s[b], rs[0]))
                                             for b, (rp, rs) in enumerate(ref))
        res["workloads"][name] = r
        print(name, json.dumps(r), flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
