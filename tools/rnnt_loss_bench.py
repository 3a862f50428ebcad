#!/usr/bin/env python
"""Time F.rnnt_loss on the GPU against torchaudio's CUDA rnnt_loss (and, for the char workload, its CPU path).

Workloads, ragged lengths in [75 %, 100 %] of the maximum:
  wordpiece     B 16, T 200,  U+1 61,  V 4097, float32 and float16 (the Emformer RNN-T joint)
  char          B 32, T 400,  U+1 151, V 29: the alpha / beta walk dominates
  long          B 4,  T 1500, U+1 301, V 1024
Per workload: forward time (logits not requiring grad) and forward + backward time (loss.backward()), each a host
clock around `reps` calls that end in a device synchronise, after warm-up; the valid-row traffic the loss needs (two
reads and one write of the valid rows) over forward + backward time against 3.35 TB/s; the peak memory one
forward + backward allocates above the inputs (the logit gradient included); the cost and gradient agreement with
torchaudio CUDA on the timed inputs; the card's name and power limit.  --profile instead writes the per-kernel split (check / rows / alpha-beta / gradient) from torch.profiler.

    python tools/rnnt_loss_bench.py [--reps 20] [--out rnnt_loss_bench.json] [--profile]
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

WORKLOADS = {
    "wordpiece_f32": (16, 200, 61, 4097, torch.float32),
    "wordpiece_f16": (16, 200, 61, 4097, torch.float16),
    "char": (32, 400, 151, 29, torch.float32),
    "long": (4, 1500, 301, 1024, torch.float32),
}
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def inputs(B, T, U1, V, dtype, seed=0):
    g = torch.Generator().manual_seed(seed)
    tl = torch.randint((3 * T + 3) // 4, T + 1, (B,), generator=g, dtype=torch.int32)
    ul = torch.randint((3 * (U1 - 1) + 3) // 4, U1, (B,), generator=g, dtype=torch.int32)
    tl[0], ul[-1] = T, U1 - 1
    tg = torch.randint(0, V - 1, (B, U1 - 1), generator=g, dtype=torch.int32)
    x = torch.randn(B, T, U1, V, generator=g).to(dtype)
    valid = int((tl.long() * (ul.long() + 1)).sum()) * V * x.element_size()
    return x.cuda(), tg.cuda(), tl.cuda(), ul.cuda(), valid


def timed(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps


def fwd_bwd(loss_fn, x, args):
    x.grad = None
    loss_fn(x, *args, reduction="sum").backward()


def peak(fn, x):
    """Bytes allocated at the peak of fn() above what was allocated before it, x's gradient freed."""
    x.grad = None
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def profile_split(x, args):
    from torch.profiler import ProfilerActivity, profile

    xg = x.detach().clone().requires_grad_()
    for _ in range(3):
        fwd_bwd(F.rnnt_loss, xg, args)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            fwd_bwd(F.rnnt_loss, xg, args)
        torch.cuda.synchronize()
    split = {"check": 0.0, "rows": 0.0, "alpha_beta": 0.0, "gradient": 0.0, "other": 0.0}
    for e in prof.key_averages():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = e.device_time_total / 5
        key = ("check" if "rnnt_check_kernel" in e.key else "rows" if "rnnt_rows_kernel" in e.key else
               "alpha_beta" if "rnnt_alpha_beta_kernel" in e.key else "gradient" if "rnnt_grad_kernel" in e.key else
               "other")
        split[key] += us
    fwd = split["check"] + split["rows"] + split["alpha_beta"]
    split["alpha_beta_share_of_forward_kernels"] = split["alpha_beta"] / fwd if fwd else None
    return {k: (round(v, 2) if isinstance(v, float) else v) for k, v in split.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    a = ap.parse_args()
    try:
        import torchaudio.functional as TF
    except Exception:  # noqa: BLE001
        TF = None
    res = {"card": card(), "workloads": {}}
    for name in a.workloads.split(","):
        B, T, U1, V, dtype = WORKLOADS[name]
        x, tg, tl, ul, valid = inputs(B, T, U1, V, dtype)
        args = (tg, tl, ul)
        r = {"shape": [B, T, U1, V], "dtype": str(dtype).split(".")[-1], "valid_row_bytes": valid}
        if a.profile:
            r["kernel_us_per_fwd_bwd"] = profile_split(x, args)
            res["workloads"][name] = r
            print(name, json.dumps(r), flush=True)
            continue
        xg = x.detach().clone().requires_grad_()
        r["ours_fwd_ms"] = timed(lambda: F.rnnt_loss(x, *args), a.reps) * 1e3
        r["ours_fwd_bwd_ms"] = timed(lambda: fwd_bwd(F.rnnt_loss, xg, args), a.reps) * 1e3
        r["ours_peak_bytes"] = peak(lambda: fwd_bwd(F.rnnt_loss, xg, args), xg)
        rate = 3 * valid / (r["ours_fwd_bwd_ms"] * 1e-3)
        r["ours_valid_traffic_TBps"] = rate / 1e12
        r["ours_share_of_3.35TBps"] = rate / HBM_BYTES_PER_S
        if TF is not None:
            xt = x.detach().clone().requires_grad_()
            r["torchaudio_cuda_fwd_ms"] = timed(lambda: TF.rnnt_loss(x, *args), a.reps) * 1e3
            r["torchaudio_cuda_fwd_bwd_ms"] = timed(lambda: fwd_bwd(TF.rnnt_loss, xt, args), a.reps) * 1e3
            r["torchaudio_cuda_peak_bytes"] = peak(lambda: fwd_bwd(TF.rnnt_loss, xt, args), xt)
            r["speedup_fwd_bwd"] = r["torchaudio_cuda_fwd_bwd_ms"] / r["ours_fwd_bwd_ms"]
            fwd_bwd(F.rnnt_loss, xg, args)
            fwd_bwd(TF.rnnt_loss, xt, args)
            c1 = F.rnnt_loss(x, *args, reduction="none").double()
            c2 = TF.rnnt_loss(x, *args, reduction="none").double()
            r["cost_max_rel_diff"] = float(((c1 - c2).abs() / c2.abs()).max())
            r["grad_max_abs_diff"] = float((xg.grad.double() - xt.grad.double()).abs().max())
            del xt
            if name == "char":
                xc = x.detach().cpu().requires_grad_()
                argc = tuple(t.cpu() for t in args)
                t0 = time.perf_counter()
                fwd_bwd(TF.rnnt_loss, xc, argc)
                r["torchaudio_cpu_fwd_bwd_ms"] = (time.perf_counter() - t0) * 1e3
        res["workloads"][name] = r
        print(name, json.dumps(r), flush=True)
        del x, xg
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
