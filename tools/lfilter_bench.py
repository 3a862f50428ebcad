"""IIR filtering on the GPU against the installed torchaudio's CUDA lfilter (its serial iir_cu_kernel plus conv1d, and
its autograd), timed with CUDA events, the arms alternated within one call after every shape is warmed up.

Workloads: highpass_biquad on 64 x 160 000 (10 s at 16 kHz); lfilter with 64 filters of order 4, batching=True, on
8 x 64 x 48 000; deemphasis on 256 x 16 000; forward + backward (waveform and coefficient gradients) of the first
shape.  Prints, per workload, the median kernel time, the achieved bytes/s from the bytes the algorithm must move (the
forward reads x twice and writes y once: 12 B/sample) against the 3.35 TB/s data-sheet HBM3 bandwidth, the speed-up
over the reference arm and the max-abs difference of the outputs; then the card name and power limit, read in the
same run.

    python tools/lfilter_bench.py [--iters 30]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import audio_b200  # noqa: E402
import audio_b200.functional as F  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data-sheet HBM3 bandwidth


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=20)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def time_once(fn):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) * 1e3  # microseconds


def median(v):
    v = sorted(v)
    return v[len(v) // 2] if v else None


def workloads():
    g = torch.Generator(device="cuda").manual_seed(0)
    x1 = 0.5 * torch.randn(64, 160000, device="cuda", generator=g)
    x2 = 0.5 * torch.randn(8, 64, 48000, device="cuda", generator=g)
    x3 = 0.5 * torch.randn(256, 16000, device="cuda", generator=g)
    # 64 order-4 filters: cascades of two resonators at spread frequencies (stable by construction)
    r = torch.linspace(0.90, 0.99, 64, device="cuda")
    w = torch.linspace(0.05, 2.5, 64, device="cuda")
    p1 = torch.stack([torch.ones_like(r), -2 * r * torch.cos(w), r * r], 1)
    p2 = torch.stack([torch.ones_like(r), -2 * r * torch.cos(w / 2), r * r], 1)
    a4 = torch.stack([p1[:, 0] * p2[:, 0], p1[:, 0] * p2[:, 1] + p1[:, 1] * p2[:, 0],
                      p1[:, 0] * p2[:, 2] + p1[:, 1] * p2[:, 1] + p1[:, 2] * p2[:, 0],
                      p1[:, 1] * p2[:, 2] + p1[:, 2] * p2[:, 1], p1[:, 2] * p2[:, 2]], 1).contiguous()
    b4 = torch.zeros_like(a4)
    b4[:, 0] = (1 - r) ** 2
    return [
        ("highpass_biquad 64x160000", x1, lambda M, x: M.highpass_biquad(x, 16000, 200.0)),
        ("lfilter 64 filters order 4, 8x64x48000", x2, lambda M, x: M.lfilter(x, a4, b4, clamp=False)),
        ("deemphasis 256x16000", x3, lambda M, x: M.deemphasis(x, 0.97)),
    ]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    args = ap.parse_args()
    try:
        import torchaudio.functional as TA

        TA.lfilter(torch.zeros(1, 8, device="cuda"), torch.tensor([1.0, 0.5], device="cuda"),
                   torch.tensor([1.0, 0.0], device="cuda"))
    except Exception as exc:  # noqa: BLE001
        print(f"reference arm unavailable: {exc}", file=sys.stderr)
        TA = None
    results = []
    for name, x, fn in workloads():
        arms = {"audio_b200": F} if TA is None else {"audio_b200": F, "torchaudio": TA}
        with torch.no_grad():
            outs = {k: fn(M, x) for k, M in arms.items()}  # warm-up, and the outputs compared
            times = {k: [] for k in arms}
            for _ in range(args.iters):
                for k, M in arms.items():
                    times[k].append(time_once(lambda: fn(M, x)))
        t = median(times["audio_b200"])
        nbytes = 12 * x.numel()
        row = {"workload": name, "us": round(t, 1), "GB/s": round(nbytes / t * 1e-3, 1),
               "of_hbm_peak": round(nbytes / (t * 1e-6) / HBM_BYTES_PER_S, 3)}
        if TA is not None:
            row["ref_us"] = round(median(times["torchaudio"]), 1)
            row["speedup"] = round(row["ref_us"] / t, 1)
            row["max_abs_diff"] = float((outs["audio_b200"] - outs["torchaudio"]).abs().max())
        results.append(row)
        print(json.dumps(row), flush=True)
    # forward + backward of the first shape: waveform and coefficient gradients
    name, x, _ = workloads()[0]
    a = torch.tensor([1.0, -1.8, 0.82], device="cuda")
    b = torch.tensor([0.9, -1.8, 0.9], device="cuda")
    up = torch.randn_like(x)

    def step(M, with_switch):
        xg, ag, bg = x.clone().requires_grad_(), a.clone().requires_grad_(), b.clone().requires_grad_()
        if with_switch:
            with audio_b200.differentiable(filtering=True):
                y = M.lfilter(xg, ag, bg)
        else:
            y = M.lfilter(xg, ag, bg)
        (y * up).sum().backward()
        return xg.grad, ag.grad, bg.grad

    arms = {"audio_b200": (F, True)} if TA is None else {"audio_b200": (F, True), "torchaudio": (TA, False)}
    grads = {k: step(*v) for k, v in arms.items()}
    times = {k: [] for k in arms}
    for _ in range(max(args.iters // 3, 5)):
        for k, v in arms.items():
            times[k].append(time_once(lambda: step(*v)))
    t = median(times["audio_b200"])
    row = {"workload": "forward+backward " + name, "us": round(t, 1)}
    if TA is not None:
        row["ref_us"] = round(median(times["torchaudio"]), 1)
        row["speedup"] = round(row["ref_us"] / t, 1)
        ours, theirs = grads["audio_b200"], grads["torchaudio"]
        row["grad_rel_diff"] = [float((o - r).abs().max() / r.abs().max().clamp_min(1e-30)) for o, r in zip(ours, theirs)]
    results.append(row)
    print(json.dumps(row), flush=True)
    name, power = card()
    print(json.dumps({"card": name, "power_limit": power}))


if __name__ == "__main__":
    main()
