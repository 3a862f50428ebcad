"""FFT convolution on the GPU against the installed torchaudio's CUDA fftconvolve (three cuFFT transforms of the full
length and a slice), timed with CUDA events, the arms alternated within one call after every shape is warmed up.

Workloads: (a) 64 x 160 000 with per-row 8 000-tap RIRs (10 s at 16 kHz, 0.5 s reverberation); (b) the same with one
shared RIR; (c) 32 x 480 000 with 48 000-tap RIRs (10 s and 1 s at 48 kHz, P = 24 partitions); (d) 256 x 160 000 with
one shared 255-tap FIR (P = 1); (e) forward + backward of (a); (f) the "same" mode of (a).  Prints, per workload, the
median time, the achieved bytes/s from the compulsory bytes 4 (N + M + L) per row (the forward reads both operands and
writes the output once; (e) counts the forward's bytes plus the backward's 4 (L + N + M) reads and 4 (N + M) writes)
against the 3.35 TB/s data-sheet HBM3 bandwidth, the speed-up over the reference arm and the max-abs difference of
the outputs; then the card name and power limit, read in the same run.

    python tools/fftconvolve_bench.py [--iters 30]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import audio_b200  # noqa: E402
import audio_b200.functional as F  # noqa: E402
from tools.lfilter_bench import HBM_BYTES_PER_S, card, median, time_once  # noqa: E402


def rir(rows, taps, g):
    decay = torch.exp(-torch.arange(taps, device="cuda") / (taps / 6))
    return torch.randn(rows, taps, device="cuda", generator=g) * decay


def workloads():
    g = torch.Generator(device="cuda").manual_seed(0)
    x16 = 0.5 * torch.randn(64, 160000, device="cuda", generator=g)
    x48 = 0.5 * torch.randn(32, 480000, device="cuda", generator=g)
    x256 = 0.5 * torch.randn(256, 160000, device="cuda", generator=g)
    h8k, h8k_shared = rir(64, 8000, g), rir(1, 8000, g)
    h48k = rir(32, 48000, g)
    fir = torch.randn(1, 255, device="cuda", generator=g) / 16
    return [
        ("(a) 64x160000, per-row 8000-tap RIRs", x16, h8k, "full"),
        ("(b) 64x160000, one shared 8000-tap RIR", x16, h8k_shared, "full"),
        ("(c) 32x480000, 48000-tap RIRs (P=24)", x48, h48k, "full"),
        ("(d) 256x160000, shared 255-tap FIR (P=1)", x256, fir, "full"),
        ("(f) 64x160000, per-row 8000-tap RIRs, same", x16, h8k, "same"),
    ]


def compulsory_bytes(x, y, out):
    rows = out.shape[0]
    return 4 * rows * (x.shape[-1] + y.shape[-1] + out.shape[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    args = ap.parse_args()
    try:
        import torchaudio.functional as TA

        TA.fftconvolve(torch.zeros(1, 8, device="cuda"), torch.ones(1, 3, device="cuda"))
    except Exception as exc:  # noqa: BLE001
        print(f"reference arm unavailable: {exc}", file=sys.stderr)
        TA = None
    arms = {"audio_b200": F} if TA is None else {"audio_b200": F, "torchaudio": TA}
    for name, x, y, mode in workloads():
        with torch.no_grad():
            outs = {k: M.fftconvolve(x, y, mode) for k, M in arms.items()}  # warm-up, and the outputs compared
            times = {k: [] for k in arms}
            for _ in range(args.iters):
                for k, M in arms.items():
                    times[k].append(time_once(lambda: M.fftconvolve(x, y, mode)))
        t = median(times["audio_b200"])
        nbytes = compulsory_bytes(x, y, outs["audio_b200"])
        row = {"workload": name, "us": round(t, 1), "GB/s": round(nbytes / t * 1e-3, 1),
               "of_hbm_peak": round(nbytes / (t * 1e-6) / HBM_BYTES_PER_S, 3)}
        if TA is not None:
            row["ref_us"] = round(median(times["torchaudio"]), 1)
            row["speedup"] = round(row["ref_us"] / t, 2)
            row["max_abs_diff"] = float((outs["audio_b200"] - outs["torchaudio"]).abs().max())
        print(json.dumps(row), flush=True)
        del outs

    # (e) forward + backward of (a): the gradients of both operands
    _, x, y, mode = workloads()[0]
    up = torch.randn(x.shape[0], x.shape[1] + y.shape[1] - 1, device="cuda")

    def step(M, with_switch):
        xg, yg = x.clone().requires_grad_(), y.clone().requires_grad_()
        if with_switch:
            with audio_b200.differentiable(filtering=True):
                out = M.fftconvolve(xg, yg)
        else:
            out = M.fftconvolve(xg, yg)
        (out * up).sum().backward()
        return xg.grad, yg.grad

    garms = {"audio_b200": (F, True)} if TA is None else {"audio_b200": (F, True), "torchaudio": (TA, False)}
    grads = {k: step(*v) for k, v in garms.items()}
    times = {k: [] for k in garms}
    for _ in range(max(args.iters // 3, 5)):
        for k, v in garms.items():
            times[k].append(time_once(lambda: step(*v)))
    t = median(times["audio_b200"])
    fwd = compulsory_bytes(x, y, up)
    nbytes = fwd + 4 * x.shape[0] * (up.shape[1] + 2 * (x.shape[1] + y.shape[1]))
    row = {"workload": "(e) forward+backward of (a)", "us": round(t, 1), "GB/s": round(nbytes / t * 1e-3, 1),
           "of_hbm_peak": round(nbytes / (t * 1e-6) / HBM_BYTES_PER_S, 3)}
    if TA is not None:
        row["ref_us"] = round(median(times["torchaudio"]), 1)
        row["speedup"] = round(row["ref_us"] / t, 2)
        ours, theirs = grads["audio_b200"], grads["torchaudio"]
        row["grad_rel_diff"] = [float((o - r).abs().max() / r.abs().max().clamp_min(1e-30)) for o, r in zip(ours, theirs)]
    print(json.dumps(row), flush=True)
    name, power = card()
    print(json.dumps({"card": name, "power_limit": power}))


if __name__ == "__main__":
    main()
