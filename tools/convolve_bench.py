"""Direct convolution on the GPU against the installed torchaudio's CUDA convolve (a grouped cuDNN conv1d) at torch's
defaults (cuDNN TF32 on: what users get) and with cuDNN TF32 off (float32), and against our fftconvolve on the same
inputs, to show where the direct method stops paying.  Timed with CUDA events, the arms alternated within one call
after every shape is warmed up.

Workloads: (a) 256 x 160 000 with one shared 255-tap FIR (the input of fftconvolve_bench (d)); (b) the same with one
shared 5-tap filter (bandwidth-bound); (c) 64 x 160 000 with per-row 32-tap filters; (d) with per-row 1024-tap
filters; (e) with per-row 4096-tap filters (the cap); (f) forward + backward of (c).  Prints, per workload, the median
time of each arm, the achieved bytes/s from the compulsory bytes 4 (N + M + L) per row against the 3.35 TB/s
data-sheet HBM3 bandwidth, the useful 2 K L flop per row and the issued TF32 MMA flop (3 MMAs per product over
ceil((K + 7) / 8) k-steps of 8 columns) against the 495 TFLOP/s data-sheet dense TF32 rate, and the max-abs difference
to each arm; then the card name and power limit, read in the same run.

    python tools/convolve_bench.py [--iters 30]
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

TF32_FLOP_PER_S = 495e12  # H100 SXM data-sheet dense TF32 tensor-core rate


class _Cudnn:
    """torchaudio's convolve with cuDNN TF32 set for the call and restored after it."""

    def __init__(self, ta, tf32):
        self.ta, self.tf32 = ta, tf32

    def convolve(self, x, y, mode="full"):
        prev = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = self.tf32
        try:
            return self.ta.convolve(x, y, mode)
        finally:
            torch.backends.cudnn.allow_tf32 = prev


class _Fft:
    def convolve(self, x, y, mode="full"):
        return F.fftconvolve(x, y, mode)


def workloads():
    g = torch.Generator(device="cuda").manual_seed(0)
    x256 = 0.5 * torch.randn(256, 160000, device="cuda", generator=g)
    x64 = 0.5 * torch.randn(64, 160000, device="cuda", generator=g)
    return [
        ("(a) 256x160000, shared 255-tap FIR", x256, torch.randn(1, 255, device="cuda", generator=g) / 16),
        ("(b) 256x160000, shared 5-tap filter", x256, torch.randn(1, 5, device="cuda", generator=g) / 2),
        ("(c) 64x160000, per-row 32-tap filters", x64, torch.randn(64, 32, device="cuda", generator=g) / 6),
        ("(d) 64x160000, per-row 1024-tap filters", x64, torch.randn(64, 1024, device="cuda", generator=g) / 32),
        ("(e) 64x160000, per-row 4096-tap filters", x64, torch.randn(64, 4096, device="cuda", generator=g) / 64),
    ]


def counts(x, y, out):
    rows, k, length = out.shape[0], min(x.shape[-1], y.shape[-1]), out.shape[-1]
    nbytes = 4 * rows * (x.shape[-1] + y.shape[-1] + length)
    useful = 2 * k * length * rows
    issued = 3 * 2 * 8 * 8 * ((k + 7 + 7) // 8) * (length // 8 + 1) * rows  # 3 m16n8k8 per 8 outputs per k-step
    return nbytes, useful, issued


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    args = ap.parse_args()
    arms = {"audio_b200": F, "fftconvolve": _Fft()}
    try:
        import torchaudio.functional as TA

        TA.convolve(torch.zeros(1, 8, device="cuda"), torch.ones(1, 3, device="cuda"))
        arms["ta_tf32"] = _Cudnn(TA, True)
        arms["ta_fp32"] = _Cudnn(TA, False)
    except Exception as exc:  # noqa: BLE001
        print(f"reference arms unavailable: {exc}", file=sys.stderr)
    for name, x, y in workloads():
        with torch.no_grad():
            outs = {k: M.convolve(x, y) for k, M in arms.items()}  # warm-up, and the outputs compared
            times = {k: [] for k in arms}
            for _ in range(args.iters):
                for k, M in arms.items():
                    times[k].append(time_once(lambda: M.convolve(x, y)))
        t = median(times["audio_b200"])
        nbytes, useful, issued = counts(x, y, outs["audio_b200"])
        row = {"workload": name, "us": round(t, 1), "GB/s": round(nbytes / t * 1e-3, 1),
               "of_hbm_peak": round(nbytes / (t * 1e-6) / HBM_BYTES_PER_S, 3),
               "useful_TFLOP/s": round(useful / t * 1e-6, 1), "issued_TFLOP/s": round(issued / t * 1e-6, 1),
               "issued_of_tf32_peak": round(issued / (t * 1e-6) / TF32_FLOP_PER_S, 3)}
        for k in arms:
            if k != "audio_b200":
                row[f"{k}_us"] = round(median(times[k]), 1)
                row[f"max_abs_diff_{k}"] = float((outs["audio_b200"] - outs[k]).abs().max())
        print(json.dumps(row), flush=True)
        del outs

    # (f) forward + backward of (c): the gradients of both operands
    _, x, y = workloads()[2]
    up = torch.randn(x.shape[0], x.shape[1] + y.shape[1] - 1, device="cuda")

    def step(M, with_switch):
        xg, yg = x.clone().requires_grad_(), y.clone().requires_grad_()
        if with_switch:
            with audio_b200.differentiable(filtering=True):
                out = M.convolve(xg, yg)
        else:
            out = M.convolve(xg, yg)
        (out * up).sum().backward()
        return xg.grad, yg.grad

    garms = {k: (M, k in ("audio_b200", "fftconvolve")) for k, M in arms.items()}
    grads = {k: step(*v) for k, v in garms.items()}
    times = {k: [] for k in garms}
    for _ in range(max(args.iters // 3, 5)):
        for k, v in garms.items():
            times[k].append(time_once(lambda: step(*v)))
    t = median(times["audio_b200"])
    fwd, _, _ = counts(x, y, up)
    nbytes = fwd + 4 * x.shape[0] * (up.shape[1] + 2 * (x.shape[1] + y.shape[1]))
    row = {"workload": "(f) forward+backward of (c)", "us": round(t, 1), "GB/s": round(nbytes / t * 1e-3, 1),
           "of_hbm_peak": round(nbytes / (t * 1e-6) / HBM_BYTES_PER_S, 3)}
    for k in garms:
        if k != "audio_b200":
            row[f"{k}_us"] = round(median(times[k]), 1)
            row[f"grad_rel_diff_{k}"] = [float((o - r).abs().max() / r.abs().max().clamp_min(1e-30))
                                         for o, r in zip(grads["audio_b200"], grads[k])]
    print(json.dumps(row), flush=True)
    name, power = card()
    print(json.dumps({"card": name, "power_limit": power}))


if __name__ == "__main__":
    main()
