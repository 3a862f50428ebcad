"""InverseMelScale on the GPU: forward, and forward + backward, at the config-2 shape (256 rows x 80 mels x 626 frames ->
513 bins), timed with CUDA events, against the same minimum-norm answer written with torch ops on the device
(P = pinv(fb^T) once in float64, then relu(P @ m) -- the reference's own lstsq refuses this underdetermined system on
CUDA).  Prints the compulsory bytes, the achieved bandwidth, and the card name and power limit read in the same run.

    python tools/inverse_mel_bench.py [--rows 256] [--iters 50]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import audio_b200  # noqa: E402
import audio_b200.transforms as T  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data-sheet HBM3 bandwidth


def timed(fn, iters, warmup=5):
    for _ in range(warmup):
        fn()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(iters):
        start.record()
        fn()
        stop.record()
        stop.synchronize()
        times.append(start.elapsed_time(stop) * 1e3)
    times.sort()
    return times[len(times) // 2]  # median, microseconds


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=20)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=256)
    ap.add_argument("--mels", type=int, default=80)
    ap.add_argument("--frames", type=int, default=626)
    ap.add_argument("--n-stft", type=int, default=513)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    torch.manual_seed(0)
    mod = T.InverseMelScale(a.n_stft, a.mels, 16000).cuda()
    # frame-major (what MelSpectrogram returns), positive
    mel = torch.rand(a.rows, a.frames, a.mels, device="cuda").transpose(1, 2)
    pinv = torch.linalg.pinv(mod.fb.double().T).float()  # (n_stft, n_mels)

    def ours():
        with torch.no_grad():
            return mod(mel)

    def dense():
        return torch.relu(pinv @ mel)

    up = torch.randn(a.rows, a.n_stft, a.frames, device="cuda")

    def ours_fb():
        x = mel.detach().requires_grad_()
        with audio_b200.differentiable(features=True):
            mod(x).backward(up)

    def dense_fb():
        x = mel.detach().requires_grad_()
        torch.relu(pinv @ x).backward(up)

    diff = (ours() - dense()).abs().max().item() / dense().abs().max().item()
    bytes_in, bytes_out = mel.numel() * 4, a.rows * a.frames * a.n_stft * 4
    rows = []
    for label, fn, nbytes in (("forward", ours, bytes_in + bytes_out), ("forward (torch dense)", dense, bytes_in + bytes_out),
                              ("forward + backward", ours_fb, None), ("forward + backward (torch dense)", dense_fb, None)):
        us = timed(fn, a.iters)
        rows.append({"what": label, "us": round(us, 1),
                     "GB_per_s": None if nbytes is None else round(nbytes / us / 1e3, 1)})
    name, power = card()
    print(f"card: {name}, power limit {power}")
    print(f"shape: {a.rows} rows x {a.mels} mels x {a.frames} frames -> {a.n_stft} bins; "
          f"compulsory forward bytes {bytes_in / 1e6:.1f} MB in + {bytes_out / 1e6:.1f} MB out, floor "
          f"{(bytes_in + bytes_out) / HBM_BYTES_PER_S * 1e6:.0f} us at {HBM_BYTES_PER_S / 1e12:.2f} TB/s")
    print(f"max |ours - dense| / max|dense| = {diff:.2e}")
    print(f"{'what':36s} {'median us':>10s} {'GB/s':>8s}")
    for r in rows:
        print(f"{r['what']:36s} {r['us']:10.1f} {'' if r['GB_per_s'] is None else r['GB_per_s']:>8}")
    print(json.dumps({"card": name, "power_limit": power, "rows": rows, "rel_diff": diff}))


if __name__ == "__main__":
    main()
