"""Timing of the spectrogram gradient of InverseSpectrogram against torch's own CUDA autograd through torch.istft.

    python tools/istft_grad_bench.py [--steps 20] [--warmup 3] [--rounds 5]

Workloads (seeded complex spectrograms and upstream gradients, the same for both arms), hop n_fft/4, 160 000 samples:
  - n_fft 1024 (256 x 513 x 626, the fused kernel), n_fft 512 (256 x 257 x 1251, fused), n_fft 2048 (64 rows, the
    composition path).
Per workload:
  - forward + backward per step, ours and torch.istft under autograd alternately, --rounds times, CUDA events over
    --steps steps; the median ms per step and the max |difference| between the two gradients;
  - the backward alone (b200audio::istft_backward) and the forward COMPLEX Spectrogram of the same geometry (which
    writes the same complex64 array) in the same call, alternately; and the bytes the backward moves (g read once,
    grad_spec written once) over its time.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import audio_b200  # noqa: E402
import audio_b200.transforms as T  # noqa: E402
from audio_b200 import _ops  # noqa: E402
from audio_b200._plans import FrontendPlan  # noqa: E402
from bench import device_info  # noqa: E402


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda")
    info = device_info(0)
    print(f"# {info['name']}, power limit {info['power_limit_w']} W")
    length = 160000
    rows_out = []
    for n_fft, batch in ((1024, 256), (512, 256), (2048, 64)):
        hop = n_fft // 4
        frames = 1 + length // hop
        bins = n_fft // 2 + 1
        gen = torch.Generator(device=dev).manual_seed(n_fft)
        z = torch.complex(torch.randn(batch, bins, frames, device=dev, generator=gen),
                          torch.randn(batch, bins, frames, device=dev, generator=gen)).requires_grad_()
        g = torch.randn(batch, hop * (frames - 1), device=dev, generator=gen)  # the returned samples
        window = torch.hann_window(n_fft, device=dev)
        ours = T.InverseSpectrogram(n_fft=n_fft, hop_length=hop).to(dev)

        def ref(s):
            return torch.istft(s, n_fft, hop, window=window, center=True)

        def step(fn):
            z.grad = None
            fn(z).backward(g)

        with audio_b200.differentiable(inverse=True):
            step(ours)
            ga = z.grad.clone()
            step(ref)
            diff = (ga - z.grad).abs().max().item()
            scale = z.grad.abs().max().item()
            t_ours, t_ref = [], []
            for _ in range(args.rounds):  # alternate the two arms
                t_ours.append(timed(lambda: step(ours), args.steps, args.warmup))
                t_ref.append(timed(lambda: step(ref), args.steps, args.warmup))
        # the backward alone against the forward COMPLEX Spectrogram of the same geometry
        plan = FrontendPlan(FrontendPlan.make_desc(n_fft, n_fft, hop, 0, True, "reflect", True, False, False, 2.0))
        ws = plan.workspace(ours.window, None, None)
        desc_i, desc_f = plan._packed_desc()
        spec = T.Spectrogram(n_fft=n_fft, hop_length=hop, power=None).to(dev)
        x = torch.randn(batch, length, device=dev, generator=gen)
        t_bwd, t_fwd = [], []
        with torch.no_grad():
            for _ in range(args.rounds):
                t_bwd.append(timed(lambda: _ops.istft_backward(g, ws, desc_i, desc_f, n_fft // 2, frames), args.steps,
                                   args.warmup))
                t_fwd.append(timed(lambda: spec(x), args.steps, args.warmup))
        moved = 4 * g.numel() + 8 * batch * frames * bins
        row = {"workload": f"InverseSpectrogram n_fft={n_fft} hop={hop} on {batch}x{bins}x{frames}",
               "audio_b200_ms": statistics.median(t_ours), "audio_b200_ms_range": [min(t_ours), max(t_ours)],
               "torch_ms": statistics.median(t_ref), "torch_ms_range": [min(t_ref), max(t_ref)],
               "max_abs_grad_diff": diff, "max_abs_grad": scale,
               "backward_ms": statistics.median(t_bwd), "backward_ms_range": [min(t_bwd), max(t_bwd)],
               "forward_complex_spectrogram_ms": statistics.median(t_fwd),
               "forward_complex_spectrogram_ms_range": [min(t_fwd), max(t_fwd)],
               "backward_over_forward": statistics.median(t_bwd) / statistics.median(t_fwd),
               "backward_bytes": moved, "backward_gb_per_s": moved / statistics.median(t_bwd) / 1e6}
        rows_out.append(row)
        print(json.dumps(row))
        del z, g, x
        torch.cuda.empty_cache()
    print(json.dumps({"device": info["name"], "power_limit_w": info["power_limit_w"], "results": rows_out}))


if __name__ == "__main__":
    main()
