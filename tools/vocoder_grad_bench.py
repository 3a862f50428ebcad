"""Timing of the spectrogram gradient of TimeStretch and the waveform gradient of PitchShift against torch's own CUDA
autograd through the reference's op sequence.

    python tools/vocoder_grad_bench.py [--steps 20] [--warmup 3] [--rounds 5]

Workloads (seeded inputs and upstream gradients, the same for both arms):
  - TimeStretch at 256 x 257 x 1251 (10 s at 16 kHz, n_fft 512, hop 128), rates 0.8 and 1.3: forward + backward per
    step, ours (inside differentiable(vocoder=True)) and torch's autograd through torchaudio.functional.phase_vocoder
    (written out with torch ops when torchaudio does not import) alternately, --rounds times, CUDA events over --steps
    steps; the median ms per step.  Then the backward alone (b200audio::phase_vocoder_backward) and the forward kernel
    alone, alternately, and the backward's compulsory bytes 8 bins rows (2 Fo + 2 Fi) -- g and o read, X read, grad_X
    written -- over its time;
  - PitchShift at 64 x 48 000 samples, n_steps +4 and -3: forward + backward per step, ours against torch's autograd
    through torchaudio.functional.pitch_shift (or the op sequence written out), alternately.
"""
import argparse
import json
import math
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import audio_b200  # noqa: E402
import audio_b200.functional as F  # noqa: E402
from audio_b200 import _ops  # noqa: E402
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


def _phase_vocoder_chain(spec, rate, pa):
    """The published phase-vocoder op sequence in torch ops (used when torchaudio does not import)."""
    shape = spec.size()
    spec = spec.reshape((-1,) + tuple(shape[-2:]))
    grid = torch.arange(0, spec.size(-1), rate, device=spec.device, dtype=spec.real.dtype)
    padded = torch.nn.functional.pad(spec, [0, 2])
    z0, z1 = padded.index_select(-1, grid.long()), padded.index_select(-1, (grid + 1).long())
    dphi = z1.angle() - z0.angle() - pa
    dphi = dphi - 2 * math.pi * torch.round(dphi / (2 * math.pi)) + pa
    phase = torch.cumsum(torch.cat([spec[..., :1].angle(), dphi[..., :-1]], dim=-1), -1)
    alpha = grid % 1.0
    out = torch.polar(alpha * z1.abs() + (1 - alpha) * z0.abs(), phase)
    return out.reshape(shape[:-2] + out.shape[1:])


def torch_arms():
    """(name, phase_vocoder, pitch_shift) of the reference under torch autograd."""
    try:
        import torchaudio.functional as TAF

        return "torchaudio", TAF.phase_vocoder, TAF.pitch_shift
    except Exception:  # noqa: BLE001
        pass

    def pitch_shift(x, sr, n_steps):
        n_fft, hop = 512, 128
        rate = 2.0 ** (-float(n_steps) / 12)
        win = torch.hann_window(n_fft, device=x.device)
        spec = torch.stft(x, n_fft, hop, n_fft, win, center=True, pad_mode="reflect", return_complex=True)
        pa = torch.linspace(0, math.pi * hop, spec.shape[-2], device=x.device)[..., None]
        y = torch.istft(_phase_vocoder_chain(spec, rate, pa), n_fft, hop, n_fft, win, length=int(round(x.shape[-1] / rate)))
        y = _torch_resample(y, int(sr / rate), sr)
        n = y.shape[-1]
        return y[..., :x.shape[-1]] if n > x.shape[-1] else torch.nn.functional.pad(y, [0, x.shape[-1] - n])

    return "torch op sequence", _phase_vocoder_chain, pitch_shift


def _torch_resample(x, orig, new):
    """conv1d polyphase resampling with this package's (reference-identical) sinc taps, under torch autograd."""
    from audio_b200._bookkeeping import resample_len
    from audio_b200._constants import sinc_resample_kernel

    gcd = math.gcd(orig, new)
    kernel, width = sinc_resample_kernel(orig, new, gcd, 6, 0.99, "sinc_interp_hann", None, x.device, x.dtype)
    o, n = orig // gcd, new // gcd
    rows, length = x.shape
    y = torch.nn.functional.conv1d(torch.nn.functional.pad(x, (width, width + o))[:, None], kernel, stride=o)
    return y.transpose(1, 2).reshape(rows, -1)[..., :resample_len(length, o, n)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda")
    info = device_info(0)
    arm_name, ref_pv, ref_ps = torch_arms()
    print(f"# {info['name']}, power limit {info['power_limit_w']} W; torch arm: {arm_name}")
    rows_out = []
    rows, bins, frames = 256, 257, 1251
    gen = torch.Generator(device=dev).manual_seed(1251)
    spec = torch.complex(torch.randn(rows, frames, bins, device=dev, generator=gen),
                         torch.randn(rows, frames, bins, device=dev, generator=gen)).transpose(1, 2)
    pa = torch.linspace(0, math.pi * 128, bins, device=dev)[..., None]
    for rate in (0.8, 1.3):
        fo = int(math.ceil(frames / rate))
        g = torch.complex(torch.randn(rows, bins, fo, device=dev, generator=gen),
                          torch.randn(rows, bins, fo, device=dev, generator=gen))
        x = spec.detach().requires_grad_()

        def step(fn):
            x.grad = None
            fn(x, rate, pa).backward(g)

        with audio_b200.differentiable(vocoder=True):
            step(F.phase_vocoder)
            t_ours, t_ref = [], []
            for _ in range(args.rounds):
                t_ours.append(timed(lambda: step(F.phase_vocoder), args.steps, args.warmup))
                t_ref.append(timed(lambda: step(ref_pv), args.steps, args.warmup))
        x.grad = None
        spec3 = spec.detach()
        out, _ = F._phase_vocoder_run(spec3, rate, pa.reshape(-1).contiguous())
        t_bwd, t_fwd = [], []
        with torch.no_grad():
            for _ in range(args.rounds):
                t_bwd.append(timed(lambda: _ops.phase_vocoder_backward(spec3, out, g, rate), args.steps, args.warmup))
                t_fwd.append(timed(lambda: F._phase_vocoder_run(spec3, rate, pa.reshape(-1)), args.steps, args.warmup))
        moved = 8 * bins * rows * (2 * fo + 2 * frames)
        row = {"workload": f"TimeStretch rate {rate} on {rows}x{bins}x{frames}",
               "audio_b200_ms": statistics.median(t_ours), "audio_b200_ms_range": [min(t_ours), max(t_ours)],
               "torch_ms": statistics.median(t_ref), "torch_ms_range": [min(t_ref), max(t_ref)], "torch_arm": arm_name,
               "backward_ms": statistics.median(t_bwd), "backward_ms_range": [min(t_bwd), max(t_bwd)],
               "forward_kernel_ms": statistics.median(t_fwd), "forward_kernel_ms_range": [min(t_fwd), max(t_fwd)],
               "backward_over_forward": statistics.median(t_bwd) / statistics.median(t_fwd),
               "backward_bytes": moved, "backward_gb_per_s": moved / statistics.median(t_bwd) / 1e6}
        rows_out.append(row)
        print(json.dumps(row))
        del x, g, out
        torch.cuda.empty_cache()
    del spec
    wave = torch.randn(64, 48000, device=dev, generator=gen)
    gw = torch.randn(64, 48000, device=dev, generator=gen)
    for n_steps in (4, -3):
        x = wave.clone().requires_grad_()

        def step(fn):
            x.grad = None
            fn(x, 16000, n_steps).backward(gw)

        with audio_b200.differentiable(vocoder=True):
            step(F.pitch_shift)
            t_ours, t_ref = [], []
            for _ in range(args.rounds):
                t_ours.append(timed(lambda: step(F.pitch_shift), args.steps, args.warmup))
                t_ref.append(timed(lambda: step(ref_ps), args.steps, args.warmup))
        row = {"workload": f"PitchShift n_steps {n_steps:+d} on 64x48000",
               "audio_b200_ms": statistics.median(t_ours), "audio_b200_ms_range": [min(t_ours), max(t_ours)],
               "torch_ms": statistics.median(t_ref), "torch_ms_range": [min(t_ref), max(t_ref)], "torch_arm": arm_name}
        rows_out.append(row)
        print(json.dumps(row))
    print(json.dumps({"device": info["name"], "power_limit_w": info["power_limit_w"], "results": rows_out}))


if __name__ == "__main__":
    main()
