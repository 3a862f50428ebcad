"""Timing of the waveform gradient of Resample against torch's own CUDA autograd through the reference's op sequence.

    python tools/resample_grad_bench.py [--steps 20] [--warmup 3] [--rounds 5]

Workloads (seeded waveforms and upstream gradients, the same for both arms):
  - config 3: 1024 x 220 500 samples, 44.1 -> 16 kHz kaiser;
  - 16 -> 44.1 kHz on 256 x 160 000 samples; 48 -> 16 kHz on 256 x 480 000 samples.
Per workload:
  - forward + backward per step, ours (Resample inside differentiable(resample=True)) and torch's autograd through
    torchaudio's _apply_sinc_resample_kernel with the same cached kernel (F.pad + conv1d + transpose + reshape + slice;
    written out with torch ops when torchaudio does not import) alternately, --rounds times, CUDA events over --steps
    steps; the median ms per step and the max |difference| between the two gradients (cuDNN's conv1d runs in TF32 when
    torch.backends.cudnn.allow_tf32 is set, the default; the value is printed);
  - the backward alone (b200audio::resample_backward) and the forward Resample alone in the same call, alternately; and
    the compulsory bytes of the backward (g read once, grad_x written once) over its time.
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
from audio_b200._bookkeeping import resample_len  # noqa: E402
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


def torch_arm():
    """(name, fn(waveform, orig, new, gcd, kernel, width)) of the reference's op sequence under torch autograd."""
    try:
        from torchaudio.functional.functional import _apply_sinc_resample_kernel

        return "torchaudio _apply_sinc_resample_kernel", _apply_sinc_resample_kernel
    except Exception:  # noqa: BLE001
        pass

    def chain(waveform, orig, new, gcd, kernel, width):
        o, n = orig // gcd, new // gcd
        rows, length = waveform.shape
        x = torch.nn.functional.pad(waveform, (width, width + o))
        y = torch.nn.functional.conv1d(x[:, None], kernel, stride=o)
        y = y.transpose(1, 2).reshape(rows, -1)
        return y[..., :resample_len(length, o, n)]

    return "F.pad + conv1d chain", chain


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda")
    info = device_info(0)
    arm_name, ref_fn = torch_arm()
    print(f"# {info['name']}, power limit {info['power_limit_w']} W; torch arm: {arm_name}, "
          f"cudnn.allow_tf32={torch.backends.cudnn.allow_tf32}")
    rows_out = []
    for orig, new, method, batch, length in ((44100, 16000, "sinc_interp_kaiser", 1024, 220500),
                                             (16000, 44100, "sinc_interp_hann", 256, 160000),
                                             (48000, 16000, "sinc_interp_hann", 256, 480000)):
        mod = T.Resample(orig, new, resampling_method=method).to(dev)
        o, n = orig // mod.gcd, new // mod.gcd
        out_len = resample_len(length, o, n)
        gen = torch.Generator(device=dev).manual_seed(orig + new)
        x = torch.randn(batch, length, device=dev, generator=gen).requires_grad_()
        g = torch.randn(batch, out_len, device=dev, generator=gen)

        def ref(t):
            return ref_fn(t, orig, new, mod.gcd, mod.kernel, mod.width)

        def step(fn):
            x.grad = None
            fn(x).backward(g)

        with audio_b200.differentiable(resample=True):
            step(mod)
            ga = x.grad.clone()
            step(ref)
            diff = (ga - x.grad).abs().max().item()
            scale = x.grad.abs().max().item()
            del ga
            t_ours, t_ref = [], []
            for _ in range(args.rounds):  # alternate the two arms
                t_ours.append(timed(lambda: step(mod), args.steps, args.warmup))
                t_ref.append(timed(lambda: step(ref), args.steps, args.warmup))
        x.grad = None
        # the backward alone against the forward alone
        plan = mod._plan
        plan.workspace(mod.kernel)
        bws = plan.backward_workspace()
        xd = x.detach()
        t_bwd, t_fwd = [], []
        with torch.no_grad():
            for _ in range(args.rounds):
                t_bwd.append(timed(lambda: _ops.resample_backward(g, bws, o, n, mod.width, length), args.steps,
                                   args.warmup))
                t_fwd.append(timed(lambda: mod(xd), args.steps, args.warmup))
        moved = 4 * (g.numel() + x.numel())
        row = {"workload": f"Resample {orig}->{new} {method} on {batch}x{length}",
               "audio_b200_ms": statistics.median(t_ours), "audio_b200_ms_range": [min(t_ours), max(t_ours)],
               "torch_ms": statistics.median(t_ref), "torch_ms_range": [min(t_ref), max(t_ref)],
               "torch_arm": arm_name, "max_abs_grad_diff": diff, "max_abs_grad": scale,
               "backward_ms": statistics.median(t_bwd), "backward_ms_range": [min(t_bwd), max(t_bwd)],
               "forward_ms": statistics.median(t_fwd), "forward_ms_range": [min(t_fwd), max(t_fwd)],
               "backward_over_forward": statistics.median(t_bwd) / statistics.median(t_fwd),
               "backward_bytes": moved, "backward_gb_per_s": moved / statistics.median(t_bwd) / 1e6}
        rows_out.append(row)
        print(json.dumps(row))
        del x, g, xd
        torch.cuda.empty_cache()
    print(json.dumps({"device": info["name"], "power_limit_w": info["power_limit_w"], "results": rows_out}))


if __name__ == "__main__":
    main()
