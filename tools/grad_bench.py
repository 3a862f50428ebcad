"""Forward + backward timing of the waveform gradient against torch's own CUDA autograd.

    python tools/grad_bench.py [--steps 20] [--warmup 3] [--rounds 5]

Workloads (seeded inputs and upstream gradients, the same for both arms):
  - config 2 MelSpectrogram (16 kHz, n_fft 1024, hop 256, 80 mels) on 256 x 160000;
  - power-1 Spectrogram at n_fft 512 / 1024 / 2048, hop n_fft/4, on 64 x 48000.
The torch arm is torchaudio's transform when it imports, else the same F.pad / torch.stft / abs / pow / matmul chain.
The two arms run alternately, --rounds times, each timed with CUDA events over --steps forward+backward steps; the
table gives the median ms per step and the max |difference| between the two gradients.
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
from bench import device_info  # noqa: E402


def torch_chain(kind, n_fft, hop, n_mels, power, dev):
    """torch CUDA autograd arm: torchaudio if installed, else its composition written out."""
    try:
        import torchaudio.transforms as TA

        if kind == "mel":
            return TA.MelSpectrogram(16000, n_fft=n_fft, hop_length=hop, n_mels=n_mels, power=power).to(dev), "torchaudio"
        return TA.Spectrogram(n_fft=n_fft, hop_length=hop, power=power).to(dev), "torchaudio"
    except Exception:  # noqa: BLE001
        pass
    window = torch.hann_window(n_fft, device=dev)
    fb = T.MelSpectrogram(16000, n_fft=n_fft, hop_length=hop, n_mels=n_mels).mel_scale.fb.to(dev) if kind == "mel" else None

    def fn(x):
        xp = torch.nn.functional.pad(x.unsqueeze(1), (n_fft // 2, n_fft // 2), mode="reflect").squeeze(1)
        s = torch.stft(xp, n_fft, hop, n_fft, window, center=False, return_complex=True).abs()
        s = s if power == 1.0 else s.pow(power)
        return torch.matmul(s.transpose(-1, -2), fb).transpose(-1, -2) if fb is not None else s

    return fn, "torch.stft chain"


def run(fn, x, g, steps, warmup):
    def step():
        x.grad = None
        fn(x).backward(g)

    for _ in range(warmup):
        step()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        step()
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
    workloads = [("mel", 1024, 256, 80, 2.0, 256, 160000)] + [("spec", n, n // 4, 0, 1.0, 64, 48000) for n in (512, 1024, 2048)]
    rows = []
    for kind, n_fft, hop, n_mels, power, batch, length in workloads:
        gen = torch.Generator(device=dev).manual_seed(n_fft)
        x = torch.randn(batch, length, device=dev, generator=gen).requires_grad_()
        if kind == "mel":
            ours = T.MelSpectrogram(16000, n_fft=n_fft, hop_length=hop, n_mels=n_mels, power=power).to(dev)
        else:
            ours = T.Spectrogram(n_fft=n_fft, hop_length=hop, power=power).to(dev)
        ref, ref_name = torch_chain(kind, n_fft, hop, n_mels, power, dev)
        with audio_b200.differentiable():
            shape = ours(x).shape
            g = torch.randn(shape, device=dev, generator=gen)
            ours(x).backward(g)
            ga = x.grad.clone()
            x.grad = None
            ref(x).backward(g)
            diff = (ga - x.grad).abs().max().item()
            scale = x.grad.abs().max().item()
            t_ours, t_ref = [], []
            for _ in range(args.rounds):  # alternate the two arms
                t_ours.append(run(ours, x, g, args.steps, args.warmup))
                t_ref.append(run(ref, x, g, args.steps, args.warmup))
        name = (f"MelSpectrogram n_fft={n_fft} hop={hop} n_mels={n_mels}" if kind == "mel" else
                f"Spectrogram power=1 n_fft={n_fft} hop={hop}") + f" on {batch}x{length}"
        row = {"workload": name, "audio_b200_ms": statistics.median(t_ours), "audio_b200_ms_range": [min(t_ours), max(t_ours)],
               "torch_ms": statistics.median(t_ref), "torch_ms_range": [min(t_ref), max(t_ref)], "torch_arm": ref_name,
               "max_abs_grad_diff": diff, "max_abs_grad": scale}
        rows.append(row)
        print(json.dumps(row))
    print(json.dumps({"device": info["name"], "power_limit_w": info["power_limit_w"], "results": rows}))


if __name__ == "__main__":
    main()
