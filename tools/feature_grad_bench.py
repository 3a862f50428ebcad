"""Forward + backward timing of the feature gradients (MFCC / LFCC / AmplitudeToDB) against torch's own CUDA autograd.

    python tools/feature_grad_bench.py [--steps 10] [--warmup 3] [--rounds 3]

Workloads (seeded inputs and upstream gradients, the same for both arms):
  - config 4: MFCC (n_fft 1024, hop 256, 80 mels, 40 coefficients) on a 2-D batch of 256 x 160000, batch-global top_db;
  - the log-mel loss at config 2: MelSpectrogram (n_fft 1024, hop 256, 80 mels) -> AmplitudeToDB(top_db=80) on
    256 x 160000;
  - LFCC at the reference's defaults (n_fft 400, 128 filters, 40 coefficients) on 64 x 48000.
The torch arm is torchaudio's transforms when they import, else the same op sequence written out.  The two arms run
alternately, --rounds times, each timed with CUDA events over --steps forward+backward steps; the table gives the median
ms per step and the max |difference| between the two gradients.  Last, the feature adjoint (b200audio::mfcc_backward)
is timed on its own at config 4, with its compulsory HBM traffic and the bandwidth that implies.
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
from audio_b200 import _lib, _ops  # noqa: E402
from audio_b200._plans import new_group_max  # noqa: E402
from bench import device_info  # noqa: E402


def _amplitude_to_db(x, top_db):
    """functional.amplitude_to_DB (functional.py:356-404) for power input, ref 1."""
    x_db = 10.0 * torch.log10(torch.clamp(x, min=1e-10))
    if top_db is not None:
        shape = x_db.size()
        packed = shape[-3] if x_db.dim() > 2 else 1
        x_db = x_db.reshape(-1, packed, shape[-2], shape[-1])
        x_db = torch.max(x_db, (x_db.amax(dim=(-3, -2, -1)) - top_db).view(-1, 1, 1, 1)).reshape(shape)
    return x_db


def torch_arm(kind, ours, dev):
    """torch CUDA autograd arm: torchaudio if installed, else its composition written out with our module's buffers."""
    try:
        import torchaudio.transforms as TA

        if kind == "mfcc":
            return TA.MFCC(16000, n_mfcc=40, melkwargs=dict(n_fft=1024, hop_length=256, n_mels=80)).to(dev), "torchaudio"
        if kind == "logmel":
            mel = TA.MelSpectrogram(16000, n_fft=1024, hop_length=256, n_mels=80).to(dev)
            db = TA.AmplitudeToDB(top_db=80.0)
            return (lambda x: db(mel(x))), "torchaudio"
        return TA.LFCC(16000).to(dev), "torchaudio"
    except Exception:  # noqa: BLE001
        pass

    def spec(x, n_fft, hop, window):
        s = torch.stft(x, n_fft, hop, n_fft, window, center=True, pad_mode="reflect", return_complex=True)
        return s.abs().pow(2.0)

    if kind == "mfcc":
        mel = ours.MelSpectrogram
        w, fb, dct = mel.spectrogram.window, mel.mel_scale.fb, ours.dct_mat

        def fn(x):
            m = torch.matmul(spec(x, 1024, 256, w).transpose(-1, -2), fb).transpose(-1, -2)
            return torch.matmul(_amplitude_to_db(m, 80.0).transpose(-1, -2), dct).transpose(-1, -2)
    elif kind == "logmel":
        w, fb = ours[0].spectrogram.window, ours[0].mel_scale.fb

        def fn(x):
            return _amplitude_to_db(torch.matmul(spec(x, 1024, 256, w).transpose(-1, -2), fb).transpose(-1, -2), 80.0)
    else:
        w, fb, dct = ours.Spectrogram.window, ours.filter_mat, ours.dct_mat

        def fn(x):
            f = torch.matmul(spec(x, 400, 200, w).transpose(-1, -2), fb).transpose(-1, -2)
            return torch.matmul(_amplitude_to_db(f, 80.0).transpose(-1, -2), dct).transpose(-1, -2)

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


def signal(rows, length, dev, seed):
    """Tones + noise at row levels over 60 dB with silent stretches, so that the top_db clamp fires."""
    gen = torch.Generator(device=dev).manual_seed(seed)
    t = torch.arange(length, device=dev) / 16000.0
    f = 100 + 3900 * torch.rand(rows, 1, device=dev, generator=gen)
    level = 10.0 ** (-3 * torch.rand(rows, 1, device=dev, generator=gen))
    x = level * (torch.sin(2 * torch.pi * f * t) + 0.05 * torch.randn(rows, length, device=dev, generator=gen))
    x[::7, length // 4: length // 2] = 0.0
    return x


def adjoint_alone(dev, steps):
    """b200audio::mfcc_backward at config 4 on its own: (ms, compulsory MB, GB/s)."""
    mod = T.MFCC(16000, n_mfcc=40, melkwargs=dict(n_fft=1024, hop_length=256, n_mels=80)).to(dev)
    x = signal(256, 160000, dev, 5)
    mel = mod.MelSpectrogram
    plan = mel._fused_plan(40, False, (10.0, 1e-10, 0.0))
    ws = plan.workspace(mel.spectrogram.window, mel.mel_scale.fb, mod.dct_mat)
    gmax = new_group_max(1, dev)
    feat = plan.run(ws, _lib.STAGE_FEAT, x, gmax, 256)
    m = plan.run(ws, _lib.STAGE_MEL, x)
    g = torch.randn(256, 626, 40, device=dev).transpose(1, 2).contiguous().transpose(1, 2)  # the strides autograd hands in
    desc_i, desc_f = plan._packed_desc()

    def call():
        return _ops.mfcc_backward(g, feat, m, gmax, ws, desc_i, desc_f, 256, 80.0)

    for _ in range(3):
        call()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        call()
    e1.record()
    e1.synchronize()
    ms = e0.elapsed_time(e1) / steps
    nbytes = 4 * (g.numel() + feat.numel() + m.numel() + m.numel())  # g, d, m read; g_m written
    return ms, nbytes / 1e6, nbytes / ms / 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda")
    info = device_info(0)
    print(f"# {info['name']}, power limit {info['power_limit_w']} W")
    rows = []
    for kind, batch, length in (("mfcc", 256, 160000), ("logmel", 256, 160000), ("lfcc", 64, 48000)):
        if kind == "mfcc":
            ours = T.MFCC(16000, n_mfcc=40, melkwargs=dict(n_fft=1024, hop_length=256, n_mels=80)).to(dev)
            fn, name = ours, "MFCC n_fft=1024 hop=256 n_mels=80 n_mfcc=40 (config 4)"
        elif kind == "logmel":
            ours = (T.MelSpectrogram(16000, n_fft=1024, hop_length=256, n_mels=80).to(dev), T.AmplitudeToDB(top_db=80.0))
            fn, name = (lambda x, o=ours: o[1](o[0](x))), "MelSpectrogram -> AmplitudeToDB(top_db=80) (config 2)"
        else:
            ours = T.LFCC(16000).to(dev)
            fn, name = ours, "LFCC reference defaults (n_fft=400, 128 filters, 40 coefficients)"
        ref, ref_name = torch_arm(kind, ours, dev)
        x = signal(batch, length, dev, batch + length).requires_grad_()
        with audio_b200.differentiable(features=True):
            g = torch.randn(fn(x).shape, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
            fn(x).backward(g)
            ga = x.grad.clone()
            x.grad = None
            ref(x).backward(g)
            diff = (ga - x.grad).abs().max().item()
            scale = x.grad.abs().max().item()
            t_ours, t_ref = [], []
            for _ in range(args.rounds):  # alternate the two arms
                t_ours.append(run(fn, x, g, args.steps, args.warmup))
                t_ref.append(run(ref, x, g, args.steps, args.warmup))
        row = {"workload": f"{name} on {batch}x{length}", "audio_b200_ms": statistics.median(t_ours),
               "audio_b200_ms_range": [min(t_ours), max(t_ours)], "torch_ms": statistics.median(t_ref),
               "torch_ms_range": [min(t_ref), max(t_ref)], "torch_arm": ref_name, "max_abs_grad_diff": diff,
               "max_abs_grad": scale}
        rows.append(row)
        print(json.dumps(row))
        del x, g, ga
        torch.cuda.empty_cache()
    ms, mb, gbs = adjoint_alone(dev, 50)
    adj = {"workload": "feature adjoint alone (mfcc_backward, config 4, clamp on)", "ms": ms, "compulsory_MB": mb,
           "GB_per_s": gbs}
    print(json.dumps(adj))
    print(json.dumps({"device": info["name"], "power_limit_w": info["power_limit_w"], "results": rows, "adjoint": adj}))


if __name__ == "__main__":
    main()
