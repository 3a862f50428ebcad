"""A/B timing of library builds in sub-processes: C2 mel, Spectrogram, C5 512/256, MFCC.

    python tools/ab_time.py NAME=VALUE[,NAME=VALUE] ...     e.g.  - B200A_LIB=/tmp/parent/libb200audio.so
Each argument is one run with those environment variables set ("-" = no change)."""
import json
import os
import subprocess
import sys

CHILD = r"""
import sys, json, statistics, warnings
sys.path.insert(0, ".")
import torch
import audio_b200.transforms as T
dev = "cuda:0"
x = torch.randn(256, 160000, device=dev)
def t(fn, iters=20, blocks=5):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(blocks):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters): fn()
        e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) / iters)
    return statistics.median(ts)
out = {}
with warnings.catch_warnings():
    warnings.simplefilter("ignore")
    mods = {"mel1024": T.MelSpectrogram(16000, n_fft=1024, hop_length=256, n_mels=80),
            "spec1024": T.Spectrogram(n_fft=1024, hop_length=256),
            "mel512": T.MelSpectrogram(16000, n_fft=512, hop_length=128, n_mels=80),
            "mel256": T.MelSpectrogram(16000, n_fft=256, hop_length=64, n_mels=80),
            "spec256": T.Spectrogram(n_fft=256, hop_length=64),
            "mel2048": T.MelSpectrogram(16000, n_fft=2048, hop_length=512, n_mels=80),
            "mfcc": T.MFCC(16000, n_mfcc=40, melkwargs=dict(n_fft=1024, hop_length=256, n_mels=80))}
with torch.inference_mode():
    for k, m in mods.items():
        m = m.to(dev)
        out[k] = round(t(lambda: m(x)) * 1e3, 1)
print(json.dumps(out))
"""

for spec in sys.argv[1:] or ["-"]:
    env = dict(os.environ)
    if spec != "-":
        for kv in spec.split(","):
            k, v = kv.split("=", 1)
            env[k] = os.path.abspath(v) if k == "B200A_LIB" else v
    r = subprocess.run([sys.executable, "-c", CHILD], env=env, capture_output=True, text=True)
    print(spec, r.stdout.strip() or r.stderr[-400:], flush=True)
