#!/usr/bin/env python
"""Time models.decoder.cuda_ctc_decoder on the GPU against torchaudio's cuda_ctc_decoder.

Workloads (CTC-like emissions: log-softmax of N(0, 2) logits, blank boosted by 8 on 60 % of the frames and one
non-blank token boosted by 6 on the others; float32, every row at full length):
  bpe        B 32, T 500,  V 500,   beam 10,  nbest 10, threshold 0.95  (the reference tutorial's setting)
  chars      B 64, T 1500, V 32,    beam 10,  nbest 1,  threshold 0.95
  noskip     B 32, T 500,  V 500,   beam 10,  nbest 1,  threshold 1.0   (every frame a step)
  largevocab B 4,  T 300,  V 32000, beam 10,  nbest 1,  threshold 0.95
  widebeam   B 8,  T 500,  V 5000,  beam 128, nbest 1,  threshold 0.95
Per workload: a host clock around `reps` calls that end in a device synchronise (each call returns host objects), after
warm-up, for ours and, with --torchaudio, torchaudio's; how many rows' hypotheses equal torchaudio's (tokens and bit-equal scores, order
free among bit-equal scores); the card's name and power limit.  --profile instead writes the kernel time per call from
torch.profiler.

    python tools/ctc_decoder_bench.py [--reps 10] [--out ctc_decoder_bench.json] [--profile] [--torchaudio]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audio_b200.models.decoder import cuda_ctc_decoder  # noqa: E402

WORKLOADS = {  # B, T, V, beam, nbest, threshold
    "bpe": (32, 500, 500, 10, 10, 0.95),
    "chars": (64, 1500, 32, 10, 1, 0.95),
    "noskip": (32, 500, 500, 10, 1, 1.0),
    "largevocab": (4, 300, 32000, 10, 1, 0.95),
    "widebeam": (8, 500, 5000, 128, 1, 0.95),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def inputs(B, T, V, seed=0):
    g = torch.Generator().manual_seed(seed)
    logits = 2 * torch.randn(B, T, V, generator=g)
    runs = torch.rand(B, T, generator=g) < 0.6
    logits[..., 0] += runs * 8.0
    tok = torch.randint(1, V, (B, T), generator=g)
    logits.scatter_add_(2, tok[..., None], (~runs)[..., None].float() * 6.0)
    return torch.log_softmax(logits, -1).cuda(), torch.full((B,), T, dtype=torch.int32).cuda()


def timed(fn, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps


def canon(hs):
    return sorted((h.score.view(torch.int32).item(), tuple(h.tokens.tolist())) for h in hs)


def profile_split(dec, lp, n):
    from torch.profiler import ProfilerActivity, profile

    for _ in range(2):
        dec(lp, n)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            dec(lp, n)
        torch.cuda.synchronize()
    split = {"decode": 0.0, "other": 0.0}
    for e in prof.key_averages():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        split["decode" if "ctc_decode_kernel" in e.key else "other"] += e.device_time_total / 5
    return {k: round(v, 2) for k, v in split.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--torchaudio", action="store_true",
                    help="also time torchaudio's decoder on the whole batch (its batched calls failed with an illegal "
                         "address on an H100 with torchaudio 2.11; see DESIGN §3.19)")
    a = ap.parse_args()
    ref_decoder = None
    if a.torchaudio:
        try:
            from torchaudio.models.decoder import cuda_ctc_decoder as ref_decoder
        except Exception:  # noqa: BLE001
            pass
    res = {"card": card(), "workloads": {}}
    for name in a.workloads.split(","):
        B, T, V, beam, nbest, thr = WORKLOADS[name]
        lp, n = inputs(B, T, V)
        vocab = [str(i) for i in range(V)]
        dec = cuda_ctc_decoder(vocab, nbest=nbest, beam_size=beam, blank_skip_threshold=thr)
        r = {"shape": [B, T, V], "beam": beam, "nbest": nbest, "threshold": thr}
        if a.profile:
            r["kernel_us_per_call"] = profile_split(dec, lp, n)
            res["workloads"][name] = r
            print(name, json.dumps(r), flush=True)
            continue
        r["ours_ms"] = timed(lambda: dec(lp, n), a.reps) * 1e3
        if ref_decoder is not None:
            ref = ref_decoder(vocab, nbest=nbest, beam_size=beam, blank_skip_threshold=thr)
            r["torchaudio_ms"] = timed(lambda: ref(lp, n), a.reps) * 1e3
            r["speedup_vs_torchaudio"] = r["torchaudio_ms"] / r["ours_ms"]
            ours, theirs = dec(lp, n), ref(lp, n)
            r["rows_equal_to_torchaudio"] = sum(int(canon(o) == canon(t)) for o, t in zip(ours, theirs))
            r["rows"] = B
        res["workloads"][name] = r
        print(name, json.dumps(r), flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
