#!/usr/bin/env python
"""Time SpecAugment masking on the GPU against the same masking as torch ops (tests/specaugment_oracle.py, the
reference's op sequence) on the same GPU, in the same process.

Workload: the recipes' feature batch, 64 utterances x 1600 frames x 80 mels, given as the (B, n_mels, T) transpose of
a contiguous (B, T, n_mels) tensor.
  (a) SpecAugment(2, 100, 2, 27, p=0.2) with the default mean fill: forward, and forward + backward of the input
      gradient (upstream gradient of ones times a random tensor, so nothing folds away);
  (b) the recipes' TrainTransform chain: FrequencyMasking(27) twice, TimeMasking(100, p=0.2) twice, forward.
Per arm: the median of CUDA-event times over `reps` calls after `warmup` calls; GB/s against the byte count from the
shapes (N float32 elements: (a) forward 3 passes of 4N bytes -- mean, read, write -- and backward 4 more -- read g,
write the masked gradient, and the mean's gradient read and written back; (b) 4 modules x 2 passes); whether ours and
the torch ops give bit-equal outputs (and gradients) from the same seed on the timed inputs; the card's name and power
limit, read in the same run.

    python tools/specaugment_bench.py [--reps 50] [--warmup 10] [--out specaugment_bench.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import audio_b200.transforms as T  # noqa: E402
import specaugment_oracle as O  # noqa: E402

B, TIME, MELS = 64, 1600, 80


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda")
    x = torch.randn(B, TIME, MELS, generator=torch.Generator().manual_seed(0)).to(dev).transpose(1, 2)
    g = torch.randn(x.shape, device=dev)
    n = x.numel()
    rows = []

    def arm(name, ns, passes, fn):
        ms = timed(fn, args.reps, args.warmup)
        rows.append({"arm": name, "impl": ns, "ms": round(ms, 4), "GB/s": round(passes * 4 * n / ms / 1e6, 1)})

    def spec(ns):
        return ns.SpecAugment(2, 100, 2, 27, p=0.2)

    def chain(ns):
        mods = [ns.FrequencyMasking(27), ns.FrequencyMasking(27), ns.TimeMasking(100, p=0.2),
                ns.TimeMasking(100, p=0.2)]

        def run(y):
            for m in mods:
                y = m(y)
            return y
        return run

    xg = x.detach().clone().requires_grad_(True)
    for label, ns in (("ours", T), ("torch ops", O.ORACLE)):
        m, c = spec(ns), chain(ns)
        with torch.no_grad():
            arm("(a) SpecAugment forward", label, 3, lambda: m(x))

        def fwd_bwd():
            xg.grad = None
            m(xg).backward(g)
        arm("(a) SpecAugment forward + backward", label, 7, fwd_bwd)
        with torch.no_grad():
            arm("(b) TrainTransform chain forward", label, 8, lambda: c(x))

    same = {}
    for key, make in (("spec", spec), ("chain", chain)):
        outs = []
        for ns in (T, O.ORACLE):
            torch.manual_seed(5)
            xi = x.detach().clone().requires_grad_(key == "spec")
            y = make(ns)(xi)
            grad = None
            if key == "spec":
                y.backward(g)
                grad = xi.grad
            outs.append((y.detach(), grad))
        (ya, ga), (yb, gb) = outs
        same[key] = {"output_bit_equal": bool(torch.equal(ya.view(torch.int32), yb.view(torch.int32))),
                     "strides_equal": ya.stride() == yb.stride()}
        if ga is not None:
            same[key]["grad_max_rel"] = float(((ga - gb).abs().max() / gb.abs().max()).item())
    result = {"card": card(), "shape": [B, MELS, TIME], "elements": n, "rows": rows, "checks": same}
    for r in rows:
        print(f"{r['arm']:38s} {r['impl']:10s} {r['ms']:8.4f} ms {r['GB/s']:8.1f} GB/s")
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
