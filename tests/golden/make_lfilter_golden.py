#!/usr/bin/env python
"""Generate tests/golden/lfilter_ref_cases.npz, the IIR-filtering fixture (needs a pytorch/audio checkout named by
AUDIO_REFERENCE; run once):

    AUDIO_REFERENCE=/path/to/audio python tests/golden/make_lfilter_golden.py

The checkout's pure-Python recurrence runs on the CPU, so the signals are short.  All arrays are float32 from the
reference unless noted:
- ``x``: a seeded (2, 3, 600) signal at 0.5 rms with a burst past +-1 (exercises the clamp);
- ``lf_n{N}_{a,b}`` / ``lf_n{N}_c{0,1}``: 1-D coefficients of filter order N (Butterworth lowpass designs scaled so
  that a0 != 1) and lfilter(x, a, b, clamp) for N in ORDERS;
- ``lf2_{a,b}`` and ``lf2_b{0,1}_c{0,1}``: three filters of order 2 as 2-D coefficients, batching True (on x) and
  False (on x[:, 0]), clamp off and on;
- ``ff_c{0,1}``: filtfilt(x, a, b, clamp) with the order-3 coefficients;
- ``bq_{name}_{i}``: each biquad at its settings in BIQUADS, on x[0] at the setting's sample rate, and ``riaa_{sr}``;
- ``pre`` / ``de``: preemphasis and deemphasis of x (coeff 0.97);
- ``g_up``, ``g_x`` / ``g_a`` / ``g_b``: a seeded upstream gradient and the autograd gradients of
  sum(g_up * lfilter(x, lf2_a, lf2_b, clamp=True)), and ``gq_x``, ``gq_cutoff``, ``gq_Q`` those of
  sum(g_up[0, 0] * lowpass_biquad(x[0, 0], 16000, cutoff, Q)) with tensor cutoff_freq = 1000 and Q = 0.9;
- ``err_*``: the reference's error strings ("<exception type>: <message>").
"""
import os
import sys

import numpy as np
import torch
from scipy import signal

REF = os.environ["AUDIO_REFERENCE"]  # a pytorch/audio checkout at the pinned version
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(REF, "src"))
import torchaudio  # noqa: E402
import torchaudio.functional as RF  # noqa: E402

assert torchaudio.__file__.startswith(REF), torchaudio.__file__
from torchaudio.functional import filtering as _RFilt  # noqa: E402

# Without its compiled extension the checkout's recurrence loop subtracts in place from the FIR output, which the FIR
# node saved for backward, so autograd refuses; run the same loop on a copy (the outputs are unchanged).
if _RFilt._lfilter_core_loop is _RFilt._lfilter_core_generic_loop:
    _RFilt._lfilter_core_loop = lambda w, a, out: _RFilt._lfilter_core_generic_loop(w.clone(), a, out)

ORDERS = (0, 1, 2, 3, 5, 9)
# name: [(sample_rate, kwargs)]
BIQUADS = {
    "allpass": [(16000, dict(central_freq=1000.0, Q=0.707)), (44100, dict(central_freq=200.0, Q=2.0))],
    "band": [(16000, dict(central_freq=1000.0, Q=0.707)), (16000, dict(central_freq=3000.0, Q=3.0, noise=True))],
    "bandpass": [(16000, dict(central_freq=1000.0, Q=0.707)), (48000, dict(central_freq=500.0, Q=4.0,
                                                                           const_skirt_gain=True))],
    "bandreject": [(16000, dict(central_freq=1000.0, Q=0.707)), (44100, dict(central_freq=60.0, Q=5.0))],
    "bass": [(16000, dict(gain=6.0)), (44100, dict(gain=-10.0, central_freq=200.0, Q=1.2))],
    "equalizer": [(16000, dict(center_freq=1000.0, gain=6.0)), (48000, dict(center_freq=8000.0, gain=-9.0, Q=2.0))],
    "highpass": [(16000, dict(cutoff_freq=100.0)), (48000, dict(cutoff_freq=3000.0, Q=1.5))],
    "lowpass": [(16000, dict(cutoff_freq=1000.0)), (48000, dict(cutoff_freq=20.0, Q=2.0)),
                (16000, dict(cutoff_freq=100.0))],
    "treble": [(16000, dict(gain=6.0)), (44100, dict(gain=-4.0, central_freq=8000.0, Q=0.5))],
    "deemph": [(44100, {}), (48000, {})],
}


def _err(fn):
    try:
        fn()
    except Exception as exc:  # noqa: BLE001
        return f"{type(exc).__name__}: {exc}"
    return "ok"


def coeffs(order, scale=1.7):
    if order == 0:
        b, a = np.array([0.8]), np.array([1.0])
    else:
        b, a = signal.butter(order, 0.15)
    return (np.asarray(a) * scale).astype(np.float32), (np.asarray(b) * scale).astype(np.float32)


def main():
    rng = np.random.default_rng(2024)
    out = {}
    x = (0.5 * rng.standard_normal((2, 3, 600))).astype(np.float32)
    x[:, :, 200:260] *= 4.0  # a burst that drives the filters past +-1
    out["x"] = x
    xt = torch.from_numpy(x)
    for n in ORDERS:
        a, b = coeffs(n)
        out[f"lf_n{n}_a"], out[f"lf_n{n}_b"] = a, b
        for c in (0, 1):
            out[f"lf_n{n}_c{c}"] = RF.lfilter(xt, torch.from_numpy(a), torch.from_numpy(b), clamp=bool(c)).numpy()
    designs = [(signal.butter(2, 0.1), 1.0), (signal.butter(2, 0.3, btype="high"), 1.7),
               (signal.butter(1, (0.2, 0.4), btype="band"), 0.6)]
    b2 = np.stack([np.asarray(ba[0]) * s for ba, s in designs]).astype(np.float32)
    a2 = np.stack([np.asarray(ba[1]) * s for ba, s in designs]).astype(np.float32)
    out["lf2_a"], out["lf2_b"] = a2, b2
    at, bt = torch.from_numpy(a2), torch.from_numpy(b2)
    for c in (0, 1):
        out[f"lf2_b1_c{c}"] = RF.lfilter(xt, at, bt, clamp=bool(c), batching=True).numpy()
        out[f"lf2_b0_c{c}"] = RF.lfilter(xt[:, 0], at, bt, clamp=bool(c), batching=False).numpy()
    a3, b3 = coeffs(3)
    for c in (0, 1):
        out[f"ff_c{c}"] = RF.filtfilt(xt, torch.from_numpy(a3), torch.from_numpy(b3), clamp=bool(c)).numpy()
    for name, settings in BIQUADS.items():
        fn = getattr(RF, f"{name}_biquad")
        for i, (sr, kw) in enumerate(settings):
            out[f"bq_{name}_{i}"] = fn(xt[0], sr, **kw).numpy()
    for sr in (44100, 48000, 88200, 96000):
        out[f"riaa_{sr}"] = RF.riaa_biquad(xt[0], sr).numpy()
    out["pre"] = RF.preemphasis(xt, 0.97).numpy()
    out["de"] = RF.deemphasis(xt, 0.97).numpy()
    # gradients
    g = rng.standard_normal(x.shape).astype(np.float32)
    out["g_up"] = g
    xg, ag, bg = xt.clone().requires_grad_(), at.clone().requires_grad_(), bt.clone().requires_grad_()
    (RF.lfilter(xg, ag, bg, clamp=True) * torch.from_numpy(g)).sum().backward()
    out["g_x"], out["g_a"], out["g_b"] = xg.grad.numpy(), ag.grad.numpy(), bg.grad.numpy()
    xq = xt[0, 0].clone().requires_grad_()
    cut, q = torch.tensor(1000.0, requires_grad=True), torch.tensor(0.9, requires_grad=True)
    (RF.lowpass_biquad(xq, 16000, cut, q) * torch.from_numpy(g[0, 0])).sum().backward()
    out["gq_x"], out["gq_cutoff"], out["gq_Q"] = xq.grad.numpy(), cut.grad.numpy(), q.grad.numpy()
    # errors
    a1, b1 = torch.from_numpy(coeffs(2)[0]), torch.from_numpy(coeffs(2)[1])
    out["err_size"] = np.array(_err(lambda: RF.lfilter(xt, a1, b1[:2])))
    out["err_ndim"] = np.array(_err(lambda: RF.lfilter(xt, at[None], bt[None])))
    out["err_batches"] = np.array(_err(lambda: RF.lfilter(xt[:, :2], at, bt)))
    out["err_wave_ndim"] = np.array(_err(lambda: RF.lfilter(torch.tensor(0.5), at, bt)))
    out["err_riaa"] = np.array(_err(lambda: RF.riaa_biquad(xt[0], 16000)))
    out["err_deemph"] = np.array(_err(lambda: RF.deemph_biquad(xt[0], 16000)))
    path = os.path.join(HERE, "lfilter_ref_cases.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes,", len(out), "arrays")


if __name__ == "__main__":
    main()
