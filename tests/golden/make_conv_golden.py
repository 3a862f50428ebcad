#!/usr/bin/env python
"""Generate tests/golden/conv_ref_cases.npz, the FFT-convolution fixture (needs a pytorch/audio checkout named by
AUDIO_REFERENCE; run once):

    AUDIO_REFERENCE=/path/to/audio python tests/golden/make_conv_golden.py

Per case ``c`` in CASES (every mode; N < M, N == M, N > M; 1-sample operands; 1-D, 2-D and 4-D inputs; broadcasts
both ways), all arrays float32 from the reference's CPU fftconvolve unless noted:
- ``x_c``, ``y_c``: the seeded operands; ``mode_c``: the mode (a string);
- ``out_c``: fftconvolve(x, y, mode);
- ``g_c``: a seeded upstream gradient, and ``gx_c`` / ``gy_c``: the autograd gradients of sum(g * fftconvolve(x, y));
- ``empty_{n}_{m}_{mode}``: the output length for an empty operand, or ``err_empty_{n}_{m}_{mode}`` its error;
- ``err_*``: the reference's error strings ("<exception type>: <message>").
"""
import os
import sys

import numpy as np
import torch

REF = os.environ["AUDIO_REFERENCE"]  # a pytorch/audio checkout at the pinned version
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(REF, "src"))
import torchaudio  # noqa: E402
import torchaudio.functional as RF  # noqa: E402

assert torchaudio.__file__.startswith(REF), torchaudio.__file__

SHAPES = {
    "n_gt_m": ((2, 900), (2, 130)),
    "n_lt_m": ((2, 130), (2, 900)),
    "n_eq_m": ((3, 300), (3, 300)),
    "one_x": ((2, 1), (2, 50)),
    "one_y": ((2, 50), (2, 1)),
    "one_one": ((2, 1), (2, 1)),
    "d1": ((700,), (60,)),
    "d4": ((2, 1, 3, 400), (1, 2, 3, 90)),
    "bcast_xy": ((3, 1, 500), (1, 4, 70)),
    "bcast_yx": ((1, 4, 70), (3, 1, 500)),
}
CASES = [(name, mode) for name in SHAPES for mode in ("full", "valid", "same")]


def err(fn):
    try:
        fn()
    except Exception as e:  # noqa: BLE001
        return f"{type(e).__name__}: {e}"
    raise AssertionError("expected an error")


def main():
    rng = np.random.default_rng(20261017)
    out = {}
    for name, mode in CASES:
        c = f"{name}_{mode}"
        xs, ys = SHAPES[name]
        x = torch.tensor(rng.standard_normal(xs), dtype=torch.float32, requires_grad=True)
        y = torch.tensor(rng.standard_normal(ys), dtype=torch.float32, requires_grad=True)
        r = RF.fftconvolve(x, y, mode)
        g = torch.tensor(rng.standard_normal(tuple(r.shape)), dtype=torch.float32)
        (r * g).sum().backward()
        out[f"x_{c}"], out[f"y_{c}"], out[f"mode_{c}"] = x.detach().numpy(), y.detach().numpy(), np.array(mode)
        out[f"out_{c}"], out[f"g_{c}"] = r.detach().numpy(), g.numpy()
        out[f"gx_{c}"], out[f"gy_{c}"] = x.grad.numpy(), y.grad.numpy()
    for n, m in ((0, 5), (5, 0), (0, 1), (1, 0), (0, 0)):
        for mode in ("full", "valid", "same"):
            try:
                out[f"empty_{n}_{m}_{mode}"] = np.array(RF.fftconvolve(torch.zeros(2, n), torch.ones(2, m), mode).shape)
            except RuntimeError as e:
                out[f"err_empty_{n}_{m}_{mode}"] = np.array(f"RuntimeError: {e}")
    out["err_ndim"] = np.array(err(lambda: RF.fftconvolve(torch.zeros(2, 3, 10), torch.zeros(3, 10))))
    out["err_bcast"] = np.array(err(lambda: RF.fftconvolve(torch.zeros(3, 10), torch.zeros(2, 4))))
    out["err_mode"] = np.array(err(lambda: RF.fftconvolve(torch.zeros(3, 10), torch.zeros(3, 4), "foo")))
    out["err_module_mode"] = np.array(err(lambda: torchaudio.transforms.FFTConvolve("foo")))
    np.savez_compressed(os.path.join(HERE, "conv_ref_cases.npz"), **out)


if __name__ == "__main__":
    main()
