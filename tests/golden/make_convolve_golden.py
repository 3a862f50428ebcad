#!/usr/bin/env python
"""Generate tests/golden/convolve_ref_cases.npz, the direct-convolution fixture (needs a pytorch/audio checkout named by
AUDIO_REFERENCE; run once):

    AUDIO_REFERENCE=/path/to/audio python tests/golden/make_convolve_golden.py

Per case ``c`` in CASES (the FFT-convolution fixture's shapes plus filters of K = 1, 7, 8, 9, 15, 16 and 17 taps, at
the edges of the 8-wide k-steps; every mode), all arrays float32 from the reference's CPU convolve unless noted:
- ``x_c``, ``y_c``: the seeded operands; ``mode_c``: the mode (a string);
- ``out_c``: convolve(x, y, mode);
- ``g_c``: a seeded upstream gradient, and ``gx_c`` / ``gy_c``: the autograd gradients of sum(g * convolve(x, y));
- ``err_empty_{n}_{m}_{mode}``: the error for an empty operand;
- ``err_*``: the reference's other error strings ("<exception type>: <message>").
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
SHAPES.update({f"k{k}": ((2, 333), (2, k)) for k in (1, 7, 8, 9, 15, 16, 17)})
CASES = [(name, mode) for name in SHAPES for mode in ("full", "valid", "same")]


def err(fn):
    try:
        fn()
    except Exception as e:  # noqa: BLE001
        return f"{type(e).__name__}: {e}"
    raise AssertionError("expected an error")


def main():
    rng = np.random.default_rng(20261018)
    out = {}
    for name, mode in CASES:
        c = f"{name}_{mode}"
        xs, ys = SHAPES[name]
        x = torch.tensor(rng.standard_normal(xs), dtype=torch.float32, requires_grad=True)
        y = torch.tensor(rng.standard_normal(ys), dtype=torch.float32, requires_grad=True)
        r = RF.convolve(x, y, mode)
        g = torch.tensor(rng.standard_normal(tuple(r.shape)), dtype=torch.float32)
        (r * g).sum().backward()
        out[f"x_{c}"], out[f"y_{c}"], out[f"mode_{c}"] = x.detach().numpy(), y.detach().numpy(), np.array(mode)
        out[f"out_{c}"], out[f"g_{c}"] = r.detach().numpy(), g.numpy()
        out[f"gx_{c}"], out[f"gy_{c}"] = x.grad.numpy(), y.grad.numpy()
    for n, m in ((0, 5), (5, 0), (0, 1), (1, 0), (0, 0)):
        for mode in ("full", "valid", "same"):
            out[f"err_empty_{n}_{m}_{mode}"] = np.array(err(lambda: RF.convolve(torch.zeros(2, n), torch.ones(2, m), mode)))
    out["err_rows"] = np.array(err(lambda: RF.convolve(torch.zeros(0, 10), torch.zeros(0, 4))))
    out["err_rows_empty"] = np.array(err(lambda: RF.convolve(torch.zeros(0, 0), torch.zeros(0, 4))))
    out["err_rows_bcast"] = np.array(err(lambda: RF.convolve(torch.zeros(3, 0, 10), torch.zeros(3, 1, 4))))
    out["err_ndim"] = np.array(err(lambda: RF.convolve(torch.zeros(2, 3, 10), torch.zeros(3, 10))))
    out["err_bcast"] = np.array(err(lambda: RF.convolve(torch.zeros(3, 10), torch.zeros(2, 4))))
    out["err_mode"] = np.array(err(lambda: RF.convolve(torch.zeros(3, 10), torch.zeros(3, 4), "foo")))
    out["err_module_mode"] = np.array(err(lambda: torchaudio.transforms.Convolve("foo")))
    np.savez_compressed(os.path.join(HERE, "convolve_ref_cases.npz"), **out)


if __name__ == "__main__":
    main()
