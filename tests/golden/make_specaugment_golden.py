#!/usr/bin/env python
"""Generate tests/golden/specaugment_ref_cases.npz, the SpecAugment masking fixture (needs a pytorch/audio checkout
named by AUDIO_REFERENCE; run once, on the CPU):

    AUDIO_REFERENCE=/path/to/audio python tests/golden/make_specaugment_golden.py

Per case ``i``, from the reference's CPU masking under ``torch.manual_seed(100 + i)``:
- ``case_i``: a repr of {"x": input spec, "op": call} (tests/specaugment_oracle.py: make_input, run_case);
- ``out_i``: the float32 output values; ``stride_i``: its strides; ``same_i``: 1 when the call returned its input;
- ``next_i``: the next ``torch.rand(4)`` after the call, which pins how much of the generator the call consumed.
Also ``err_k`` with ``errcase_k``: the reference's error strings ("<exception type>: <message>").
"""
import os
import sys

import numpy as np
import torch

REF = os.environ["AUDIO_REFERENCE"]  # a pytorch/audio checkout at the pinned version
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(REF, "src"))
sys.path.insert(0, os.path.dirname(HERE))
import torchaudio  # noqa: E402
import torchaudio.functional as RF  # noqa: E402
import torchaudio.transforms as RT  # noqa: E402

import specaugment_oracle as O  # noqa: E402

assert torchaudio.__file__.startswith(REF), torchaudio.__file__

A = {"shape": (2, 8, 12), "seed": 1}                  # (batch, freq, time)
B = {"shape": (2, 16, 6), "seed": 2, "view": "t"}      # the recipes' (B, T, n_mels).transpose(1, 2)
C = {"shape": (2, 2, 6, 10), "seed": 3}               # 4-D
D = {"shape": (6, 10), "seed": 4}                     # 2-D
E = {"shape": (2, 5, 12), "seed": 5, "view": "step"}   # a sliced step on time
P = {"shape": (2, 10, 2, 6), "seed": 6, "view": "perm"}  # 4-D with the channel dimension innermost

CASES = [
    (A, ("iid", 5, 0.0, 2, 1.0)),
    (A, ("iid", 5, -1.5, 1, 1.0)),
    (B, ("iid", 5, ("t", 0.7), 1, 1.0)),
    (B, ("iid", 5, ("t", 0.7), 2, 0.2)),
    (B, ("iid", 5, 0.0, 2, 0.2)),
    (A, ("iid", 40, 0.0, 2, 1.0)),           # mask_param > size: negative starts
    (A, ("iid", 40, ("t", 2.0), 1, 1.0)),
    (A, ("iid", 0, 0.0, 2, 1.0)),            # nothing drawn, the input returned
    (A, ("iid", 1, 0.0, 1, 1.0)),
    (A, ("iid", 5, 0.0, 2, 0.0)),            # p = 0: nothing drawn
    (C, ("iid", 7, 3.0, 3, 0.2)),
    (C, ("iid", 4, ("t", 2.0), 2, 1.0)),
    (E, ("iid", 4, 1.0, 2, 1.0)),
    (E, ("iid", 4, ("t", 1.0), 1, 1.0)),
    (D, ("axis", 5, 0.0, 1, 1.0)),
    (D, ("axis", 5, 0.0, 0, 0.2)),
    (A, ("axis", 5, 2.5, 2, 0.2)),
    (B, ("axis", 40, 0.0, 2, 1.0)),
    (B, ("axis", 4, 0.0, 1, 1.0)),
    (C, ("axis", 3, 0.0, 3, 1.0)),
    (A, ("axis", 0, 0.0, 1, 1.0)),
    (E, ("axis", 4, 1.0, 1, 1.0)),
    (B, ("freq", 5, False, 0.0)),
    (B, ("freq", 5, True, ("t", 0.3))),
    (A, ("freq", 4, False, ("t", 0.5))),
    (B, ("time", 10, False, 0.2, 0.0)),
    (C, ("time", 10, True, 1.0, 1.5)),
    (B, ("spec", 2, 10, 2, 5, True, 1.0, False)),
    (B, ("spec", 2, 10, 2, 5, True, 0.2, False)),
    (B, ("spec", 2, 10, 2, 5, False, 1.0, False)),
    (A, ("spec", 2, 10, 2, 5, True, 1.0, True)),
    (A, ("spec", 2, 10, 2, 5, False, 0.2, True)),
    (A, ("spec", 0, 10, 0, 5, True, 1.0, False)),  # no masks: the input returned
    (A, ("spec", 1, 10, 0, 5, True, 1.0, False)),
    (C, ("spec", 6, 4, 6, 3, True, 1.0, False)),
    (D, ("spec", 2, 5, 2, 4, True, 1.0, False)),   # 2-D: the shared-mask path
    (A, ("spec", 3, 5, 3, 4, False, 0.0, False)),  # p = 0: every mask skipped
    (P, ("spec", 2, 50, 2, 50, True, 1.0, False)),
    (E, ("spec", 2, 4, 2, 3, True, 1.0, False)),
]

ERRORS = [
    (D, ("iid", 5, 0.0, 1, 1.0)),
    (A, ("iid", 5, 0.0, 0, 1.0)),
    (A, ("iid", 5, 0.0, 2, 1.5)),
    ({"shape": (16,), "seed": 7}, ("axis", 5, 0.0, 0, 1.0)),
    (A, ("axis", 5, 0.0, 3, 1.0)),
    (A, ("axis", 5, 0.0, 1, -0.5)),
    (A, ("time", 5, False, -0.1, 0.0)),
    ({"shape": (16,), "seed": 7}, ("spec", 1, 5, 0, 4, True, 1.0, False)),
]


def main():
    ns = O.SimpleNamespace(mask_along_axis_iid=RF.mask_along_axis_iid, mask_along_axis=RF.mask_along_axis,
                           FrequencyMasking=RT.FrequencyMasking, TimeMasking=RT.TimeMasking,
                           SpecAugment=RT.SpecAugment)
    out = {}
    for i, (xs, op) in enumerate(CASES):
        x = O.make_input(xs)
        torch.manual_seed(100 + i)
        y = O.run_case(ns, op, x)
        out[f"case_{i}"] = np.array(repr({"x": xs, "op": op}))
        out[f"out_{i}"] = y.detach().numpy().astype(np.float32)
        out[f"stride_{i}"] = np.array(y.stride(), dtype=np.int64)
        out[f"same_{i}"] = np.array(int(y is x))
        out[f"next_{i}"] = torch.rand(4).numpy()
    for k, (xs, op) in enumerate(ERRORS):
        try:
            O.run_case(ns, op, O.make_input(xs))
        except Exception as e:  # noqa: BLE001
            out[f"err_{k}"] = np.array(f"{type(e).__name__}: {e}")
        else:
            raise AssertionError(f"expected an error from {op}")
        out[f"errcase_{k}"] = np.array(repr({"x": xs, "op": op}))
    np.savez_compressed(os.path.join(HERE, "specaugment_ref_cases.npz"), **out)
    print(f"{len(CASES)} cases, {len(ERRORS)} errors")


if __name__ == "__main__":
    main()
