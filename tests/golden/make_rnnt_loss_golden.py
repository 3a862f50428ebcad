#!/usr/bin/env python
"""Generate tests/golden/rnnt_loss_ref_cases.npz, the rnnt_loss fixture (run once, with torchaudio installed at the
pinned reference version and AUDIO_REFERENCE naming a pytorch/audio checkout of it):

    AUDIO_REFERENCE=/path/to/audio python tests/golden/make_rnnt_loss_golden.py

torchaudio's rnnt_loss runs on the CPU here, the reference's parity target.  Stored:
- ``fx_<name>_*``: the reference's hand-worked fixtures (test/torchaudio_unittest/common_utils/rnnt_utils.py:
  B1_T2_U3_D5, B2_T4_U3_D3, and B1_T10_U3_D4 without the fused log-softmax) as arrays -- logits, targets, lengths,
  blank, fused -- with the reference CPU's costs and gradients;
- ``rc_<i>``: seeded recipes (tests/rnnt_loss_oracle.py:case_inputs) with ``fused_<i>``, ``clamp_<i>`` and the
  reference CPU's costs ``cost_<i>``; the full gradient ``grad_<i>`` for small cases, and for every case the
  reference's own error against the float64 oracle (``cerr_<i>`` max relative cost error, ``gerr_<i>`` max-abs
  gradient error), the bar the GPU must meet within a factor of two;
- ``nonfinite_cost``: the reference CPU's costs of a batch with a blank logit at -inf in one sequence (NaN there);
- ``err_<key>``: the reference's error strings ("<exception type>: <message>").
"""
import importlib.util
import os
import re
import sys

import numpy as np
import torch

REF = os.environ["AUDIO_REFERENCE"]
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import torchaudio  # noqa: E402
import torchaudio.functional as RF  # noqa: E402

import rnnt_loss_oracle as O  # noqa: E402

# rnnt_utils.py alone: the package around it needs test-only dependencies
_spec = importlib.util.spec_from_file_location(
    "rnnt_utils", os.path.join(REF, "test", "torchaudio_unittest", "common_utils", "rnnt_utils.py"))
rnnt_utils = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(rnnt_utils)

with open(os.path.join(REF, "version.txt")) as fh:
    PINNED = fh.read().strip()
assert torchaudio.__version__.split("+")[0] == PINNED.split("a")[0], (torchaudio.__version__, PINNED)

FULL_GRAD_MAX = 4096  # elements: larger cases store only the reference's error against the oracle

RECIPES = [  # (seed, B, maxT, maxU, V, blank, half, scale), fused, clamp
    ((10, 3, 7, 5, 6, -1, 0, 1.0), True, -1.0),
    ((11, 3, 7, 5, 6, 0, 0, 1.0), False, -1.0),
    ((12, 2, 6, 4, 29, 14, 0, 1.0), True, 0.05),
    ((13, 2, 6, 4, 29, 14, 0, 1.0), False, 0.01),
    ((14, 3, 5, 3, 7, -1, 1, 1.0), True, -1.0),
    ((15, 2, 1, 4, 3, -1, 0, 1.0), True, -1.0),
    ((16, 2, 4, 1, 5, -1, 0, 1.0), True, -1.0),
    ((17, 2, 4, 3, 1, -1, 0, 1.0), True, -1.0),
    ((20, 2, 150, 40, 32, -1, 0, 1.0), True, -1.0),
    ((21, 1, 400, 60, 16, -1, 0, 1.0), True, -1.0),
    ((22, 2, 150, 40, 32, -1, 1, 1.0), True, -1.0),
    ((23, 2, 100, 30, 29, 0, 0, 1.0), False, -1.0),
    ((24, 2, 60, 20, 1024, 7, 0, 2.0), True, 0.001),
]


def ref(logits, targets, tl, ul, blank, clamp, fused):
    x = torch.from_numpy(logits).requires_grad_()
    c = RF.rnnt_loss(x, torch.from_numpy(targets), torch.from_numpy(tl), torch.from_numpy(ul), blank=blank,
                     clamp=clamp, reduction="none", fused_log_softmax=fused)
    c.sum().backward()
    return c.detach().double().numpy(), x.grad.double().numpy()


def err(fn):
    try:
        fn()
    except Exception as e:  # noqa: BLE001
        msg = re.sub(r"^\w+, \S+:\d+, ", "", str(e).splitlines()[0])  # the C++ check's "<function>, <file>:<line>, "
        return f"{type(e).__name__}: {msg}"
    raise AssertionError("expected an error")


def main():
    out = {}
    fixtures = {
        "B1_T2_U3_D5": rnnt_utils.get_B1_T2_U3_D5_data()[0],
        "B2_T4_U3_D3": rnnt_utils.get_B2_T4_U3_D3_data()[0],
        "B1_T10_U3_D4": rnnt_utils.get_B1_T10_U3_D4_data(),
    }
    for name, d in fixtures.items():
        lg = d["logits"].detach().float().numpy()
        fused = d.get("fused_log_softmax", True)
        args = (d["targets"].numpy(), d["logit_lengths"].numpy(), d["target_lengths"].numpy())
        c, g = ref(lg, *args, d["blank"], -1.0, fused)
        out.update({f"fx_{name}_logits": lg, f"fx_{name}_targets": args[0], f"fx_{name}_tl": args[1],
                    f"fx_{name}_ul": args[2], f"fx_{name}_blank": np.array(d["blank"]),
                    f"fx_{name}_fused": np.array(fused), f"fx_{name}_cost": c, f"fx_{name}_grad": g})
        print(name, c)
    for i, (rc, fused, clamp) in enumerate(RECIPES):
        lg, tg, tl, ul = O.case_inputs(rc)
        c, g = ref(lg, tg, tl, ul, rc[5], clamp, fused)
        oc, og = O.rnnt_loss(lg, tg, tl, ul, rc[5], clamp, fused)
        out.update({f"rc_{i}": np.array(rc, dtype=np.float64), f"fused_{i}": np.array(fused),
                    f"clamp_{i}": np.array(clamp), f"cost_{i}": c,
                    f"cerr_{i}": np.array(np.max(np.abs(c - oc) / np.abs(oc))),
                    f"gerr_{i}": np.array(np.max(np.abs(g - og)))})
        if g.size <= FULL_GRAD_MAX:
            out[f"grad_{i}"] = g
        print(i, rc, fused, clamp, "cost err", out[f"cerr_{i}"], "grad err", out[f"gerr_{i}"])

    lg, tg, tl, ul = O.case_inputs((30, 3, 6, 4, 5, -1, 0, 1.0))
    lg[1, :, :, 4] = -np.inf  # every path of sequence 1 has probability 0
    out["nonfinite_cost"] = ref(lg, tg, tl, ul, -1, -1.0, True)[0]
    assert np.isnan(out["nonfinite_cost"][1]) and np.isfinite(out["nonfinite_cost"][[0, 2]]).all()

    lg, tg, tl, ul = (torch.from_numpy(a) for a in O.case_inputs((31, 2, 4, 3, 5, -1, 0, 1.0)))
    call = lambda **kw: lambda: RF.rnnt_loss(**{**dict(logits=lg, targets=tg, logit_lengths=tl,  # noqa: E731
                                                        target_lengths=ul), **kw})
    errors = {
        "reduction": call(reduction="avg"),
        "dtype_f64": call(logits=lg.double()),
        "dtype_bf16": call(logits=lg.bfloat16()),
        "targets_dtype": call(targets=tg.long()),
        "logit_lengths_dtype": call(logit_lengths=tl.long()),
        "target_lengths_dtype": call(target_lengths=ul.long()),
        "logits_contiguous": call(logits=lg.transpose(1, 2).contiguous().transpose(1, 2)),
        "targets_contiguous": call(targets=torch.cat([tg, tg], 1)[:, ::2]),
        "logits_dim": call(logits=lg[0]),
        "targets_dim": call(targets=tg[0]),
        "logit_lengths_dim": call(logit_lengths=tl[None]),
        "target_lengths_dim": call(target_lengths=ul[None]),
        "batch_logit_lengths": call(logit_lengths=tl[:1]),
        "batch_target_lengths": call(target_lengths=ul[:1]),
        "batch_targets": call(targets=tg[:1]),
        "blank": call(blank=5),
        "input_length": call(logit_lengths=tl - 1),
        "output_length": call(target_lengths=ul - 1),
        "target_length": call(targets=torch.cat([tg, tg], 1)),
    }
    for k, fn in errors.items():
        out[f"err_{k}"] = np.array(err(fn))
        print(k, out[f"err_{k}"])
    np.savez_compressed(os.path.join(HERE, "rnnt_loss_ref_cases.npz"), **out)


if __name__ == "__main__":
    main()
