"""SpecAugment masking without a GPU: the reference's ValueErrors (raised before any device work or random draw), the
explicit rejection of CPU inputs and foreign fills, the surface, and the C ABI's argument statuses."""
import ast
import ctypes
import os

import numpy as np
import pytest
import torch

import specaugment_oracle as O
from audio_b200 import _lib

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "specaugment_ref_cases.npz")


def _ns():
    import audio_b200.functional as F
    import audio_b200.transforms as T

    return O.SimpleNamespace(mask_along_axis_iid=F.mask_along_axis_iid, mask_along_axis=F.mask_along_axis,
                             FrequencyMasking=T.FrequencyMasking, TimeMasking=T.TimeMasking, SpecAugment=T.SpecAugment)


def test_reference_errors_before_device_work():
    with np.load(GOLDEN) as z:
        ref = {k: z[k] for k in z.files}
    k = 0
    while f"err_{k}" in ref:
        case = ast.literal_eval(str(ref[f"errcase_{k}"]))
        x = O.make_input(case["x"])
        state = torch.get_rng_state()
        with pytest.raises(ValueError) as e:
            O.run_case(_ns(), case["op"], x)
        assert f"ValueError: {e.value}" == str(ref[f"err_{k}"])
        assert torch.equal(torch.get_rng_state(), state), case
        k += 1


def test_cpu_input_raises_before_drawing():
    ns = _ns()
    x = torch.randn(2, 8, 12)
    for op in (("iid", 5, 0.0, 2, 1.0), ("axis", 5, 0.0, 1, 1.0), ("spec", 2, 5, 2, 4, True, 1.0, False),
               ("spec", 2, 5, 2, 4, False, 1.0, True)):
        state = torch.get_rng_state()
        with pytest.raises(RuntimeError, match="no CPU or ATen fallback"):
            O.run_case(ns, op, x)
        assert torch.equal(torch.get_rng_state(), state), op


def test_skipped_masks_return_the_input_on_any_device():
    ns = _ns()
    x = torch.randn(2, 8, 12)
    assert ns.mask_along_axis_iid(x, 0, 0.0, 2) is x
    assert ns.mask_along_axis(x, 5, 0.0, 1, p=0.0) is x
    assert ns.SpecAugment(0, 5, 0, 4)(x) is x


def test_surface():
    import audio_b200.functional as F
    import audio_b200.transforms as T

    assert {"mask_along_axis", "mask_along_axis_iid"} <= set(F.__all__)
    assert {"FrequencyMasking", "TimeMasking", "SpecAugment"} <= set(T.__all__)
    assert T.FrequencyMasking.__constants__ == ["mask_param", "axis", "iid_masks", "p"]
    assert T.SpecAugment.__constants__ == ["n_time_masks", "time_mask_param", "n_freq_masks", "freq_mask_param",
                                           "iid_masks", "p", "zero_masking"]
    fm, tm = T.FrequencyMasking(27), T.TimeMasking(100, p=0.2)
    assert (fm.mask_param, fm.axis, fm.iid_masks, fm.p) == (27, 1, False, 1.0)
    assert (tm.mask_param, tm.axis, tm.iid_masks, tm.p) == (100, 2, False, 0.2)
    sa = T.SpecAugment(2, 100, 2, 27)
    assert (sa.iid_masks, sa.p, sa.zero_masking) == (True, 1.0, False)


def _desc(**kw):
    f = dict(rows0=2, rows1=1, freq=8, time=12, n_masks=1, fill=0.0)
    f.update(kw)
    d = _lib.MaskDesc(f["rows0"], f["rows1"], f["freq"], f["time"], (ctypes.c_int64 * 4)(96, 0, 12, 1),
                      (ctypes.c_int64 * 4)(96, 0, 12, 1), f["n_masks"], f["fill"])
    return d


def test_c_abi_statuses():
    lib = _lib.lib()
    assert ctypes.sizeof(_lib.MaskSpec) == 40 and ctypes.sizeof(_lib.MaskDesc) == 104
    d = _desc()
    need = lib.b200a_mask_workspace_bytes(ctypes.byref(d))
    assert need >= 1024 * 8
    p = ctypes.c_void_p(256)  # never dereferenced: every call below fails its checks first
    shared = (_lib.MaskSpec * 1)(_lib.MaskSpec(_lib.MASK_AXIS_TIME, 0, 2, 5, None, None))
    run, bwd = lib.b200a_mask_run, lib.b200a_mask_backward
    assert run(None, shared, p, p, None, p, need, None) == _lib.EINVAL
    assert run(ctypes.byref(d), None, p, p, None, p, need, None) == _lib.EINVAL  # n_masks 1, no table
    assert run(ctypes.byref(d), shared, None, p, None, p, need, None) == _lib.EINVAL
    assert run(ctypes.byref(d), shared, p, None, None, p, need, None) == _lib.EINVAL
    assert run(ctypes.byref(d), shared, p, p, None, None, need, None) == _lib.EINVAL
    assert run(ctypes.byref(d), shared, p, p, None, p, need - 1, None) == _lib.EWORKSPACE
    assert bwd(ctypes.byref(d), shared, p, None, None, p, need, None) == _lib.EINVAL  # nothing to produce
    assert bwd(ctypes.byref(d), shared, p, p, None, p, need - 1, None) == _lib.EWORKSPACE
    for bad in (dict(rows0=-1), dict(rows1=-1), dict(freq=-1), dict(time=-1), dict(n_masks=-1)):
        b = _desc(**bad)
        assert lib.b200a_mask_workspace_bytes(ctypes.byref(b)) == 0, bad
        assert run(ctypes.byref(b), shared, p, p, None, p, need, None) == _lib.EINVAL, bad
    for spec in (_lib.MaskSpec(2, 0, 2, 5, None, None), _lib.MaskSpec(-1, 0, 2, 5, None, None),
                 _lib.MaskSpec(_lib.MASK_AXIS_FREQ, 0, 0, 0, 256, 256),  # per-row mask with mask_param 0
                 _lib.MaskSpec(_lib.MASK_AXIS_FREQ, 3, 0, 0, 256, None)):  # per-row mask without start draws
        t = (_lib.MaskSpec * 1)(spec)
        assert run(ctypes.byref(d), t, p, p, None, p, need, None) == _lib.EINVAL
    assert lib.b200a_mask_workspace_bytes(None) == 0
