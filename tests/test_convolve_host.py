"""Direct convolution without a GPU: the float64 oracle's direct form (tests/conv_oracle.py) against the reference
fixture (tests/golden/make_convolve_golden.py), the reference's errors that the Python surface raises before any
launch, the ABI statuses of b200a_convolve_run / b200a_convolve_backward, and the module surface."""
import ast
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import conv_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "convolve_ref_cases.npz")


@pytest.fixture(scope="module")
def ref():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def test_oracle_matches_fixture(ref):
    cases = [k[4:] for k in ref if k.startswith("out_")]
    assert len(cases) == 51
    for c in cases:
        x, y, g, mode = ref[f"x_{c}"], ref[f"y_{c}"], ref[f"g_{c}"], str(ref[f"mode_{c}"])
        scale = np.abs(x).max() * np.abs(y).max() * min(x.shape[-1], y.shape[-1])
        out = O.fftconvolve(x, y, mode, direct=True)
        assert out.shape == ref[f"out_{c}"].shape, c
        assert np.abs(out - ref[f"out_{c}"]).max() < 1e-5 * scale, c
        dx, dy = O.vjp(x, y, g, mode, direct=True)
        assert np.abs(dx - ref[f"gx_{c}"]).max() < 1e-5 * np.abs(g).max() * np.abs(y).sum(-1).max(), c
        assert np.abs(dy - ref[f"gy_{c}"]).max() < 1e-5 * np.abs(g).max() * np.abs(x).sum(-1).max() * 10, c


def test_reference_errors_are_recorded(ref):
    import audio_b200.functional as F
    import audio_b200.transforms as T

    for key, fn in (("err_ndim", lambda: F.convolve(torch.zeros(2, 3, 10), torch.zeros(3, 10))),
                    ("err_bcast", lambda: F.convolve(torch.zeros(3, 10), torch.zeros(2, 4))),
                    ("err_mode", lambda: F.convolve(torch.zeros(3, 10), torch.zeros(3, 4), "foo")),
                    ("err_module_mode", lambda: T.Convolve("foo"))):
        with pytest.raises(ValueError) as info:
            fn()
        assert f"ValueError: {info.value}" == str(ref[key]), key


def test_surface_rejects_cpu_and_other_dtypes():
    import audio_b200.functional as F

    with pytest.raises(RuntimeError, match="no CPU or ATen fallback"):
        F.convolve(torch.zeros(2, 10), torch.zeros(2, 3))
    with pytest.raises(RuntimeError, match="no CPU or ATen fallback"):
        F.convolve(torch.zeros(2, 10, dtype=torch.float64), torch.zeros(2, 3, dtype=torch.float64))


def test_switch_and_message():
    import audio_b200
    from audio_b200 import _plans

    assert "F.convolve, Convolve" in audio_b200.is_filtering_differentiable.__doc__
    assert "F.convolve, Convolve" in audio_b200.set_differentiable.__doc__
    with pytest.raises(RuntimeError, match=r"F\.convolve, Convolve.*differentiable\(filtering=True\)"):
        _plans._no_autograd(torch.zeros(1, requires_grad=True))


def test_surface():
    import audio_b200.functional as F
    import audio_b200.transforms as T
    from audio_b200 import _lib

    assert "convolve" in F.__all__ and "Convolve" in T.__all__
    assert T.Convolve().mode == "full" and T.Convolve("valid").mode == "valid"
    assert T.Convolve().state_dict() == {}
    assert _lib.CONVOLVE_MAX_TAPS == 4096


def test_reference_switch_covers_convolve():
    """B200A_REFERENCE=1 routes T.Convolve to the reference module (on the CPU, so the result is checkable here)."""
    code = ("import torch, audio_b200.transforms as T;"
            "m = T.Convolve('same');"
            "print(m(torch.ones(1, 5), torch.ones(1, 3)).tolist())")
    env = dict(os.environ, B200A_REFERENCE="1")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=root, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    got = np.array(ast.literal_eval(r.stdout.strip().splitlines()[-1]))
    assert np.allclose(got, [[2.0, 3.0, 3.0, 3.0, 2.0]], atol=1e-5)


# ---- the C ABI ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from audio_b200 import _lib

    return _lib.lib()


def _desc(**kw):
    from audio_b200 import _lib

    fake = 0x1000  # never dereferenced: every call below returns before a launch
    base = dict(n=1000, m=300, out_len=1299, start=0, rows=2, x_rows=2, y_rows=1, x_index=fake, y_index=fake,
                x_stride=1000, y_stride=300)
    base.update(kw)
    return _lib.FftconvolveDesc(**base)


def test_abi_statuses(lib):
    from audio_b200 import _lib

    fake = 0x1000
    ws_bytes, bw_bytes = lib.b200a_convolve_workspace_bytes, lib.b200a_convolve_backward_workspace_bytes
    run, bw = lib.b200a_convolve_run, lib.b200a_convolve_backward
    d = _desc()
    nb, nbb = ws_bytes(ctypes.byref(d)), bw_bytes(ctypes.byref(d))
    # K = 300: one filter row's fragments, ceil(307 / 8) = 39 k-steps of 32 float4, rounded up to 256 bytes
    assert nb == (39 * 32 * 16 + 255) // 256 * 256
    # the backward adds the filter-gradient partials: 2 rows x ceil(1007 / 2048) tiles x 300 taps
    assert nbb == nb + (2 * 1 * 300 * 4 + 255) // 256 * 256
    cap = _lib.CONVOLVE_MAX_TAPS
    at_cap = _desc(n=cap + 10, m=cap, out_len=2 * cap + 9, x_stride=cap + 10, y_stride=cap)
    assert ws_bytes(ctypes.byref(at_cap)) > 0 and bw_bytes(ctypes.byref(at_cap)) > 0
    over = _desc(n=cap + 10, m=cap + 1, out_len=2 * cap + 10, x_stride=cap + 10, y_stride=cap + 1)
    assert ws_bytes(ctypes.byref(over)) == 0 and bw_bytes(ctypes.byref(over)) == 0
    assert run(ctypes.byref(over), fake, fake, fake, fake, 1 << 40, None) == _lib.EUNSUPPORTED
    assert bw(ctypes.byref(over), fake, fake, fake, fake, fake, fake, 1 << 40, None) == _lib.EUNSUPPORTED
    swapped = _desc(n=cap + 1, m=cap + 10, out_len=2 * cap + 10, x_stride=cap + 1, y_stride=cap + 10)
    assert run(ctypes.byref(swapped), fake, fake, fake, fake, 1 << 40, None) == _lib.EUNSUPPORTED  # K = min(n, m)
    long = _desc(n=1 << 31, m=2, out_len=1, x_stride=1 << 31, y_stride=2)
    assert run(ctypes.byref(long), fake, fake, fake, fake, 1 << 40, None) == _lib.EUNSUPPORTED
    for bad in (dict(n=0), dict(m=0), dict(rows=-1), dict(x_rows=0), dict(y_rows=0), dict(out_len=-1),
                dict(start=-1), dict(start=1, out_len=1299), dict(x_stride=-1), dict(y_stride=-1)):
        assert run(ctypes.byref(_desc(**bad)), fake, fake, fake, fake, 1 << 40, None) == _lib.EINVAL, bad
        assert bw(ctypes.byref(_desc(**bad)), fake, fake, fake, fake, fake, fake, 1 << 40, None) == _lib.EINVAL, bad
        assert ws_bytes(ctypes.byref(_desc(**bad))) == 0 and bw_bytes(ctypes.byref(_desc(**bad))) == 0, bad
    assert run(None, fake, fake, fake, fake, 1 << 40, None) == _lib.EINVAL
    assert bw(None, fake, fake, fake, fake, fake, fake, 1 << 40, None) == _lib.EINVAL
    assert ws_bytes(None) == 0 and bw_bytes(None) == 0
    for i in range(4):  # x, y, out, workspace
        args = [fake] * 4
        args[i] = None
        assert run(ctypes.byref(d), *args, nb, None) == _lib.EINVAL, i
    for field in ("x_index", "y_index"):
        assert run(ctypes.byref(_desc(**{field: None})), fake, fake, fake, fake, nb, None) == _lib.EINVAL, field
    assert run(ctypes.byref(d), fake, fake, fake, fake, nb - 1, None) == _lib.EWORKSPACE
    assert run(ctypes.byref(_desc(rows=0)), None, None, None, None, 0, None) == _lib.OK  # nothing to enqueue
    assert run(ctypes.byref(_desc(out_len=0)), None, None, None, None, 0, None) == _lib.OK
    for i in range(6):  # x, y, grad, grad_x, grad_y, workspace
        args = [fake] * 6
        args[i] = None
        assert bw(ctypes.byref(d), *args, nbb, None) == _lib.EINVAL, i
    assert bw(ctypes.byref(d), fake, fake, fake, fake, fake, fake, nbb - 1, None) == _lib.EWORKSPACE
    assert bw(ctypes.byref(d), fake, fake, fake, fake, fake, fake, nb, None) == _lib.EWORKSPACE  # the forward's size
    assert bw(ctypes.byref(_desc(rows=0)), None, None, None, None, None, None, 0, None) == _lib.OK
