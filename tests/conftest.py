import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def _load(name):
    with np.load(os.path.join(GOLDEN, name)) as z:
        return {k: z[k] for k in z.files}


@pytest.fixture(scope="session")
def librosa_transforms():
    return _load("librosa_transforms.npz")


@pytest.fixture(scope="session")
def librosa_melfb():
    return _load("librosa_melfb.npz")


@pytest.fixture(scope="session")
def ref_cases():
    return _load("ref_cases.npz")


@pytest.fixture(scope="session")
def ref_integers():
    return _load("ref_integers.npz")


def assert_close(actual, expected, rtol, atol, what=""):
    """|a - e| <= atol + rtol * |e| elementwise (torch.testing / unittest assertEqual rule)."""
    cplx = np.iscomplexobj(actual) or np.iscomplexobj(expected)
    a = np.asarray(actual, dtype=np.complex128 if cplx else np.float64)
    e = np.asarray(expected, dtype=np.complex128 if cplx else np.float64)
    assert a.shape == e.shape, f"{what}: shape {a.shape} vs {e.shape}"
    err = np.abs(a - e)
    tol = atol + rtol * np.abs(e)
    bad = err > tol
    if bad.any():
        i = np.unravel_index(np.argmax(err - tol), err.shape)
        raise AssertionError(
            f"{what}: {bad.sum()} / {bad.size} elements out of tolerance (rtol={rtol}, atol={atol}); "
            f"worst at {i}: actual={a[i]!r} expected={e[i]!r} |diff|={err[i]:.3e}"
        )


def scaled_tol_close(actual, expected, rel=1e-4, what=""):
    """The parity rule of SURVEY.md 8(c): |a-e| <= rel*|e| + rel*rms(e)."""
    e = np.asarray(expected)
    rms = float(np.sqrt(np.mean(np.abs(e) ** 2))) if e.size else 0.0
    assert_close(actual, expected, rtol=rel, atol=rel * rms, what=what)
