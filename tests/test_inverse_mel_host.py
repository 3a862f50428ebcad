"""InverseMelScale without a GPU: the float64 oracle against the reference's outputs and gradients
(tests/golden/make_inverse_mel_golden.py), the host-side plan of the C ABI against a dense float64 factorisation, and
the module surface."""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import scaled_tol_close
from inverse_mel_oracle import inverse_mel_scale, inverse_mel_scale_vjp

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CONFIGS = ("c201_64_8k", "c513_128_16k", "c513_80_16k", "c1025_128_22k_slaney", "c257_40_16k_band", "c201_40_16k")


@pytest.fixture(scope="module")
def inv_ref():
    with np.load(os.path.join(GOLDEN, "inverse_mel_ref_cases.npz")) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("name", CONFIGS)
def test_oracle_matches_reference(inv_ref, name):
    fb = inv_ref[f"{name}_fb"]
    for kind in ("speech", "rand"):
        scaled_tol_close(inverse_mel_scale(inv_ref[f"{name}_{kind}_in"], fb), inv_ref[f"{name}_{kind}_out"], 1e-5,
                         f"{name} {kind}")
    got = inverse_mel_scale_vjp(inv_ref[f"{name}_grad_in"], fb, inv_ref[f"{name}_grad_up"])
    scaled_tol_close(got, inv_ref[f"{name}_grad"], 1e-4, f"{name} grad")


def test_reference_raises_on_rank_deficient_banks(inv_ref):
    for name in ("s201_128_16k", "s65_128_16k"):
        assert "does not have full rank" in str(inv_ref[f"{name}_gels"])
        for drv in ("gelsy", "gelsd", "gelss"):
            assert str(inv_ref[f"{name}_{drv}"]) == "ok"


# ---------------- the host-side plan --------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from audio_b200 import _lib

    return _lib.lib()


def _plan(lib, fb, driver=0):
    from audio_b200 import _lib

    fb = np.ascontiguousarray(fb, dtype=np.float32)
    n_stft, n_mels = fb.shape
    nbytes = lib.b200a_inverse_mel_plan_bytes(n_stft, n_mels)
    blob = np.zeros(nbytes // 4, dtype=np.int32)
    bw, piv = ctypes.c_int32(), ctypes.c_int32()
    rc = lib.b200a_inverse_mel_plan(fb.ctypes.data, n_stft, n_mels, driver, blob.ctypes.data, nbytes, ctypes.byref(bw),
                                    ctypes.byref(piv))
    assert nbytes == 4 * (4 + n_mels * (_lib.INVERSE_MEL_MAX_BANDWIDTH + 3) + n_stft * (_lib.INVERSE_MEL_MAX_BANDWIDTH + 3))
    return rc, blob, bw.value, piv.value


def _unpack(blob, n_stft, n_mels):
    from audio_b200 import _lib

    kb = _lib.INVERSE_MEL_MAX_BANDWIDTH
    f = blob.view(np.float32)
    o = 4
    lsub = f[o:o + n_mels * kb].reshape(n_mels, kb); o += n_mels * kb
    inv_d = f[o:o + n_mels]; o += n_mels
    bfirst = blob[o:o + n_stft]; o += n_stft
    bcount = blob[o:o + n_stft]; o += n_stft
    bvals = f[o:o + n_stft * (kb + 1)].reshape(n_stft, kb + 1); o += n_stft * (kb + 1)
    ffirst = blob[o:o + n_mels]; o += n_mels
    fcount = blob[o:o + n_mels]
    return lsub, inv_d, bfirst, bcount, bvals, ffirst, fcount


@pytest.mark.parametrize("name", CONFIGS)
def test_plan_matches_dense_factorisation(inv_ref, lib, name):
    from audio_b200 import _lib

    fb = inv_ref[f"{name}_fb"]
    n_stft, n_mels = fb.shape
    rc, blob, bw, piv = _plan(lib, fb)
    assert rc == _lib.OK and bw == 1 and piv == -1
    assert tuple(blob[:3]) == (n_stft, n_mels, 1)
    lsub, inv_d, bfirst, bcount, bvals, ffirst, fcount = _unpack(blob, n_stft, n_mels)
    G = fb.astype(np.float64).T @ fb.astype(np.float64)
    L = np.eye(n_mels) + np.diag(lsub[1:, 0].astype(np.float64), -1)
    assert not lsub[:, 1:].any() and lsub[0, 0] == 0
    recon = L @ np.diag(1.0 / inv_d.astype(np.float64)) @ L.T
    assert np.abs(recon - G).max() <= 1e-6 * np.abs(G).max()
    # G^-1 through the stored factors against a dense float64 solve
    b = np.random.default_rng(0).random((n_mels, 3))
    z = np.linalg.solve(L.T, np.linalg.solve(L, b) * inv_d[:, None].astype(np.float64))
    assert np.abs(z - np.linalg.solve(G, b)).max() <= 1e-5 * np.abs(np.linalg.solve(G, b)).max()
    for k in range(n_stft):
        nz = np.flatnonzero(fb[k])
        assert bcount[k] == (0 if nz.size == 0 else nz[-1] - nz[0] + 1)
        if nz.size:
            assert bfirst[k] == nz[0] and np.array_equal(bvals[k, :bcount[k]], fb[k, nz[0]:nz[-1] + 1])
    for m in range(n_mels):
        nz = np.flatnonzero(fb[:, m])
        assert ffirst[m] == nz[0] and fcount[m] == nz[-1] - nz[0] + 1


def test_plan_statuses(inv_ref, lib):
    import audio_b200.functional as F
    from audio_b200 import _lib

    for n_stft, n_mels, sr in ((201, 128, 16000), (65, 128, 16000)):
        fb = F.melscale_fbanks(n_stft, 0.0, sr / 2, n_mels, sr).numpy()
        rc, _, _, piv = _plan(lib, fb, 0)
        assert rc == _lib.ESINGULAR and piv >= 0
    # the rank-revealing drivers: singular underdetermined banks are ESINGULAR (raised as "not supported"), tall ones
    # EUNSUPPORTED
    fb = F.melscale_fbanks(201, 0.0, 8000.0, 128, 16000).numpy()
    assert _plan(lib, fb, 2)[0] == _lib.ESINGULAR
    fb = F.melscale_fbanks(65, 0.0, 8000.0, 128, 16000).numpy()
    assert _plan(lib, fb, 2)[0] == _lib.EUNSUPPORTED
    # bandwidth cap: a bin touching cap + 1 filters is fine, cap + 2 is not
    cap = _lib.INVERSE_MEL_MAX_BANDWIDTH
    base = inv_ref["c201_40_16k_fb"].copy()
    f0 = int(np.flatnonzero(base[100])[0])
    ok = base.copy(); ok[100, f0:f0 + 1 + cap] = 0.25
    rc, _, bw, _ = _plan(lib, ok)
    assert rc == _lib.OK and bw == cap
    bad = base.copy(); bad[100, f0:f0 + 2 + cap] = 0.25
    rc, _, bw, _ = _plan(lib, bad)
    assert rc == _lib.EUNSUPPORTED and bw == cap + 1
    # n_mels cap: a linear (identity-like) bank of MAX_MELS filters is fine, one more is not
    for n_mels, want in ((_lib.INVERSE_MEL_MAX_MELS, _lib.OK), (_lib.INVERSE_MEL_MAX_MELS + 1, _lib.EUNSUPPORTED)):
        eye = np.zeros((2 * n_mels, n_mels), dtype=np.float32)
        eye[np.arange(n_mels) * 2, np.arange(n_mels)] = 1.0
        assert _plan(lib, eye)[0] == want
    # a too-small blob
    bw, piv = ctypes.c_int32(), ctypes.c_int32()
    buf = np.zeros(16, dtype=np.int32)
    fb = np.ascontiguousarray(base)
    assert lib.b200a_inverse_mel_plan(fb.ctypes.data, 201, 40, 0, buf.ctypes.data, 64, ctypes.byref(bw),
                                      ctypes.byref(piv)) == _lib.EWORKSPACE


def test_abi_rejects_null_pointers_and_bad_sizes(lib):
    from audio_b200 import _lib

    bw, piv = ctypes.c_int32(), ctypes.c_int32()
    fb = np.ones((4, 2), dtype=np.float32)
    buf = np.zeros(1024, dtype=np.int32)
    assert lib.b200a_inverse_mel_plan(None, 4, 2, 0, buf.ctypes.data, 4096, ctypes.byref(bw), ctypes.byref(piv)) == _lib.EINVAL
    assert lib.b200a_inverse_mel_plan(fb.ctypes.data, 4, 2, 0, None, 4096, ctypes.byref(bw), ctypes.byref(piv)) == _lib.EINVAL
    assert lib.b200a_inverse_mel_plan(fb.ctypes.data, 4, 2, 0, buf.ctypes.data, 4096, None, ctypes.byref(piv)) == _lib.EINVAL
    assert lib.b200a_inverse_mel_plan(fb.ctypes.data, 0, 2, 0, buf.ctypes.data, 4096, ctypes.byref(bw), ctypes.byref(piv)) == _lib.EINVAL
    assert lib.b200a_inverse_mel_plan(fb.ctypes.data, 4, 2, 7, buf.ctypes.data, 4096, ctypes.byref(bw), ctypes.byref(piv)) == _lib.EINVAL
    assert lib.b200a_inverse_mel_plan_bytes(0, 2) == 0 and lib.b200a_inverse_mel_plan_bytes(4, -1) == 0
    assert lib.b200a_inverse_mel_run(None, 4, 2, None, 1, 1, 8, 4, 1, None, None) == _lib.EINVAL
    assert lib.b200a_inverse_mel_run(None, 0, 2, None, 1, 1, 8, 4, 1, None, None) == _lib.EINVAL
    assert lib.b200a_inverse_mel_backward(None, 4, 2, None, 1, 1, 8, 4, 1, None, 4, 4, 1, None, None) == _lib.EINVAL
    assert lib.b200a_inverse_mel_backward(None, 4, -2, None, 1, 1, 8, 4, 1, None, 4, 4, 1, None, None) == _lib.EINVAL
    assert lib.b200a_strerror(_lib.ESINGULAR) == b"rank-deficient system (singular Gram matrix)"


# ---------------- the module surface ---------------------------------------------------------------------------
def test_module_surface_cpu():
    import audio_b200.transforms as T

    assert "InverseMelScale" in T.__all__
    m = T.InverseMelScale(513, 80)
    assert (m.n_mels, m.sample_rate, m.f_min, m.f_max, m.driver) == (80, 16000, 0.0, 8000.0, "gels")
    assert T.InverseMelScale.__constants__ == ["n_stft", "n_mels", "sample_rate", "f_min", "f_max"]
    assert set(m.state_dict()) == {"fb"} and tuple(m.fb.shape) == (513, 80)
    assert T.InverseMelScale(201, 40, 16000, f_max=0.0).f_max == 8000.0  # `f_max or ...`, as the reference
    with pytest.raises(ValueError, match=r"Require f_min: 9000.0 <= f_max: 8000.0"):
        T.InverseMelScale(513, 80, f_min=9000.0)
    with pytest.raises(ValueError, match=r'driver must be one of \["gels", "gelsy", "gelsd", "gelss"\]. Found qr.'):
        T.InverseMelScale(513, 80, driver="qr")
    with pytest.raises(ValueError, match="Expected an input with 80 mel bins. Found: 40"):
        m(torch.rand(2, 40, 5))
    with pytest.raises(RuntimeError, match="no CPU or ATen fallback"):
        m(torch.rand(2, 80, 5))
    import audio_b200

    with audio_b200.differentiable(features=True):
        with pytest.raises(RuntimeError, match="no CPU or ATen fallback"):
            m(torch.rand(2, 80, 5, requires_grad=True))


def test_forward_only_message_names_inverse_mel_scale():
    from audio_b200._plans import _no_autograd

    with pytest.raises(RuntimeError, match=r"MelScale, InverseMelScale, SpectralCentroid.*differentiable\(features=True\)"):
        _no_autograd(torch.zeros(1, requires_grad=True))
