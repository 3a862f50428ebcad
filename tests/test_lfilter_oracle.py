"""IIR filtering without a GPU: the float64 oracle (tests/lfilter_oracle.py) and its VJPs against float64 autograd
through the installed torchaudio's lfilter and filtfilt, the oracle against the reference fixture
(tests/golden/make_lfilter_golden.py), the biquad designs through scipy against the fixture, the ABI statuses of
b200a_lfilter_run / b200a_lfilter_backward, and the Python surface's checks that run before any launch."""
import os

import numpy as np
import pytest
import torch

import lfilter_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lfilter_ref_cases.npz")


@pytest.fixture(scope="module")
def ref():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def _ta():
    return pytest.importorskip("torchaudio.functional")


# a0 are powers of two, so the float32 normalisation is exact and float64 autograd sees the same coefficients
A2 = np.array([[2.0, -0.5, 0.25], [0.5, 0.3, 0.1], [1.0, -1.6, 0.7]], np.float32)
B2 = np.array([[0.3, 0.2, 0.1], [1.0, 0.5, -0.2], [0.05, 0.1, 0.05]], np.float32)


@pytest.mark.parametrize("clamp", (False, True))
def test_vjp_matches_float64_autograd(clamp):
    ta = _ta()
    rng = np.random.default_rng(1)
    x = rng.standard_normal((2, 3, 257)) * 0.7
    g = rng.standard_normal(x.shape)
    xt = torch.tensor(x, requires_grad=True)
    at, bt = torch.tensor(A2.astype(np.float64), requires_grad=True), torch.tensor(B2.astype(np.float64), requires_grad=True)
    y = ta.lfilter(xt, at, bt, clamp=clamp)
    assert np.abs(O.lfilter(x, A2, B2, clamp) - y.detach().numpy()).max() < 1e-12
    (y * torch.tensor(g)).sum().backward()
    dx, da, db = O.lfilter_vjp(x, A2, B2, g, clamp)
    scale = max(np.abs(xt.grad.numpy()).max(), 1.0)
    assert np.abs(dx - xt.grad.numpy()).max() < 1e-10 * scale
    assert np.abs(da - at.grad.numpy()).max() < 1e-10 * max(np.abs(da).max(), 1.0)
    assert np.abs(db - bt.grad.numpy()).max() < 1e-10 * max(np.abs(db).max(), 1.0)
    if clamp:
        assert (np.abs(O.lfilter(x, A2, B2, False)) > 1).any()  # the clamp mask is exercised


@pytest.mark.parametrize("clamp", (False, True))
def test_filtfilt_vjp_matches_float64_autograd(clamp):
    ta = _ta()
    rng = np.random.default_rng(2)
    x = rng.standard_normal((3, 300)) * 0.8
    g = rng.standard_normal(x.shape)
    a, b = A2[0], B2[0]
    xt = torch.tensor(x, requires_grad=True)
    at, bt = torch.tensor(a.astype(np.float64), requires_grad=True), torch.tensor(b.astype(np.float64), requires_grad=True)
    y = ta.filtfilt(xt, at, bt, clamp=clamp)
    assert np.abs(O.filtfilt(x, a, b, clamp) - y.detach().numpy()).max() < 1e-12
    (y * torch.tensor(g)).sum().backward()
    dx, da, db = O.filtfilt_vjp(x, a, b, g, clamp)
    assert np.abs(dx - xt.grad.numpy()).max() < 1e-10 * max(np.abs(dx).max(), 1.0)
    assert np.abs(da - at.grad.numpy()).max() < 1e-10 * max(np.abs(da).max(), 1.0)
    assert np.abs(db - bt.grad.numpy()).max() < 1e-10 * max(np.abs(db).max(), 1.0)


def test_oracle_matches_fixture(ref):
    """The reference's float32 outputs lie within float32 rounding (amplified by the filters) of the oracle.  The
    order-9 Butterworth in direct form is ill-conditioned: the reference's own float32 error there is 5.7e-3."""
    x = ref["x"]
    for n in (0, 1, 2, 3, 5, 9):
        for c in (0, 1):
            exp = ref[f"lf_n{n}_c{c}"]
            tol = 1e-2 if n == 9 else 1e-4
            assert np.abs(O.lfilter(x, ref[f"lf_n{n}_a"], ref[f"lf_n{n}_b"], bool(c)) - exp).max() < tol, n
    a, b = ref["lf2_a"], ref["lf2_b"]
    for c in (0, 1):
        assert np.abs(O.lfilter(x, a, b, bool(c)) - ref[f"lf2_b1_c{c}"]).max() < 1e-4
        assert np.abs(O.lfilter(np.stack([x[:, 0]] * 3, -2), a, b, bool(c)) - ref[f"lf2_b0_c{c}"]).max() < 1e-4
        assert np.abs(O.filtfilt(x, ref["lf_n3_a"], ref["lf_n3_b"], bool(c)) - ref[f"ff_c{c}"]).max() < 1e-4
    assert np.abs(O.lfilter(x, [1.0, -0.97], [1.0, 0.0]) - ref["de"]).max() < 1e-4
    assert np.abs(O.lfilter(x, [1.0, 0.0], [1.0, -0.97], False) - ref["pre"]).max() < 1e-6
    dx, da, db = O.lfilter_vjp(x, a, b, ref["g_up"], True)
    for got, exp in ((dx, ref["g_x"]), (da, ref["g_a"]), (db, ref["g_b"])):
        assert np.abs(got - exp).max() <= 1e-4 * np.abs(exp).max()


BIQUADS = {
    "allpass": [(16000, dict(central_freq=1000.0, Q=0.707)), (44100, dict(central_freq=200.0, Q=2.0))],
    "band": [(16000, dict(central_freq=1000.0, Q=0.707)), (16000, dict(central_freq=3000.0, Q=3.0, noise=True))],
    "bandpass": [(16000, dict(central_freq=1000.0, Q=0.707)),
                 (48000, dict(central_freq=500.0, Q=4.0, const_skirt_gain=True))],
    "bandreject": [(16000, dict(central_freq=1000.0, Q=0.707)), (44100, dict(central_freq=60.0, Q=5.0))],
    "bass": [(16000, dict(gain=6.0)), (44100, dict(gain=-10.0, central_freq=200.0, Q=1.2))],
    "equalizer": [(16000, dict(center_freq=1000.0, gain=6.0)), (48000, dict(center_freq=8000.0, gain=-9.0, Q=2.0))],
    "highpass": [(16000, dict(cutoff_freq=100.0)), (48000, dict(cutoff_freq=3000.0, Q=1.5))],
    "lowpass": [(16000, dict(cutoff_freq=1000.0)), (48000, dict(cutoff_freq=20.0, Q=2.0)),
                (16000, dict(cutoff_freq=100.0))],
    "treble": [(16000, dict(gain=6.0)), (44100, dict(gain=-4.0, central_freq=8000.0, Q=0.5))],
    "deemph": [(44100, {}), (48000, {})],
}


@pytest.mark.parametrize("name", sorted(BIQUADS))
def test_biquad_designs_match_fixture(ref, name):
    """Each design helper on CPU tensors, its float32 coefficients through scipy in float64, against the reference's
    float32 output of the same biquad: within the reference's own float32 recurrence error (3.1e-4 for the stiffest
    setting, a 60 Hz notch with Q = 5 at 44.1 kHz)."""
    x = ref["x"][0]
    for i, (sr, kw) in enumerate(BIQUADS[name]):
        a, b = O.biquad_coeffs(name, sr, kw)
        exp = ref[f"bq_{name}_{i}"]
        err = np.abs(O.lfilter(x, a, b) - exp).max()
        assert err < 1e-3 * max(1.0, np.abs(exp).max()), f"{name}[{i}]: {err:.3e}"


@pytest.mark.parametrize("sr", (44100, 48000, 88200, 96000))
def test_riaa_design_matches_fixture(ref, sr):
    a, b = O.biquad_coeffs("riaa", sr, {})
    assert np.abs(O.lfilter(ref["x"][0], a, b) - ref[f"riaa_{sr}"]).max() < 2e-4


def test_reference_errors_are_recorded(ref):
    assert str(ref["err_size"]).startswith("ValueError: Expected coeffs to be the same size.Found:")
    assert str(ref["err_riaa"]) == "ValueError: Sample rate must be 44.1k, 48k, 88.2k, or 96k"
    import audio_b200.functional as F

    x = torch.zeros(2, 3, 10)
    for key, fn in (("err_size", lambda: F.lfilter(x, torch.ones(3), torch.ones(2))),
                    ("err_ndim", lambda: F.lfilter(x, torch.ones(1, 3, 3), torch.ones(1, 3, 3))),
                    ("err_batches", lambda: F.lfilter(x[:, :2], torch.ones(3, 3), torch.ones(3, 3))),
                    ("err_wave_ndim", lambda: F.lfilter(torch.tensor(0.5), torch.ones(3, 3), torch.ones(3, 3))),
                    ("err_riaa", lambda: F.riaa_biquad(x[0], 16000)),
                    ("err_deemph", lambda: F.deemph_biquad(x[0], 16000))):
        with pytest.raises(ValueError) as info:
            fn()
        if key in ("err_riaa", "err_deemph"):
            assert f"ValueError: {info.value}" == str(ref[key])
        elif key != "err_size":  # the size message prints torch.Size of these tensors
            assert f"ValueError: {info.value}".split("Found")[0] == str(ref[key]).split("Found")[0]


def test_surface_rejects_cpu():
    import audio_b200.functional as F

    with pytest.raises(RuntimeError, match="no CPU or ATen fallback"):
        F.lfilter(torch.zeros(2, 10), torch.tensor([1.0, 0.5]), torch.tensor([1.0, 0.0]))
    with pytest.raises(RuntimeError, match="no CPU or ATen fallback"):
        F.deemphasis(torch.zeros(2, 10))


def test_switch_and_message():
    import audio_b200
    from audio_b200 import _plans

    assert not audio_b200.is_filtering_differentiable()
    with audio_b200.differentiable(filtering=True):
        assert audio_b200.is_filtering_differentiable()
        with audio_b200.differentiable(features=True):
            assert not audio_b200.is_filtering_differentiable()
        assert audio_b200.is_filtering_differentiable()
    with audio_b200.differentiable(False, filtering=True):  # only together with mode
        assert not audio_b200.is_filtering_differentiable()
    assert not audio_b200.is_filtering_differentiable()
    with pytest.raises(RuntimeError, match=r"forward-only.*differentiable\(filtering=True\)"):
        _plans._no_autograd(torch.zeros(1, requires_grad=True))


def test_transforms_surface():
    import audio_b200.transforms as T

    assert "Preemphasis" in T.__all__ and "Deemphasis" in T.__all__
    assert T.Preemphasis().coeff == 0.97 and T.Deemphasis(0.5).coeff == 0.5
    assert T.Preemphasis().state_dict() == {}


# ---- the C ABI ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from audio_b200 import _lib

    return _lib.lib()


def test_abi_statuses(lib):
    from audio_b200 import _lib

    cap = _lib.LFILTER_MAX_ORDER
    assert lib.b200a_lfilter_workspace_bytes(4, 1000, cap + 1, 2) > 0  # order cap: accepted
    assert lib.b200a_lfilter_workspace_bytes(4, 1000, cap + 2, 2) == 0  # cap + 1: refused
    assert lib.b200a_lfilter_workspace_bytes(4, 1000, 1, 2) > 0  # n_order = 1: a pure gain
    assert lib.b200a_lfilter_workspace_bytes(4, 1000, 0, 2) == 0
    assert lib.b200a_lfilter_backward_workspace_bytes(4, 1000, 3, 2) > lib.b200a_lfilter_workspace_bytes(4, 1000, 3, 2)
    fake = 0x1000  # never dereferenced: every call below returns before a launch
    run = lib.b200a_lfilter_run
    nb = lib.b200a_lfilter_workspace_bytes(2, 100, 3, 1)
    assert run(fake, fake, 1, cap + 2, fake, 2, 100, 100, 0, 1, 0, fake, None, fake, 1 << 30, None) == _lib.EUNSUPPORTED
    assert run(fake, fake, 1, 0, fake, 2, 100, 100, 0, 1, 0, fake, None, fake, 1 << 30, None) == _lib.EINVAL
    assert run(fake, fake, 0, 3, fake, 2, 100, 100, 0, 1, 0, fake, None, fake, 1 << 30, None) == _lib.EINVAL
    for nulls in range(5):
        args = [fake, fake, fake, fake, fake]  # a, b, x, y, workspace
        args[nulls] = None
        a, b, x, y, ws = args
        assert run(a, b, 1, 3, x, 2, 100, 100, 0, 1, 0, y, None, ws, nb, None) == _lib.EINVAL, nulls
    assert run(fake, fake, 1, 3, fake, 2, 100, 100, 0, 1, 0, fake, None, fake, nb - 1, None) == _lib.EWORKSPACE
    assert run(None, None, 1, 3, None, 0, 100, 100, 0, 1, 0, None, None, None, 0, None) == _lib.OK  # empty batch
    assert run(fake, fake, 1, 3, fake, -1, 100, 100, 0, 1, 0, fake, None, fake, nb, None) == _lib.EINVAL
    bw = lib.b200a_lfilter_backward
    nbb = lib.b200a_lfilter_backward_workspace_bytes(2, 100, 3, 1)
    assert bw(fake, fake, 1, cap + 2, fake, 2, 100, 100, 0, fake, fake, 1, 0, fake, fake, fake, fake, 1 << 30,
              None) == _lib.EUNSUPPORTED
    assert bw(fake, fake, 1, 3, fake, 2, 100, 100, 0, None, fake, 1, 0, fake, fake, fake, fake, nbb, None) == _lib.EINVAL
    assert bw(fake, fake, 1, 3, fake, 2, 100, 100, 0, fake, None, 1, 0, fake, fake, fake, fake, nbb, None) == _lib.EINVAL
    assert bw(fake, fake, 1, 3, fake, 2, 100, 100, 0, fake, fake, 1, 0, fake, fake, fake, fake, nbb - 1,
              None) == _lib.EWORKSPACE
    assert bw(fake, fake, 1, 3, fake, 2, 100, 100, 0, fake, fake, 1, 0, fake, fake, fake, fake, nb,
              None) == _lib.EWORKSPACE  # the forward's workspace is too small for the backward
