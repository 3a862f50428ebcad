"""lfilter, filtfilt, the biquads and pre-/de-emphasis on the GPU: parity with the reference fixture
(tests/golden/make_lfilter_golden.py) and the float64 oracle (tests/lfilter_oracle.py), long stiff filters, shapes and
boundaries, bitwise properties, gradients under differentiable(filtering=True), and what must raise.

The parity bar is evidence-based: the reference's own float32 error against the float64 oracle is measured on the
same case (from the fixture, or from the installed torchaudio's CPU float32 lfilter when the case is not in the
fixture), and ours may be at most twice that plus 1e-6 of the output's rms.  The chunked scan carries in double, so
it is usually below the reference's serial float32 error, not just within twice it."""
import os

import numpy as np
import pytest
import torch

import lfilter_oracle as O

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lfilter_ref_cases.npz")
CHUNK, TILE = 32, 4096  # kChunk and the tile of csrc/lfilter.cu


@pytest.fixture(scope="module")
def ref():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def F():
    import audio_b200.functional as F

    return F


def cuda(a):
    return torch.as_tensor(np.asarray(a), dtype=torch.float32).cuda()


def rms(a):
    return float(np.sqrt(np.mean(np.square(a)))) if np.size(a) else 0.0


def check_bar(got, exact, ref_out, what):
    """|ours - f64| <= 2 |ref - f64| + 1e-6 rms (max-abs over the case)."""
    got = got.detach().double().cpu().numpy() if isinstance(got, torch.Tensor) else got
    ours = np.abs(got - exact).max() if exact.size else 0.0
    theirs = np.abs(np.asarray(ref_out, np.float64) - exact).max() if exact.size else 0.0
    bar = 2 * theirs + 1e-6 * max(rms(exact), 1e-3)
    assert ours <= bar, f"{what}: max err {ours:.3e} vs bar {bar:.3e} (reference float32 error {theirs:.3e})"


def ref_float32(x, a, b, clamp=True, batching=True):
    """The installed torchaudio's float32 CPU lfilter, when importable (the reference error of cases off the fixture)."""
    ta = pytest.importorskip("torchaudio.functional")
    return ta.lfilter(torch.as_tensor(x, dtype=torch.float32), torch.as_tensor(a), torch.as_tensor(b), clamp=clamp,
                      batching=batching).numpy()


# ---- parity ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", (0, 1, 2, 3, 5, 9))
@pytest.mark.parametrize("clamp", (0, 1))
def test_lfilter_1d_matches_fixture(ref, n, clamp):
    x, a, b = ref["x"], ref[f"lf_n{n}_a"], ref[f"lf_n{n}_b"]
    got = F().lfilter(cuda(x), cuda(a), cuda(b), clamp=bool(clamp))
    check_bar(got, O.lfilter(x, a, b, bool(clamp)), ref[f"lf_n{n}_c{clamp}"], f"order {n} clamp {clamp}")


@pytest.mark.parametrize("batching", (0, 1))
@pytest.mark.parametrize("clamp", (0, 1))
def test_lfilter_2d_matches_fixture(ref, batching, clamp):
    x, a, b = ref["x"], ref["lf2_a"], ref["lf2_b"]
    xin = x if batching else x[:, 0]
    got = F().lfilter(cuda(xin), cuda(a), cuda(b), clamp=bool(clamp), batching=bool(batching))
    xs = x if batching else np.stack([x[:, 0]] * 3, -2)
    exp = O.lfilter(xs, a, b, bool(clamp))
    assert tuple(got.shape) == exp.shape
    check_bar(got, exp, ref[f"lf2_b{batching}_c{clamp}"], f"2-D batching {batching} clamp {clamp}")


@pytest.mark.parametrize("clamp", (0, 1))
def test_filtfilt_matches_fixture(ref, clamp):
    x, a, b = ref["x"], ref["lf_n3_a"], ref["lf_n3_b"]
    got = F().filtfilt(cuda(x), cuda(a), cuda(b), clamp=bool(clamp))
    check_bar(got, O.filtfilt(x, a, b, bool(clamp)), ref[f"ff_c{clamp}"], f"filtfilt clamp {clamp}")


BIQUAD_SETTINGS = {
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


@pytest.mark.parametrize("name", sorted(BIQUAD_SETTINGS))
def test_biquads_match_fixture(ref, name):
    """The kernel's error is measured against the oracle on the coefficients this package designed on the device; the
    reference's against the oracle on the same design evaluated on the CPU (device sin / cos may round differently,
    which a stiff filter amplifies: that is the design's rounding, not the recurrence's)."""
    x = ref["x"][0]
    for i, (sr, kw) in enumerate(BIQUAD_SETTINGS[name]):
        got = getattr(F(), f"{name}_biquad")(cuda(x), sr, **kw)
        a_dev, b_dev = O.biquad_coeffs(name, sr, kw, "cuda")
        a_cpu, b_cpu = O.biquad_coeffs(name, sr, kw, "cpu")
        exact = O.lfilter(x, a_dev, b_dev)
        theirs = ref[f"bq_{name}_{i}"] - O.lfilter(x, a_cpu, b_cpu) + exact  # the reference's error, moved onto exact
        check_bar(got, exact, theirs, f"{name}[{i}]")


@pytest.mark.parametrize("sr", (44100, 48000, 88200, 96000))
def test_riaa_matches_fixture(ref, sr):
    x = ref["x"][0]
    a, b = O.biquad_coeffs("riaa", sr, {})
    check_bar(F().riaa_biquad(cuda(x), sr), O.lfilter(x, a, b), ref[f"riaa_{sr}"], f"riaa {sr}")


def test_emphasis_matches_fixture(ref):
    x = ref["x"]
    assert np.abs(F().preemphasis(cuda(x), 0.97).cpu().numpy() - ref["pre"]).max() <= 1e-6
    de = F().deemphasis(cuda(x), 0.97).cpu().numpy()
    check_bar(de, O.lfilter(x, [1.0, -0.97], [1.0, 0.0], True), ref["de"], "deemphasis")
    assert np.abs(de).max() <= 1.0  # the reference's default clamp


def test_reference_error_strings(ref):
    import audio_b200.functional as F

    x = cuda(ref["x"])
    a1, b1 = cuda(ref["lf_n2_a"]), cuda(ref["lf_n2_b"])
    a2, b2 = cuda(ref["lf2_a"]), cuda(ref["lf2_b"])
    cases = {"err_size": lambda: F.lfilter(x, a1, b1[:2]), "err_ndim": lambda: F.lfilter(x, a2[None], b2[None]),
             "err_batches": lambda: F.lfilter(x[:, :2], a2, b2),
             "err_wave_ndim": lambda: F.lfilter(torch.tensor(0.5, device="cuda"), a2, b2),
             "err_riaa": lambda: F.riaa_biquad(x[0], 16000), "err_deemph": lambda: F.deemph_biquad(x[0], 16000)}
    for key, fn in cases.items():
        with pytest.raises(ValueError) as info:
            fn()
        assert f"ValueError: {info.value}" == str(ref[key]), key


# ---- long and stiff ----------------------------------------------------------------------------------------------
def test_long_stiff_lowpass():
    """64 x 480 000 samples (10 s at 48 kHz) through a 20 Hz, Q = 2 lowpass: 118 tiles of carries per row."""
    import audio_b200.functional as F

    g = torch.Generator().manual_seed(5)
    x = 0.5 * torch.randn(64, 480000, generator=g)
    got = F.lowpass_biquad(x.cuda(), 48000, 20.0, 2.0).cpu().numpy()
    from audio_b200._filtering import _design_lowpass

    b, a = [[float(c) for c in cs] for cs in _design_lowpass(48000, 20.0, 2.0, torch.float32, "cpu")]
    rows = [0, 17, 63]
    exact = O.lfilter(x[rows].numpy(), np.float32(a), np.float32(b), clamp=True)
    theirs = ref_float32(x[rows].numpy(), np.float32(a), np.float32(b))
    check_bar(got[rows], exact, theirs, "20 Hz lowpass, 480 000 samples")


# ---- boundaries and shapes ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("length", (1, CHUNK - 1, CHUNK, CHUNK + 1, TILE - 1, TILE, TILE + 1, 3 * TILE + 777))
@pytest.mark.parametrize("n", (0, 2, 16))
def test_lengths_and_orders(length, n):
    import audio_b200.functional as F
    from scipy import signal

    rng = np.random.default_rng(length + n)
    x = (0.3 * rng.standard_normal((3, length))).astype(np.float32)
    if n == 0:
        a, b = np.float32([1.3]), np.float32([0.7])
    else:
        bb, aa = signal.cheby1(n, 1, 0.3) if n <= 8 else signal.butter(n, 0.4)
        a, b = (aa * 1.25).astype(np.float32), (bb * 1.25).astype(np.float32)
    got = F.lfilter(cuda(x), cuda(a), cuda(b), clamp=False)
    check_bar(got, O.lfilter(x, a, b, clamp=False), ref_float32(x, a, b, clamp=False), f"length {length} order {n}")


def test_order_cap():
    import audio_b200.functional as F

    x = torch.randn(2, 5000, device="cuda") * 0.1
    a = torch.zeros(17, device="cuda")
    a[0] = 1.0
    a[16] = 0.2
    b = torch.zeros(17, device="cuda")
    b[0] = 1.0
    got = F.lfilter(x, a, b, clamp=False)
    check_bar(got, O.lfilter(x.cpu().numpy(), a.cpu().numpy(), b.cpu().numpy(), False),
              ref_float32(x.cpu().numpy(), a.cpu().numpy(), b.cpu().numpy(), False), "order 16")
    with pytest.raises(RuntimeError, match="not supported.*16"):
        F.lfilter(x, torch.ones(18, device="cuda"), torch.ones(18, device="cuda"))


def test_strides_and_leading_dims(ref):
    import audio_b200.functional as F

    x, a, b = ref["x"], ref["lf_n2_a"], ref["lf_n2_b"]
    xt = cuda(x)
    base = F.lfilter(xt, cuda(a), cuda(b)).cpu()
    wide = torch.zeros(2, 3, 1300, device="cuda")
    wide[..., 100:700] = xt
    assert torch.equal(F.lfilter(wide[..., 100:700], cuda(a), cuda(b)).cpu(), base)  # row stride 1300
    t = xt.transpose(0, 1).contiguous().transpose(0, 1)  # non-contiguous leading dims
    assert torch.equal(F.lfilter(t, cuda(a), cuda(b)).cpu(), base)
    strided = torch.zeros(2, 3, 1200, device="cuda")
    strided[..., ::2] = xt
    assert torch.equal(F.lfilter(strided[..., ::2], cuda(a), cuda(b)).cpu(), base)  # time stride 2
    assert torch.equal(F.lfilter(xt.reshape(6, 600), cuda(a), cuda(b)).cpu(), base.reshape(6, 600))


# ---- bitwise properties ------------------------------------------------------------------------------------------
def test_reruns_and_batch_independence():
    import audio_b200
    import audio_b200.functional as F

    g = torch.Generator().manual_seed(11)
    x = (0.4 * torch.randn(64, 3 * TILE + 123, generator=g)).cuda()
    a = torch.tensor([1.0, -1.8, 0.81], device="cuda")
    b = torch.tensor([0.01, 0.02, 0.01], device="cuda")
    y1, y2 = F.lfilter(x, a, b), F.lfilter(x, a, b)
    assert torch.equal(y1, y2)
    for r in (0, 37, 63):
        assert torch.equal(F.lfilter(x[r:r + 1], a, b), y1[r:r + 1])
    up = torch.randn(x.shape, generator=g).cuda()
    grads = []
    with audio_b200.differentiable(filtering=True):
        for rows in (slice(None), slice(None), slice(37, 38)):
            xg = x[rows].clone().requires_grad_()
            ag, bg = a.clone().requires_grad_(), b.clone().requires_grad_()
            (F.lfilter(xg, ag, bg) * up[rows]).sum().backward()
            grads.append((xg.grad, ag.grad, bg.grad))
    assert all(torch.equal(p, q) for p, q in zip(grads[0], grads[1]))
    assert torch.equal(grads[2][0], grads[0][0][37:38])


# ---- gradients ---------------------------------------------------------------------------------------------------
def _grad_close(got, exp, what, rel=2e-4):
    got = got.detach().double().cpu().numpy()
    err = np.abs(got - exp).max()
    assert err <= rel * max(np.abs(exp).max(), 1e-6), f"{what}: {err:.3e} vs max {np.abs(exp).max():.3e}"


@pytest.mark.parametrize("clamp", (0, 1))
def test_lfilter_gradients_match_oracle(ref, clamp):
    import audio_b200
    import audio_b200.functional as F

    x, a, b, g = ref["x"], ref["lf2_a"], ref["lf2_b"], ref["g_up"]
    xg, ag, bg = cuda(x).requires_grad_(), cuda(a).requires_grad_(), cuda(b).requires_grad_()
    with audio_b200.differentiable(filtering=True):
        y = F.lfilter(xg, ag, bg, clamp=bool(clamp))
    (y * cuda(g)).sum().backward()
    dx, da, db = O.lfilter_vjp(x, a, b, g, clamp=bool(clamp))
    _grad_close(xg.grad, dx, "dx")
    _grad_close(ag.grad, da, "da")
    _grad_close(bg.grad, db, "db")
    if clamp:  # the reference's own autograd on the same case
        _grad_close(xg.grad, ref["g_x"].astype(np.float64), "dx vs reference", 1e-3)
        _grad_close(ag.grad, ref["g_a"].astype(np.float64), "da vs reference", 1e-3)
        _grad_close(bg.grad, ref["g_b"].astype(np.float64), "db vs reference", 1e-3)


def test_batching_false_gradient(ref):
    import audio_b200
    import audio_b200.functional as F

    x, a, b = ref["x"][:, 0], ref["lf2_a"], ref["lf2_b"]
    g = ref["g_up"]
    xg = cuda(x).requires_grad_()
    with audio_b200.differentiable(filtering=True):
        y = F.lfilter(xg, cuda(a), cuda(b), clamp=False, batching=False)
    (y * cuda(g)).sum().backward()
    dx, _, _ = O.lfilter_vjp(np.stack([x] * 3, -2), a, b, g, clamp=False)
    _grad_close(xg.grad, dx.sum(-2), "batching=False dx")


def test_filtfilt_gradient(ref):
    import audio_b200
    import audio_b200.functional as F

    x, a, b, g = ref["x"], ref["lf_n3_a"], ref["lf_n3_b"], ref["g_up"]
    xg, ag, bg = cuda(x).requires_grad_(), cuda(a).requires_grad_(), cuda(b).requires_grad_()
    with audio_b200.differentiable(filtering=True):
        (F.filtfilt(xg, ag, bg) * cuda(g)).sum().backward()
    dx, da, db = O.filtfilt_vjp(x, a, b, g)
    _grad_close(xg.grad, dx, "filtfilt dx")
    _grad_close(ag.grad, da, "filtfilt da", 1e-3)
    _grad_close(bg.grad, db, "filtfilt db", 1e-3)


def test_biquad_parameter_gradients(ref):
    import audio_b200
    import audio_b200.functional as F

    x, g = ref["x"][0, 0], ref["g_up"][0, 0]
    xq = cuda(x).requires_grad_()
    cut = torch.tensor(1000.0, device="cuda", requires_grad=True)
    q = torch.tensor(0.9, device="cuda", requires_grad=True)
    with audio_b200.differentiable(filtering=True):
        (F.lowpass_biquad(xq, 16000, cut, q) * cuda(g)).sum().backward()
    _grad_close(xq.grad, ref["gq_x"].astype(np.float64), "biquad dx", 1e-3)
    _grad_close(cut.grad.reshape(1), ref["gq_cutoff"].astype(np.float64).reshape(1), "d cutoff", 1e-2)
    _grad_close(q.grad.reshape(1), ref["gq_Q"].astype(np.float64).reshape(1), "d Q", 1e-2)


def test_emphasis_gradients(ref):
    import audio_b200
    import audio_b200.transforms as T
    import audio_b200.functional as F

    x, g = ref["x"], ref["g_up"]
    for fn, a, b, clamp in ((T.Preemphasis(0.9), [1.0, 0.0], [1.0, -0.9], False),
                            (lambda w: F.deemphasis(w, 0.95), [1.0, -0.95], [1.0, 0.0], True)):
        xg = cuda(x).requires_grad_()
        with audio_b200.differentiable(filtering=True):
            (fn(xg) * cuda(g)).sum().backward()
        dx, _, _ = O.lfilter_vjp(x, np.float32(a), np.float32(b), g, clamp=clamp)
        _grad_close(xg.grad, dx, "emphasis dx")


# ---- what must raise ---------------------------------------------------------------------------------------------
def test_forward_only_and_errors(ref):
    import audio_b200
    import audio_b200.functional as F

    x, a, b = cuda(ref["x"]), cuda(ref["lf_n2_a"]), cuda(ref["lf_n2_b"])
    with pytest.raises(RuntimeError, match=r"forward-only.*differentiable\(filtering=True\)"):
        F.lfilter(x.clone().requires_grad_(), a, b)
    with pytest.raises(RuntimeError, match="forward-only"):  # only a_coeffs requires grad
        F.lfilter(x, a.clone().requires_grad_(), b)
    with audio_b200.differentiable():  # the plain switch does not cover filtering
        with pytest.raises(RuntimeError, match="forward-only"):
            F.lowpass_biquad(x, 16000, torch.tensor(500.0, device="cuda", requires_grad=True))
    with torch.no_grad():
        F.lfilter(x.clone().requires_grad_(), a, b)
    with pytest.raises(TypeError):
        F.lfilter(x.double(), a.double(), b.double())
    with audio_b200.differentiable(filtering=True):
        xg = x.clone().requires_grad_()
        y = F.lfilter(xg, a, b)
        (gx,) = torch.autograd.grad(y.sum(), xg, create_graph=True)
        with pytest.raises(RuntimeError):  # double backward
            gx.sum().backward()
        xg = x.clone().requires_grad_()
        xin = xg * 1.0
        y = F.lfilter(xin, a, b)
        xin.mul_(2.0)  # the saved input edited in place before backward
        with pytest.raises(RuntimeError, match="modified by an inplace operation"):
            y.sum().backward()


# ---- the torchaudio wheel's CUDA lfilter -------------------------------------------------------------------------
def test_against_torchaudio_cuda(ref):
    ta = pytest.importorskip("torchaudio.functional")
    import audio_b200.functional as F

    g = torch.Generator().manual_seed(3)
    x = (0.5 * torch.randn(8, 20000, generator=g)).cuda()
    try:
        exp = ta.highpass_biquad(x, 16000, 200.0)
    except Exception as exc:  # noqa: BLE001
        pytest.skip(f"torchaudio's CUDA lfilter is unavailable: {exc}")
    got = F.highpass_biquad(x, 16000, 200.0)
    assert (got - exp).abs().max().item() <= 1e-4
