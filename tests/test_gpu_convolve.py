"""convolve and Convolve on the GPU: parity with the float64 oracle (tests/conv_oracle.py, direct form) and the reference
fixture (tests/golden/make_convolve_golden.py), k-step edges, the swap, tile and halo edges, strides, broadcasting,
bitwise properties, gradients under differentiable(filtering=True), and what must raise.

The parity bar is evidence-based: the reference's own float32 error against the float64 oracle is measured on the same
inputs (the installed torchaudio's convolve on the same CUDA tensors: a grouped cuDNN conv1d), and ours may be at most
twice that plus 2e-6 of the exact output's rms.  cuDNN's TF32 mode is off for the whole module: at torch's default it
is on, and the reference's error would then be about 1000 times larger than its float32 error."""
import os

import numpy as np
import pytest
import torch

import conv_oracle as O

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "convolve_ref_cases.npz")
MODES = ("full", "valid", "same")


@pytest.fixture(scope="module", autouse=True)
def _float32_reference_and_release():
    """The reference arm in float32 (cuDNN TF32 off), restored afterwards; and the full-size cases' memory given back
    when the module ends, so later modules start from the state they would see without it."""
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = prev
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def F():
    import audio_b200.functional as F

    return F


def ta():
    return pytest.importorskip("torchaudio.functional")


def rms(a):
    return float(np.sqrt(np.mean(np.square(a)))) if np.size(a) else 0.0


def randn(*shape, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g).cuda()


def check_bar(got, exact, theirs, what):
    """|ours - f64| <= 2 |ref - f64| + 2e-6 rms (max-abs over the case)."""
    got = got.detach().double().cpu().numpy()
    theirs = theirs.detach().double().cpu().numpy() if isinstance(theirs, torch.Tensor) else np.asarray(theirs)
    assert got.shape == exact.shape, (what, got.shape, exact.shape)
    if not exact.size:
        return
    ours = np.abs(got - exact).max()
    ref_err = np.abs(theirs - exact).max()
    bar = 2 * ref_err + 2e-6 * max(rms(exact), 1e-6)
    assert ours <= bar, f"{what}: max err {ours:.3e} vs bar {bar:.3e} (reference float32 error {ref_err:.3e})"


def parity(x, y, mode, what):
    got = F().convolve(x, y, mode)
    exact = O.fftconvolve(x.double().cpu().numpy(), y.double().cpu().numpy(), mode, direct=True)
    check_bar(got, exact, ta().convolve(x, y, mode), what)
    return got


# ---- parity ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("k", list(range(1, 18)) + [63, 64, 65, 127, 128, 129, 1023, 1024, 1025, 4095, 4096])
def test_kstep_edges(k, mode):
    """K at every k-step edge (ceil((K + 7) / 8) steps), at the M-tile edges of the filter gradient (128 taps), the
    fragment staging limit and the cap."""
    x, y = randn(3, 5000 + k, seed=k), randn(3, k, seed=k + 1)
    parity(x, y, mode, f"K={k} {mode}")


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("n, m", [(1, 1), (1, 700), (700, 1), (300, 1000), (1000, 300), (777, 777), (20, 15),
                                  (15, 20), (2048, 33), (2049, 33), (4200, 4096), (100, 3000)])
def test_shapes(n, m, mode):
    """1-sample operands, N < M (the swap), N == M, signals shorter than K + 7 and than one 2048-output tile, and
    lengths at the tile edge."""
    parity(randn(2, n, seed=n), randn(2, m, seed=m + 7), mode, f"{n} x {m} {mode}")


@pytest.mark.parametrize("mode", ("same", "valid"))
def test_mid_tile_starts(mode):
    """"same" with odd and even K and "valid": the first output is not a multiple of 8 into the full range."""
    for m in (30, 31, 301, 1500, 2600):
        parity(randn(2, 9000, seed=m), randn(2, m, seed=m + 1), mode, f"m={m} {mode}")


@pytest.mark.parametrize("mode", MODES)
def test_broadcasting(mode):
    x, y = randn(3, 1, 5000, seed=1), randn(1, 4, 90, seed=2)
    got = parity(x, y, mode, f"(3,1,T) * (1,4,M) {mode}")
    assert got.shape[:2] == (3, 4)
    parity(randn(1, 4, 90, seed=3), randn(3, 1, 5000, seed=4), mode, f"(1,4,M) * (3,1,T) {mode}")
    parity(randn(2, 1, 3, 1, 700, seed=5), randn(1, 5, 1, 2, 210, seed=6), mode, f"5-D {mode}")
    parity(randn(4000, seed=7), randn(300, seed=8), mode, f"1-D {mode}")


def test_strided_and_offset_views():
    base = randn(4, 3, 12000, seed=3)
    x = base[:, 1, 1000:11000]  # row stride 36000, offset 1000 + 12000
    y = randn(2000, 4, seed=4).t()[:, 5:305]  # non-unit time stride: made contiguous
    for mode in MODES:
        parity(x, y, mode, f"views {mode}")
        parity(x[::2], randn(2, 1, 333, seed=5)[:, 0], mode, f"row step {mode}")


def test_fixture_cases():
    with np.load(GOLDEN) as z:
        ref = {k: z[k] for k in z.files}
    for key in ref:
        if not key.startswith("out_"):
            continue
        case = key[4:]
        x, y, mode = ref[f"x_{case}"], ref[f"y_{case}"], str(ref[f"mode_{case}"])
        got = F().convolve(torch.as_tensor(x).cuda(), torch.as_tensor(y).cuda(), mode)
        check_bar(got, O.fftconvolve(x, y, mode, direct=True), ref[key], case)


@pytest.mark.parametrize("shared", (False, True))
def test_full_size(shared):
    """64 x 160 000 with per-row 1024-tap filters, or one shared 4096-tap filter."""
    x = randn(64, 160000, seed=11)
    y = randn(1, 4096, seed=12) / 64 if shared else randn(64, 1024, seed=13) / 32
    parity(x, y, "full", f"full size shared={shared}")


# ---- properties --------------------------------------------------------------------------------------------------
def test_bitwise_properties():
    x, y = randn(8, 30000, seed=21), randn(8, 300, seed=22)
    a = F().convolve(x, y)
    assert torch.equal(a, F().convolve(x, y)), "rerun"
    for rows in ([3], [0, 5], [7, 1, 2]):
        alone = F().convolve(x[rows], y[rows])
        assert torch.equal(alone, a[rows]), rows
    ys = randn(1, 300, seed=23)
    assert torch.equal(F().convolve(x, ys), F().convolve(x, ys.expand(8, 300).contiguous())), "broadcast"
    assert torch.equal(F().convolve(ys, x), F().convolve(ys.expand(8, 300).contiguous(), x)), "broadcast x"
    xs = randn(1, 30000, seed=24)
    assert torch.equal(F().convolve(xs, y), F().convolve(xs.expand(8, 30000).contiguous(), y)), "broadcast signal"
    import audio_b200
    import audio_b200.transforms as T

    for mode in MODES:
        assert torch.equal(T.Convolve(mode)(x, y), F().convolve(x, y, mode)), mode
    with audio_b200.differentiable(filtering=True):
        xg = x.clone().requires_grad_()
        assert torch.equal(F().convolve(xg, y), a), "forward with grad"


# ---- gradients ---------------------------------------------------------------------------------------------------
def grads(x, y, g, mode):
    import audio_b200

    xg, yg = x.clone().requires_grad_(), y.clone().requires_grad_()
    with audio_b200.differentiable(filtering=True):
        (F().convolve(xg, yg, mode) * g).sum().backward()
    return xg.grad, yg.grad


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("shapes", [((4, 6000), (4, 70)), ((4, 70), (4, 6000)), ((3, 1, 5000), (1, 2, 250)),
                                    ((1, 2, 900), (3, 1, 4100)), ((2, 3000), (2, 3000)), ((2, 777), (2, 777)),
                                    ((2, 9000), (2, 1)), ((2, 20000), (2, 1025))])
def test_gradients_match_oracle(shapes, mode):
    (xs, ys) = shapes
    x, y = randn(*xs, seed=31), randn(*ys, seed=32)
    out_shape = F().convolve(x, y, mode).shape
    g = randn(*out_shape, seed=33)
    gx, gy = grads(x, y, g, mode)
    ex, ey = O.vjp(x.double().cpu().numpy(), y.double().cpu().numpy(), g.double().cpu().numpy(), mode, direct=True)
    # the reference's float32 autograd (cuDNN, TF32 off) on the same tensors
    xr, yr = x.clone().requires_grad_(), y.clone().requires_grad_()
    (ta().convolve(xr, yr, mode) * g).sum().backward()
    check_bar(gx, ex, xr.grad, f"dx {shapes} {mode}")
    check_bar(gy, ey, yr.grad, f"dy {shapes} {mode}")


def test_gradients_bitwise():
    x, y = randn(6, 9000, seed=51), randn(6, 200, seed=52)
    g = randn(6, 9199, seed=53)
    gx, gy = grads(x, y, g, "full")
    gx2, gy2 = grads(x, y, g, "full")
    assert torch.equal(gx, gx2) and torch.equal(gy, gy2), "rerun"
    gxs, gys = grads(x[2:4], y[2:4], g[2:4], "full")
    assert torch.equal(gxs, gx[2:4]) and torch.equal(gys, gy[2:4]), "row subset"


def test_adjoint_identity_full_size():
    x, y = randn(64, 160000, seed=41), randn(64, 1024, seed=42) / 30
    g = randn(64, 161023, seed=43)
    gx, gy = grads(x, y, g, "full")
    out = F().convolve(x, y).double()
    lhs = float((g.double() * out).sum())
    for name, v, d in (("x", x, gx), ("y", y, gy)):
        rhs = float((v.double() * d.double()).sum())
        assert abs(lhs - rhs) <= 1e-5 * (abs(lhs) + float((g.double() * out).abs().sum()) * 1e-3), (name, lhs, rhs)


def test_forward_only_and_double_backward():
    import audio_b200

    x, y = randn(2, 1000).requires_grad_(), randn(2, 100)
    with pytest.raises(RuntimeError, match=r"forward-only.*filtering=True"):
        F().convolve(x, y)
    with pytest.raises(RuntimeError, match=r"forward-only.*filtering=True"):
        F().convolve(y.detach(), randn(2, 50).requires_grad_())
    with audio_b200.differentiable(filtering=True):
        out = F().convolve(x, y)
        (gx,) = torch.autograd.grad(out.sum(), x, create_graph=True)
        with pytest.raises(RuntimeError):
            gx.sum().backward()


# ---- errors ------------------------------------------------------------------------------------------------------
def test_errors():
    f = F()
    with pytest.raises(ValueError, match=r"The operands must be the same dimension \(got 3 and 2\)\."):
        f.convolve(randn(2, 3, 10), randn(3, 10))
    with pytest.raises(ValueError, match="Leading dimensions of x and y are not broadcastable"):
        f.convolve(randn(3, 10), randn(2, 4))
    with pytest.raises(ValueError, match=r"Unrecognized mode value 'foo'\. Please specify one of \['full', 'valid', 'same'\]\."):
        f.convolve(randn(3, 10), randn(3, 4), "foo")
    with pytest.raises(RuntimeError, match="not supported.*4096.*fftconvolve"):
        f.convolve(randn(1, 10000), randn(1, 4097))
    with pytest.raises(RuntimeError, match="not supported.*4096.*fftconvolve"):
        f.convolve(randn(1, 4097), randn(1, 10000))
    assert f.convolve(randn(1, 10000), randn(1, 4096)).shape == (1, 14095)
    with pytest.raises(RuntimeError, match="no CPU or ATen fallback"):
        f.convolve(torch.zeros(2, 10), torch.zeros(2, 3))
    with pytest.raises(TypeError, match="float32"):
        f.convolve(randn(2, 10).double(), randn(2, 3).double())
    import audio_b200.transforms as T

    with pytest.raises(ValueError, match="Unrecognized mode value"):
        T.Convolve("circular")


def _same_error(fn_ref, fn_ours):
    with pytest.raises(RuntimeError) as theirs:
        fn_ref()
    with pytest.raises(RuntimeError) as ours:
        fn_ours()
    assert str(ours.value) == str(theirs.value)


def test_empty_operands_as_reference():
    """Zero-length operands and zero output rows: exactly the reference's RuntimeError text."""
    for n, m in ((0, 5), (5, 0), (0, 1), (1, 0), (0, 0)):
        for mode in MODES:
            _same_error(lambda: ta().convolve(torch.zeros(2, n).cuda(), torch.ones(2, m).cuda(), mode),
                        lambda: F().convolve(torch.zeros(2, n).cuda(), torch.ones(2, m).cuda(), mode))
    for xs, ys in (((0, 10), (0, 4)), ((0, 0), (0, 4)), ((3, 0, 10), (3, 1, 4)), ((1, 4), (0, 10))):
        _same_error(lambda: ta().convolve(torch.zeros(xs).cuda(), torch.ones(ys).cuda()),
                    lambda: F().convolve(torch.zeros(xs).cuda(), torch.ones(ys).cuda()))
