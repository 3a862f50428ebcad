"""fftconvolve and FFTConvolve on the GPU: parity with the float64 oracle (tests/conv_oracle.py) and the reference
fixture (tests/golden/make_conv_golden.py), block-size edges, strides, broadcasting, bitwise properties, gradients
under differentiable(filtering=True), and what must raise.

The parity bar is evidence-based: the reference's own float32 error against the float64 oracle is measured on the same
inputs (the installed torchaudio's fftconvolve on the same CUDA tensors: three cuFFT transforms of the full length), and
ours may be at most twice that plus 2e-6 of the exact output's rms."""
import os

import numpy as np
import pytest
import torch

import conv_oracle as O

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "conv_ref_cases.npz")
MODES = ("full", "valid", "same")


@pytest.fixture(scope="module", autouse=True)
def _release_device_memory():
    """The full-size cases and the cuFFT reference arm leave gigabytes in the caching allocator and the cuFFT plan
    cache; give them back when the module ends, so later modules start from the state they would see without it."""
    yield
    torch.cuda.synchronize()
    torch.backends.cuda.cufft_plan_cache.clear()
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
    got = F().fftconvolve(x, y, mode)
    exact = O.fftconvolve(x.double().cpu().numpy(), y.double().cpu().numpy(), mode)
    check_bar(got, exact, ta().fftconvolve(x, y, mode), what)
    return got


# ---- parity ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("block", (256, 512, 1024, 2048))
@pytest.mark.parametrize("dk", (-1, 0, 1))
def test_block_edges(block, dk, mode):
    """K at B - 1, B and B + 1 of each block size (B + 1 moves to the next size, or to P = 2 at 2048)."""
    k = block + dk
    x, y = randn(3, 6000 + block, seed=k), randn(3, k, seed=k + 1)
    parity(x, y, mode, f"K={k} {mode}")


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("taps", (255, 2 * 2048, 24 * 2048 - 100))
def test_partitions(taps, mode):
    """P = 1, 2 and 24."""
    x, y = randn(2, 60000, seed=taps), randn(2, taps, seed=1)
    parity(x, y, mode, f"{taps} taps {mode}")


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("n, m", [(1, 1), (1, 700), (700, 1), (1000, 300), (300, 1000), (777, 777), (100, 3000),
                                  (5000, 4999), (300, 200)])
def test_shapes(n, m, mode):
    """1-sample operands, N < M (the swap), N == M, N > M, signals shorter than one block."""
    parity(randn(2, n, seed=n), randn(2, m, seed=m + 7), mode, f"{n} x {m} {mode}")


@pytest.mark.parametrize("mode", MODES)
def test_mid_block_starts(mode):
    """"same" with an odd filter and "valid" start at min - 1: outputs begin mid-block."""
    for m in (301, 1500, 2600):
        parity(randn(2, 9000, seed=m), randn(2, m, seed=m + 1), mode, f"m={m} {mode}")


@pytest.mark.parametrize("mode", MODES)
def test_broadcasting(mode):
    x, y = randn(3, 1, 5000, seed=1), randn(1, 4, 900, seed=2)
    got = parity(x, y, mode, f"(3,1,T) * (1,4,M) {mode}")
    assert got.shape[:2] == (3, 4)
    parity(randn(2, 1, 3, 1, 700), randn(1, 5, 1, 2, 2100), mode, f"4-D {mode}")
    parity(randn(4000), randn(300), mode, f"1-D {mode}")


def test_strided_and_offset_views():
    base = randn(4, 3, 12000, seed=3)
    x = base[:, 1, 1000:11000]  # row stride 36000, offset 1000 + 12000
    y = randn(2000, 4, seed=4).t()[:, 5:1805]  # non-unit time stride: made contiguous
    for mode in MODES:
        parity(x, y, mode, f"views {mode}")
        parity(x[::2], randn(2, 1, 333, seed=5)[:, 0], mode, f"row step {mode}")


def test_fixture_cases():
    if not os.path.exists(GOLDEN):
        pytest.skip("no fixture")
    with np.load(GOLDEN) as z:
        ref = {k: z[k] for k in z.files}
    for key in ref:
        if not key.startswith("out_"):
            continue
        case = key[4:]
        x, y, mode = ref[f"x_{case}"], ref[f"y_{case}"], str(ref[f"mode_{case}"])
        got = F().fftconvolve(torch.as_tensor(x).cuda(), torch.as_tensor(y).cuda(), mode)
        check_bar(got, O.fftconvolve(x, y, mode), ref[key], case)


@pytest.mark.parametrize("shared", (False, True))
def test_full_size_rir(shared):
    """64 x 160 000 with 8 000-tap RIRs, per row or one shared."""
    x = randn(64, 160000, seed=11)
    y = randn(1 if shared else 64, 8000, seed=12) * torch.exp(-torch.arange(8000, device="cuda") / 2000.0)
    parity(x, y, "full", f"full size shared={shared}")


# ---- properties --------------------------------------------------------------------------------------------------
def test_bitwise_properties():
    x, y = randn(8, 30000, seed=21), randn(8, 3000, seed=22)
    a = F().fftconvolve(x, y)
    assert torch.equal(a, F().fftconvolve(x, y)), "rerun"
    for rows in ([3], [0, 5], [7, 1, 2]):
        alone = F().fftconvolve(x[rows], y[rows])
        assert torch.equal(alone, a[rows]), rows
    ys = randn(1, 3000, seed=23)
    assert torch.equal(F().fftconvolve(x, ys), F().fftconvolve(x, ys.expand(8, 3000).contiguous())), "broadcast"
    assert torch.equal(F().fftconvolve(ys, x), F().fftconvolve(ys.expand(8, 3000).contiguous(), x)), "broadcast x"
    import audio_b200
    import audio_b200.transforms as T

    for mode in MODES:
        assert torch.equal(T.FFTConvolve(mode)(x, y), F().fftconvolve(x, y, mode)), mode
    with audio_b200.differentiable(filtering=True):
        xg = x.clone().requires_grad_()
        assert torch.equal(F().fftconvolve(xg, y), a), "forward with grad"


# ---- gradients ---------------------------------------------------------------------------------------------------
def grads(x, y, g, mode):
    import audio_b200

    xg, yg = x.clone().requires_grad_(), y.clone().requires_grad_()
    with audio_b200.differentiable(filtering=True):
        (F().fftconvolve(xg, yg, mode) * g).sum().backward()
    return xg.grad, yg.grad


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("shapes", [((4, 6000), (4, 700)), ((4, 700), (4, 6000)), ((3, 1, 5000), (1, 2, 2500)),
                                    ((1, 2, 900), (3, 1, 4100)), ((2, 3000), (2, 3000))])
def test_gradients_match_oracle(shapes, mode):
    (xs, ys) = shapes
    x, y = randn(*xs, seed=31), randn(*ys, seed=32)
    out_shape = F().fftconvolve(x, y, mode).shape
    g = randn(*out_shape, seed=33)
    gx, gy = grads(x, y, g, mode)
    ex, ey = O.vjp(x.double().cpu().numpy(), y.double().cpu().numpy(), g.double().cpu().numpy(), mode)
    # the reference's float32 autograd (cuFFT) on the same tensors
    xr, yr = x.clone().requires_grad_(), y.clone().requires_grad_()
    (ta().fftconvolve(xr, yr, mode) * g).sum().backward()
    check_bar(gx, ex, xr.grad, f"dx {shapes} {mode}")
    check_bar(gy, ey, yr.grad, f"dy {shapes} {mode}")


def test_adjoint_identity_full_size():
    x, y = randn(64, 160000, seed=41), randn(64, 8000, seed=42) / 30
    g = randn(64, 167999, seed=43)
    gx, gy = grads(x, y, g, "full")
    out = F().fftconvolve(x, y).double()
    lhs = float((g.double() * out).sum())
    for name, v, d in (("x", x, gx), ("y", y, gy)):
        rhs = float((v.double() * d.double()).sum())
        assert abs(lhs - rhs) <= 1e-5 * (abs(lhs) + float((g.double() * out).abs().sum()) * 1e-3), (name, lhs, rhs)


def test_forward_only_and_double_backward():
    import audio_b200

    x, y = randn(2, 1000).requires_grad_(), randn(2, 100)
    with pytest.raises(RuntimeError, match=r"forward-only.*filtering=True"):
        F().fftconvolve(x, y)
    with audio_b200.differentiable(filtering=True):
        out = F().fftconvolve(x, y)
        (gx,) = torch.autograd.grad(out.sum(), x, create_graph=True)
        with pytest.raises(RuntimeError):
            gx.sum().backward()


# ---- errors ------------------------------------------------------------------------------------------------------
def test_errors():
    f = F()
    with pytest.raises(ValueError, match=r"The operands must be the same dimension \(got 3 and 2\)\."):
        f.fftconvolve(randn(2, 3, 10), randn(3, 10))
    with pytest.raises(ValueError, match="Leading dimensions of x and y are not broadcastable"):
        f.fftconvolve(randn(3, 10), randn(2, 4))
    with pytest.raises(ValueError, match=r"Unrecognized mode value 'foo'\. Please specify one of \['full', 'valid', 'same'\]\."):
        f.fftconvolve(randn(3, 10), randn(3, 4), "foo")
    with pytest.raises(RuntimeError, match="not supported.*128"):
        f.fftconvolve(randn(1, 128 * 2048 + 1), randn(1, 128 * 2048 + 5))
    assert f.fftconvolve(randn(1, 300000), randn(1, 128 * 2048)).shape == (1, 300000 + 128 * 2048 - 1)
    with pytest.raises(RuntimeError, match="no CPU or ATen fallback"):
        f.fftconvolve(torch.zeros(2, 10), torch.zeros(2, 3))
    with pytest.raises(TypeError, match="float32"):
        f.fftconvolve(randn(2, 10).double(), randn(2, 3).double())
    import audio_b200.transforms as T

    with pytest.raises(ValueError, match="Unrecognized mode value"):
        T.FFTConvolve("circular")


def test_empty_operands_as_reference():
    """Zero-length operands: the reference's output shape (zeros), or its torch.fft error when N + M - 1 < 1."""
    for n, m in ((0, 5), (5, 0), (0, 1), (0, 0)):
        for mode in MODES:
            try:
                exp = ta().fftconvolve(torch.zeros(2, n), torch.ones(2, m), mode)
            except RuntimeError as e:
                with pytest.raises(RuntimeError, match=str(e).replace("(", r"\(").replace(")", r"\)")):
                    F().fftconvolve(torch.zeros(2, n).cuda(), torch.ones(2, m).cuda(), mode)
                continue
            got = F().fftconvolve(torch.zeros(2, n).cuda(), torch.ones(2, m).cuda(), mode)
            assert got.shape == exp.shape and not got.any(), (n, m, mode)
