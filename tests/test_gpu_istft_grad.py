"""Spectrogram gradients of InverseSpectrogram / F.inverse_spectrogram on the GPU, inside
audio_b200.differentiable(inverse=True).

n_fft 256 / 512 / 1024 take the COMPLEX Spectrogram kernel in its iSTFT-adjoint variant (one kernel); every other size
the composition of the g / env prescale kernel, the forward COMPLEX kernel and a per-bin scale kernel."""
import numpy as np
import pytest
import torch

import audio_b200
import audio_b200.functional as F
import audio_b200.transforms as T
from audio_b200 import _ops
from audio_b200._plans import FrontendPlan
from oracle import frontend_oracle as O

import grad_oracle as GV
import istft_grad_oracle as V

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")


def close(got, exp, rel=1e-4):
    got = got.detach().cpu().numpy().astype(np.complex128)
    err = np.abs(got - exp)
    tol = rel * np.abs(exp) + rel * float(np.sqrt(np.mean(np.abs(exp) ** 2)))
    assert (err <= tol).all(), f"max err {err.max():.3e}, worst ratio {(err / tol).max():.3f}"


def _window(win_length, seed=0):
    rng = np.random.default_rng(seed)
    return O.hann_window(win_length) + 0.1 * rng.random(win_length)


def _rand_complex(shape, gen):
    return torch.complex(torch.randn(shape, generator=gen), torch.randn(shape, generator=gen))


CASES = [
    # n_fft, hop, win_length, pad, length ("short" / "long" / None), normalized, center
    (256, 64, None, 0, None, False, True),
    (512, 128, None, 0, None, False, True),
    (1024, 256, None, 0, None, False, True),
    (1024, 256, None, 7, "long", False, True),
    (512, 100, 400, 13, "short", "window", True),
    (256, 60, 200, 5, "short", "frame_length", True),
    (1024, 300, None, 0, None, True, False),
    (512, 128, None, 0, "short", False, False),
    (400, 100, None, 3, "short", False, True),
    (2048, 512, None, 0, None, False, True),
    (2048, 512, None, 0, "long", "window", False),
]


def _length(kind, n_fft, hop, frames, center):
    full = n_fft + hop * (frames - 1) - (2 * (n_fft // 2) if center else 0)
    return None if kind is None else (full - 3 * hop - 7 if kind == "short" else full + 200)


@pytest.mark.parametrize("case", CASES, ids=lambda c: "-".join(str(v) for v in c))
@pytest.mark.parametrize("lead", [(), (3,), (2, 2)], ids=["1d", "2d", "3d"])
def test_inverse_spectrogram_grad(case, lead):
    n_fft, hop, win_length, pad, kind, normalized, center = case
    win_length = win_length or n_fft
    frames = 1 + 9000 // hop
    length = _length(kind, n_fft, hop, frames, center)
    gen = torch.Generator().manual_seed(n_fft + hop + len(lead))
    z = _rand_complex(lead + (n_fft // 2 + 1, frames), gen)
    mod = T.InverseSpectrogram(n_fft=n_fft, win_length=win_length, hop_length=hop, pad=pad, normalized=normalized,
                               center=center).to(DEV)
    mod.window.copy_(torch.tensor(_window(win_length), dtype=torch.float32))
    with audio_b200.differentiable(inverse=True):
        zt = z.to(DEV).requires_grad_()
        y = mod(zt, length)
        g = torch.randn(y.shape, generator=gen)
        y.backward(g.to(DEV))
        # the functional entry point computes the same
        zf = z.to(DEV).requires_grad_()
        F.inverse_spectrogram(zf, length, pad, mod.window, n_fft, hop, win_length, normalized, center).backward(g.to(DEV))
    assert zt.grad.shape == z.shape and zt.grad.dtype == torch.complex64
    exp = V.inverse_spectrogram_vjp(g.double().numpy(), frames, length, pad, mod.window.double().cpu().numpy(), n_fft, hop,
                                    win_length, normalized, center)
    close(zt.grad, exp)
    assert torch.equal(zf.grad, zt.grad)


@pytest.mark.parametrize("n_fft", [1024, 400])
def test_frame_major_input_and_expanded_or_strided_grads(n_fft):
    """The transposed view our own forward returns as input; expanded (stride 0) and strided upstream gradients."""
    hop, frames, rows = n_fft // 4, 50, 3
    gen = torch.Generator().manual_seed(11)
    leaf = _rand_complex((rows, frames, n_fft // 2 + 1), gen).to(DEV).requires_grad_()
    mod = T.InverseSpectrogram(n_fft=n_fft, hop_length=hop).to(DEV)
    w = mod.window.double().cpu().numpy()
    with audio_b200.differentiable(inverse=True):
        y = mod(leaf.transpose(1, 2))
        y.sum().backward()  # the upstream gradient is ones expanded: every stride 0
    exp = V.inverse_spectrogram_vjp(np.ones(tuple(y.shape)), frames, None, 0, w, n_fft, hop, n_fft)
    close(leaf.grad.transpose(1, 2), exp)
    big = torch.randn(rows, 2 * y.shape[-1] + 1, generator=gen)
    g = big[:, 1::2]  # strided, and not 16-byte aligned
    leaf.grad = None
    with audio_b200.differentiable(inverse=True):
        mod(leaf.transpose(1, 2)).backward(g.to(DEV))
    close(leaf.grad.transpose(1, 2), V.inverse_spectrogram_vjp(g.double().numpy(), frames, None, 0, w, n_fft, hop, n_fft))
    row = torch.randn(1, y.shape[-1], generator=gen)  # one row expanded over the batch: row stride 0
    leaf.grad = None
    with audio_b200.differentiable(inverse=True):
        mod(leaf.transpose(1, 2)).backward(row.expand(rows, -1).to(DEV))
    close(leaf.grad.transpose(1, 2),
          V.inverse_spectrogram_vjp(row.expand(rows, -1).double().numpy(), frames, None, 0, w, n_fft, hop, n_fft))


def test_odd_n_fft_through_the_op():
    """Odd n_fft, as torch.istft takes it: the forward inverts through the Stockham frame stage, the adjoint takes the
    composition path."""
    n_fft, hop, frames, rows, start = 77, 20, 40, 2, 38
    window = _window(n_fft, 3)
    window_t = torch.tensor(window, dtype=torch.float32, device=DEV)
    plan = FrontendPlan(FrontendPlan.make_desc(n_fft, n_fft, hop, 0, True, "reflect", True, False, False, 2.0))
    ws = plan.workspace(window_t, None, None)
    gen = torch.Generator().manual_seed(n_fft)
    w32 = np.asarray(torch.tensor(window, dtype=torch.float32), dtype=np.float64)
    spec = _rand_complex((rows, n_fft // 2 + 1, frames), gen)
    y = F.inverse_spectrogram(spec.to(DEV), None, 0, window_t, n_fft, hop, n_fft, False)
    close(y, O.inverse_spectrogram(spec.numpy(), None, 0, w32, n_fft, hop, n_fft))
    g_len = n_fft + hop * (frames - 1) - 2 * start
    assert tuple(y.shape) == (rows, g_len)
    g = torch.randn(rows, g_len, generator=gen)
    got = _ops.istft_backward(g.to(DEV), ws, *plan._packed_desc(), start, frames)
    got = torch.view_as_complex(got).transpose(1, 2)
    close(got, V.inverse_spectrogram_vjp(g.double().numpy(), frames, None, 0, w32, n_fft, hop, n_fft))


def _full_size():
    gen = torch.Generator(device=DEV).manual_seed(7)
    z = torch.complex(torch.randn(256, 513, 626, device=DEV, generator=gen),
                      torch.randn(256, 513, 626, device=DEV, generator=gen))
    return T.InverseSpectrogram(n_fft=1024, hop_length=256).to(DEV), z, torch.randn(256, 160000, device=DEV, generator=gen)


def _grad(mod, z, g):
    with audio_b200.differentiable(inverse=True):
        zt = z.detach().clone().requires_grad_()
        y = mod(zt)
        y.backward(g)
    return y, zt.grad


def test_full_size_adjoint_deterministic_and_row_independent():
    """256 rows x 626 frames x 513 bins, n_fft 1024, hop 256: sum g istft(Z) = sum Re(conj(grad) Z); bit-identical
    reruns; any rows alone give bit for bit the gradient they get in the batch."""
    mod, z, g = _full_size()
    y, a = _grad(mod, z, g)
    lhs = (g.double() * y.double()).sum().item()
    rhs = (a.real.double() * z.real.double() + a.imag.double() * z.imag.double()).sum().item()
    assert abs(lhs - rhs) <= 1e-5 * (g.double() * y.double()).abs().sum().item()
    _, b = _grad(mod, z, g)
    assert torch.equal(a, b)
    _, part = _grad(mod, z[37:42].clone(), g[37:42].clone())
    assert torch.equal(part, a[37:42])
    assert torch.isfinite(torch.view_as_real(a)).all()
    assert (a[:, 0].imag == 0).all() and (a[:, 512].imag == 0).all()


def test_vocos_style_chain():
    """Leaf spectrogram -> InverseSpectrogram -> MelSpectrogram -> L1 loss, against the numpy composition of the two
    VJPs (the mel VJP is evaluated at the waveform the GPU produced)."""
    gen = torch.Generator().manual_seed(21)
    n_fft, hop, frames = 1024, 256, 80
    z = (_rand_complex((2, n_fft // 2 + 1, frames), gen) * 3.0).to(DEV).requires_grad_()
    inv = T.InverseSpectrogram(n_fft=n_fft, hop_length=hop).to(DEV)
    mel = T.MelSpectrogram(22050, n_fft=n_fft, hop_length=hop, n_mels=80).to(DEV)
    target = torch.rand(2, 80, frames, generator=gen).to(DEV)
    with audio_b200.differentiable(inverse=True):
        y = inv(z)
        m = mel(y)
        loss = (m - target).abs().mean()
        loss.backward()
    gm = (torch.sign(m - target) / m.numel()).detach().double().cpu().numpy()
    gy = GV.mel_spectrogram_vjp(y.detach().double().cpu().numpy(), gm, 22050, n_fft=n_fft, hop_length=hop,
                                fb=mel.mel_scale.fb.double().cpu().numpy())
    exp = V.inverse_spectrogram_vjp(gy, frames, None, 0, inv.window.double().cpu().numpy(), n_fft, hop, n_fft)
    close(z.grad, exp)


def test_window_edited_after_forward():
    gen = torch.Generator().manual_seed(6)
    z = _rand_complex((2, 513, 40), gen).to(DEV)
    mod = T.InverseSpectrogram(n_fft=1024, hop_length=256).to(DEV)
    g = torch.randn(2, 256 * 39, generator=gen).to(DEV)
    _, ref = _grad(mod, z, g)
    with audio_b200.differentiable(inverse=True):
        zt = z.clone().requires_grad_()
        y = mod(zt)
        with torch.no_grad():
            mod.window.mul_(3.0)
        mod(z)  # a forward in between rebuilds the workspace
        y.backward(g)
    assert torch.equal(zt.grad, ref)


def test_what_still_raises():
    x = torch.randn(2, 8000, device=DEV)
    spec = T.Spectrogram(n_fft=512, power=None).to(DEV)(x)
    mag = spec.abs()
    with audio_b200.differentiable():  # without the keyword the inverse stays forward-only
        with pytest.raises(RuntimeError, match=r"forward-only.*differentiable\(inverse=True\)"):
            T.InverseSpectrogram(n_fft=512).to(DEV)(spec.clone().requires_grad_())
    with audio_b200.differentiable(inverse=True):
        for fn in (
            lambda: T.GriffinLim(n_fft=512, n_iter=2).to(DEV)(mag.clone().requires_grad_()),
            lambda: T.TimeStretch(n_freq=257, fixed_rate=1.3).to(DEV)(spec.clone().requires_grad_()),
            lambda: F.phase_vocoder(spec.clone().requires_grad_(), 1.3,
                                    torch.linspace(0, 3.14159 * 128, 257, device=DEV)[..., None]),
            lambda: T.PitchShift(16000, 4).to(DEV)(x.clone().requires_grad_()),
        ):
            with pytest.raises(RuntimeError, match="forward-only"):
                fn()
        mod = T.InverseSpectrogram(n_fft=512).to(DEV)
        mod.window.requires_grad_()
        with pytest.raises(RuntimeError, match="window requires grad"):
            mod(spec.clone().requires_grad_())
    with pytest.raises(RuntimeError, match="forward-only"):  # switched off again
        T.InverseSpectrogram(n_fft=512).to(DEV)(spec.clone().requires_grad_())


def test_double_backward_raises():
    spec = T.Spectrogram(n_fft=512, power=None).to(DEV)(torch.randn(2, 8000, device=DEV))
    with audio_b200.differentiable(inverse=True):
        z = spec.clone().requires_grad_()
        y = T.InverseSpectrogram(n_fft=512).to(DEV)(z)
        (gz,) = torch.autograd.grad(y.pow(2).sum(), z, create_graph=True)
        with pytest.raises(RuntimeError):
            gz.abs().sum().backward()
