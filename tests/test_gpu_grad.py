"""Waveform gradients of Spectrogram / MelSpectrogram / F.spectrogram on the GPU, inside audio_b200.differentiable().

n_fft 256 / 512 / 1024 (one-sided) take the fused register-FFT backward kernel; every other size, and two-sided output,
the composition of the forward complex kernel, the spectrum VJP kernel and the iSTFT frame stage.  Both end in the
deterministic fold kernel."""
import numpy as np
import pytest
import torch

import audio_b200
import audio_b200.compliance.kaldi as K
import audio_b200.functional as F
import audio_b200.transforms as T
from oracle import frontend_oracle as O

import grad_oracle as V

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")

# p < 2 divides by |X| (p = 1) or scales by |X|^(p-1): a bin whose |X| is a few float32 ulps of the frame's energy gets a
# direction of float32 accuracy relative to |X| itself, so the per-sample bar is relaxed to 1e-3 there; for p = 0.5 the
# factor |X|^-0.5 also amplifies that error (observed up to 1.1e-3), so its bar is 3e-3
BAR = {None: 1e-4, 0.5: 3e-3, 1.0: 1e-3, 2.0: 1e-4, 3.0: 1e-4}


def close(got, exp, rel=1e-4):
    got = got.detach().double().cpu().numpy()
    err = np.abs(got - exp)
    tol = rel * np.abs(exp) + rel * float(np.sqrt(np.mean(exp**2)))
    assert (err <= tol).all(), f"max err {err.max():.3e}, worst ratio {(err / tol).max():.3f}"


def grad_of(fn, x, g):
    with audio_b200.differentiable():
        xt = x.detach().to(DEV, copy=True).requires_grad_()
        y = fn(xt)
        y.backward(g.to(DEV))
    return xt.grad


def _window(win_length, seed=0):
    rng = np.random.default_rng(seed)
    return O.hann_window(win_length) + 0.1 * rng.random(win_length)


SPEC_CASES = [
    # n_fft, hop, win_length, pad, power, normalized, center, pad_mode, onesided
    (256, 64, None, 0, 2.0, False, True, "reflect", True),
    (512, 128, None, 0, 1.0, False, True, "reflect", True),
    (1024, 256, None, 0, 2.0, False, True, "reflect", True),
    (1024, 256, None, 0, None, False, True, "reflect", True),
    (512, 100, 400, 13, 2.0, "window", True, "replicate", True),
    (256, 60, 200, 5, 3.0, "frame_length", True, "circular", True),
    (512, 128, None, 0, 0.5, True, True, "constant", True),
    (1024, 300, None, 0, 2.0, False, False, "reflect", True),
    (2048, 512, None, 0, 2.0, False, True, "reflect", True),
    (2048, 512, None, 0, None, False, True, "reflect", True),
    (400, 100, None, 3, 1.0, False, True, "reflect", True),
    (77, 20, 60, 0, 2.0, True, True, "circular", True),
    (77, 20, None, 0, None, False, True, "reflect", False),
    (512, 128, None, 0, 2.0, False, True, "reflect", False),
    (1024, 256, None, 0, None, "frame_length", True, "replicate", False),
    (97, 31, None, 0, 2.0, False, True, "reflect", True),
    (4096, 1024, None, 0, None, False, True, "reflect", True),
    (2187, 500, None, 0, None, False, True, "reflect", False),
    (600, 150, 401, 0, 2.0, "window", True, "constant", True),
]


@pytest.mark.parametrize("case", SPEC_CASES, ids=lambda c: "-".join(str(v) for v in c))
@pytest.mark.parametrize("shape", [(9000,), (3, 9000), (2, 2, 9000)], ids=["1d", "2d", "3d"])
def test_spectrogram_grad(case, shape):
    n_fft, hop, win_length, pad, power, normalized, center, pad_mode, onesided = case
    win_length = win_length or n_fft
    w = _window(win_length)
    gen = torch.Generator().manual_seed(n_fft + hop)
    x = torch.randn(shape, generator=gen)
    mod = T.Spectrogram(n_fft=n_fft, win_length=win_length, hop_length=hop, pad=pad, power=power, normalized=normalized,
                        center=center, pad_mode=pad_mode, onesided=onesided).to(DEV)
    mod.window.copy_(torch.tensor(w, dtype=torch.float32))
    kw = dict(pad=pad, window=mod.window.double().cpu().numpy(), n_fft=n_fft, hop=hop, win_length=win_length, power=power,
              normalized=normalized, center=center, pad_mode=pad_mode, onesided=onesided)
    y = O.spectrogram(x.numpy(), **kw)
    g = torch.randn(y.shape, generator=gen)
    if power is None:
        g = torch.complex(g, torch.randn(y.shape, generator=gen))
    got = grad_of(mod, x, g)
    close(got, V.spectrogram_vjp(x.double().numpy(), g.numpy(), **kw), BAR[power])
    # the functional entry point computes the same
    got_f = grad_of(lambda t: F.spectrogram(t, pad, mod.window, n_fft, hop, win_length, power, normalized, center, pad_mode,
                                            onesided), x, g)
    assert torch.equal(got_f, got)


@pytest.mark.parametrize("n_fft,hop,n_mels,sr,norm,mel_scale,power", [
    (1024, 256, 80, 16000, None, "htk", 2.0),
    (1024, 256, 80, 22050, "slaney", "slaney", 1.0),
    (512, 128, 64, 16000, None, "htk", 2.0),
    (256, 64, 128, 16000, "slaney", "slaney", 2.0),
    (2048, 512, 128, 16000, None, "htk", 2.0),
    (400, 160, 40, 16000, None, "htk", 1.0),
])
def test_mel_spectrogram_grad(n_fft, hop, n_mels, sr, norm, mel_scale, power):
    gen = torch.Generator().manual_seed(n_mels)
    x = torch.randn(2, 3, 12000, generator=gen)
    mod = T.MelSpectrogram(sr, n_fft=n_fft, hop_length=hop, n_mels=n_mels, norm=norm, mel_scale=mel_scale,
                           power=power).to(DEV)
    fb = mod.mel_scale.fb.double().cpu().numpy()
    y = O.mel_spectrogram(x.numpy(), sr, n_fft=n_fft, hop_length=hop, n_mels=n_mels, power=power, fb=fb)
    g = torch.randn(y.shape, generator=gen)
    got = grad_of(mod, x, g)
    close(got, V.mel_spectrogram_vjp(x.double().numpy(), g.numpy(), sr, n_fft=n_fft, hop_length=hop, power=power, fb=fb),
          BAR[power])


def _config2():
    return T.MelSpectrogram(16000, n_fft=1024, hop_length=256, n_mels=80).to(DEV)


def test_config2_rows_against_oracle():
    mod = _config2()
    gen = torch.Generator().manual_seed(2)
    x = torch.randn(32, 160000, generator=gen)
    g = torch.randn(32, 80, 626, generator=gen)
    got = grad_of(mod, x, g)
    fb = mod.mel_scale.fb.double().cpu().numpy()
    close(got, V.mel_spectrogram_vjp(x.double().numpy(), g.numpy(), 16000, n_fft=1024, hop_length=256, fb=fb))


def test_config2_batch_deterministic_and_row_independent():
    mod = _config2()
    gen = torch.Generator(device=DEV).manual_seed(3)
    x = torch.randn(256, 160000, device=DEV, generator=gen)
    g = torch.randn(256, 80, 626, device=DEV, generator=gen)
    a = grad_of(mod, x, g)
    b = grad_of(mod, x, g)
    assert torch.equal(a, b)
    part = grad_of(mod, x[37:42].clone(), g[37:42].clone())
    assert torch.equal(part, a[37:42])
    assert torch.isfinite(a).all()


@pytest.mark.parametrize("n_fft,onesided", [(1024, True), (2048, True), (400, True), (512, False)])
def test_complex_adjoint(n_fft, onesided):
    """<F x, y> = <x, F^T y> with the forward kernel for F and the backward kernel for F^T."""
    gen = torch.Generator(device=DEV).manual_seed(n_fft)
    mod = T.Spectrogram(n_fft=n_fft, hop_length=n_fft // 4, power=None, onesided=onesided).to(DEV)
    x = torch.randn(4, 20000, device=DEV, generator=gen)
    X = mod(x)
    y = torch.complex(torch.randn(X.shape, device=DEV, generator=gen), torch.randn(X.shape, device=DEV, generator=gen))
    gx = grad_of(mod, x, y)
    lhs = (X.real.double() * y.real.double() + X.imag.double() * y.imag.double()).sum().item()
    rhs = (x.double() * gx.double()).sum().item()
    assert abs(lhs - rhs) <= 1e-5 * (X.abs().double() * y.abs().double()).sum().item()


def test_expanded_and_non_contiguous_grads():
    gen = torch.Generator().manual_seed(4)
    x = torch.randn(3, 9000, generator=gen)
    for n_fft in (512, 400):
        mod = T.Spectrogram(n_fft=n_fft, hop_length=128).to(DEV)
        with audio_b200.differentiable():
            xt = x.to(DEV).requires_grad_()
            mod(xt).sum().backward()
        kw = dict(pad=0, window=mod.window.double().cpu().numpy(), n_fft=n_fft, hop=128, win_length=n_fft, power=2.0)
        y = O.spectrogram(x.numpy(), **kw)
        close(xt.grad, V.spectrogram_vjp(x.double().numpy(), np.ones(y.shape), **kw))
        big = torch.randn(y.shape[:-1] + (2 * y.shape[-1],), generator=gen)
        g = big[..., ::2]  # non-contiguous upstream gradient
        close(grad_of(mod, x, g), V.spectrogram_vjp(x.double().numpy(), g.numpy(), **kw))
    cmod = T.Spectrogram(n_fft=1024, hop_length=256, power=None).to(DEV)
    with audio_b200.differentiable():
        xt = x.to(DEV).requires_grad_()
        cmod(xt).real.sum().backward()
    kw = dict(pad=0, window=cmod.window.double().cpu().numpy(), n_fft=1024, hop=256, win_length=1024, power=None)
    y = O.spectrogram(x.numpy(), **kw)
    close(xt.grad, V.spectrogram_vjp(x.double().numpy(), np.ones(y.shape, dtype=np.complex128), **kw))


@pytest.mark.parametrize("n_fft", [512, 400])
def test_zero_input_nan_rule(n_fft):
    x = torch.zeros(2, 8000)
    for power, nan in ((0.5, True), (1.0, False), (2.0, False)):
        mod = T.Spectrogram(n_fft=n_fft, hop_length=128, power=power).to(DEV)
        g = torch.ones(2, n_fft // 2 + 1, 1 + 8000 // 128)
        got = grad_of(mod, x, g)
        assert torch.isnan(got).all() if nan else (got == 0).all()


def test_nan_stays_in_its_frames():
    """p < 1 with one silent stretch: NaN exactly where torch's gradient is NaN (the partner frame of the shared
    complex transform stays clean)."""
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(1, 8000, generator=gen)
    x[:, 3000:4200] = 0
    for n_fft in (512, 400):
        mod = T.Spectrogram(n_fft=n_fft, hop_length=128, power=0.5).to(DEV)
        kw = dict(pad=0, window=mod.window.double().cpu().numpy(), n_fft=n_fft, hop=128, win_length=n_fft, power=0.5)
        y = O.spectrogram(x.numpy(), **kw)
        g = torch.randn(y.shape, generator=gen)
        got = grad_of(mod, x, g).cpu().numpy()
        exp = V.spectrogram_vjp(x.double().numpy(), g.numpy(), **kw)
        assert np.isnan(exp).any()
        assert (np.isnan(got) == np.isnan(exp)).all()


def test_forward_only_entry_points_still_raise():
    x = torch.randn(2, 8000, device=DEV, requires_grad=True)
    spec = T.Spectrogram(n_fft=512, power=None).to(DEV)(x.detach())
    mag = spec.abs()
    with audio_b200.differentiable():
        for fn in (
            lambda: T.MFCC(16000, n_mfcc=13, melkwargs=dict(n_fft=512, n_mels=40)).to(DEV)(x),
            lambda: T.LFCC(16000, n_lfcc=13, speckwargs=dict(n_fft=512)).to(DEV)(x),
            lambda: T.SpectralCentroid(16000, n_fft=512).to(DEV)(x),
            lambda: T.MelScale(40, 16000, n_stft=257).to(DEV)(mag.clone().requires_grad_()),
            lambda: T.AmplitudeToDB()(x.abs()),
            lambda: T.InverseSpectrogram(n_fft=512).to(DEV)(spec.clone().requires_grad_()),
            lambda: T.GriffinLim(n_fft=512, n_iter=2).to(DEV)(mag.clone().requires_grad_()),
            lambda: T.Resample(16000, 8000).to(DEV)(x),
            lambda: K.fbank_batch(x * 1000),
        ):
            with pytest.raises(RuntimeError, match="forward-only"):
                fn()
        mod = T.Spectrogram(n_fft=512).to(DEV)
        mod.window.requires_grad_()
        with pytest.raises(RuntimeError, match="window requires grad"):
            mod(x)
        mel = T.MelSpectrogram(16000, n_fft=512, n_mels=40).to(DEV)
        mel.mel_scale.fb.requires_grad_()
        with pytest.raises(RuntimeError, match="fb requires grad"):
            mel(x)
    with pytest.raises(RuntimeError, match="forward-only"):  # switched off again
        T.Spectrogram(n_fft=512).to(DEV)(x)


def test_double_backward_raises():
    x = torch.randn(2, 8000, device=DEV, requires_grad=True)
    with audio_b200.differentiable():
        y = T.Spectrogram(n_fft=512).to(DEV)(x)
        (gx,) = torch.autograd.grad(y.sum(), x, create_graph=True)
        with pytest.raises(RuntimeError):
            gx.sum().backward()


@pytest.mark.parametrize("n_fft", [1024, 2048])
def test_window_edited_after_forward(n_fft):
    gen = torch.Generator().manual_seed(6)
    x = torch.randn(2, 12000, generator=gen)
    mod = T.MelSpectrogram(16000, n_fft=n_fft, hop_length=n_fft // 4, n_mels=64).to(DEV)
    g = torch.randn(2, 64, 1 + 12000 // (n_fft // 4), generator=gen).to(DEV)
    ref = grad_of(mod, x, g)
    with audio_b200.differentiable():
        xt = x.to(DEV).requires_grad_()
        y = mod(xt)
        with torch.no_grad():
            mod.spectrogram.window.mul_(3.0)
            mod.mel_scale.fb.mul_(0.5)
        mod(x.to(DEV))  # a forward in between rebuilds the module's workspace
        y.backward(g)
    assert torch.equal(xt.grad, ref)


def test_in_place_edit_of_waveform_is_caught():
    with audio_b200.differentiable():
        x = torch.randn(2, 8000, device=DEV, requires_grad=True)
        w = x * 1.0
        y = T.Spectrogram(n_fft=512).to(DEV)(w)
        w.mul_(2.0)
        with pytest.raises(RuntimeError, match="modified by an inplace operation"):
            y.sum().backward()
