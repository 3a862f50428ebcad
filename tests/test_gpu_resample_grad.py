"""Waveform gradients of Resample / F.resample / Speed / SpeedPerturbation on the GPU, inside
audio_b200.differentiable(resample=True).

Ratios whose tables and tile fit (new' <= 1024 phases, staged g rows + D tile within shared memory) take
resample_backward_mma_kernel; 2003 -> 1999 (new' > 1024) and 2003 -> 1000 (a 16-frame tile of g rows plus D exceeds
shared memory) take resample_backward_direct_kernel."""
import numpy as np
import pytest
import torch
from golden_cases import RESAMPLE

import audio_b200
import audio_b200.functional as F
import audio_b200.transforms as T
from oracle import frontend_oracle as O

import grad_oracle as GV
import resample_grad_oracle as V

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")

CASES = {key: (kw, cut) for key, (cut, kw) in RESAMPLE.items()}
CASES["rs_2003_1999"] = (dict(orig_freq=2003, new_freq=1999), None)
CASES["rs_2003_1000"] = (dict(orig_freq=2003, new_freq=1000), None)


def _bar(got, exp):
    got = got.detach().double().cpu().numpy()
    assert got.shape == exp.shape
    err = np.abs(got - exp).max()
    assert err <= 1e-4 * np.abs(exp).max(), f"max err {err:.3e} vs max |e| {np.abs(exp).max():.3e}"


def close(got, exp, rel=1e-4):
    got = got.detach().double().cpu().numpy()
    err = np.abs(got - exp)
    tol = rel * np.abs(exp) + rel * float(np.sqrt(np.mean(np.abs(exp) ** 2)))
    assert (err <= tol).all(), f"max err {err.max():.3e}, worst ratio {(err / tol).max():.3f}"


def _vjp(mod, g, length):
    k = mod.kernel.double().cpu().numpy()
    return V.resample_vjp(g.double().cpu().numpy(), mod.orig_freq, mod.new_freq, mod.gcd, k, mod.width, length)


def _grad(fn, x, g):
    with audio_b200.differentiable(resample=True):
        xt = x.detach().clone().requires_grad_()
        y = fn(xt)
        y.backward(g)
    return y, xt.grad


@pytest.mark.parametrize("key", sorted(CASES))
@pytest.mark.parametrize("lead", [(), (3,), (2, 2)], ids=["1d", "2d", "3d"])
def test_resample_grad(key, lead):
    kw, cut = CASES[key]
    length = cut if cut is not None else 6001
    gen = torch.Generator().manual_seed(len(key) + len(lead))
    x = torch.randn(lead + (length,), generator=gen).to(DEV)
    mod = T.Resample(**kw).to(DEV)
    out_len = O.resample_len(length, mod.orig_freq // mod.gcd, mod.new_freq // mod.gcd)
    g = torch.randn(lead + (out_len,), generator=gen).to(DEV)
    y, gx = _grad(mod, x, g)
    assert y.shape == lead + (out_len,) and gx.shape == x.shape
    _bar(gx, _vjp(mod, g, length))
    # F.resample builds its taps per call, in the input's dtype on its device (as the reference does)
    method = kw.get("resampling_method", "sinc_interp_hann")
    lpw, rolloff = kw.get("lowpass_filter_width", 6), kw.get("rolloff", 0.99)
    _, gf = _grad(lambda t: F.resample(t, kw["orig_freq"], kw["new_freq"], lpw, rolloff, method), x, g)
    kf, wf = F._get_sinc_resample_kernel(kw["orig_freq"], kw["new_freq"], mod.gcd, lpw, rolloff, method, None, DEV,
                                         torch.float32)
    exp = V.resample_vjp(g.double().cpu().numpy(), kw["orig_freq"], kw["new_freq"], mod.gcd,
                         kf.double().cpu().numpy(), wf, length)
    _bar(gf, exp)


def test_speed_and_perturbation_match_resample():
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(3, 8000, generator=gen).to(DEV)
    for factor, (src, dst) in ((1.1, (11, 10)), (0.9, (9, 10))):
        ref_mod = T.Resample(src, dst).to(DEV)
        g = torch.randn(3, O.resample_len(8000, src, dst), generator=gen).to(DEV)
        _, ref = _grad(ref_mod, x, g)
        _, gs = _grad(lambda t: T.Speed(16000, factor).to(DEV)(t)[0], x, g)
        assert torch.equal(gs, ref)
        _, gfs = _grad(lambda t: F.speed(t, 16000, factor)[0], x, g)
        _bar(gfs, _vjp(ref_mod, g, 8000))  # F.speed -> F.resample: float32 taps built per call
        torch.manual_seed(0)
        _, gp = _grad(lambda t: T.SpeedPerturbation(16000, [factor]).to(DEV)(t)[0], x, g)
        assert torch.equal(gp, ref)


def test_reference_autograd_cases():
    """The reference's own autograd cases: Resample 8000 <-> 4000 on 2 x 400, Speed(1000, 1.1) and
    SpeedPerturbation(1000, [0.9]) on (3, 2, 200)."""
    gen = torch.Generator().manual_seed(9)
    x = torch.randn(2, 400, generator=gen).to(DEV)
    for o, n in ((8000, 4000), (4000, 8000)):
        mod = T.Resample(o, n).to(DEV)
        g = torch.randn(2, O.resample_len(400, o // mod.gcd, n // mod.gcd), generator=gen).to(DEV)
        _bar(_grad(mod, x, g)[1], _vjp(mod, g, 400))
    x3 = torch.randn(3, 2, 200, generator=gen).to(DEV)
    for mod in (T.Speed(1000, 1.1).to(DEV), T.SpeedPerturbation(1000, [0.9]).to(DEV)):
        res = mod.resampler if isinstance(mod, T.Speed) else mod.speeders[0].resampler
        g = torch.randn(3, 2, O.resample_len(200, res.orig_freq // res.gcd, res.new_freq // res.gcd), generator=gen).to(DEV)
        _bar(_grad(lambda t: mod(t)[0], x3, g)[1], _vjp(res, g, 200))


@pytest.mark.parametrize("kw", [dict(orig_freq=44100, new_freq=16000), dict(orig_freq=2003, new_freq=1999)],
                         ids=["mma", "direct"])
def test_expanded_strided_and_unaligned_grads(kw):
    mod = T.Resample(**kw).to(DEV)
    gen = torch.Generator().manual_seed(3)
    rows, length = 3, 9000
    x = torch.randn(rows, length, generator=gen).to(DEV)
    out_len = O.resample_len(length, mod.orig_freq // mod.gcd, mod.new_freq // mod.gcd)
    with audio_b200.differentiable(resample=True):
        xt = x.clone().requires_grad_()
        mod(xt).sum().backward()  # ones expanded: every stride 0
    _bar(xt.grad, _vjp(mod, torch.ones(rows, out_len), length))
    big = torch.randn(rows, 2 * out_len + 1, generator=gen).to(DEV)
    _, gs = _grad(mod, x, big[:, 1::2])  # element stride 2
    _bar(gs, _vjp(mod, big[:, 1::2], length))
    row = torch.randn(1, out_len, generator=gen).to(DEV)
    _, ge = _grad(mod, x, row.expand(rows, -1))  # row stride 0
    _bar(ge, _vjp(mod, row.expand(rows, -1), length))
    g = torch.randn(rows, out_len, generator=gen).to(DEV)
    ref = _grad(mod, x, g)[1]
    for off in range(4):  # g at every 4-byte offset from a 16-byte boundary: the same arithmetic
        view = torch.empty(rows, out_len + 8, device=DEV)[:, off:off + out_len]
        view.copy_(g)
        assert view.stride(1) == 1 and view.data_ptr() % 16 == 4 * off
        assert torch.equal(_grad(mod, x, view)[1], ref), off


def test_forward_with_grad_matches_no_grad_forward():
    for kw in (dict(orig_freq=44100, new_freq=16000), dict(orig_freq=16000, new_freq=44100), dict(orig_freq=2003, new_freq=1999)):
        mod = T.Resample(**kw).to(DEV)
        x = torch.randn(2, 3, 7001, generator=torch.Generator().manual_seed(1)).to(DEV)
        y0 = mod(x)
        with audio_b200.differentiable(resample=True):
            y1 = mod(x.clone().requires_grad_())
        assert y1.requires_grad and torch.equal(y0, y1.detach())
        assert y0.stride() == y1.stride()


def _full_size():
    gen = torch.Generator(device=DEV).manual_seed(7)
    x = torch.randn(1024, 220500, device=DEV, generator=gen)
    mod = T.Resample(44100, 16000, resampling_method="sinc_interp_kaiser").to(DEV)
    g = torch.randn(1024, O.resample_len(220500, 441, 160), device=DEV, generator=gen)
    return mod, x, g


def test_full_size_adjoint_deterministic_and_row_independent():
    """Config 3 (1024 x 220 500, 44.1 -> 16 kHz kaiser): sum g R(x) = sum x R^T(g); bit-identical reruns; rows alone
    give bit for bit their gradient in the batch."""
    mod, x, g = _full_size()
    y, a = _grad(mod, x, g)
    gy = g.double() * y.double()
    lhs = gy.sum().item()
    rhs = (x.double() * a.double()).sum().item()
    assert abs(lhs - rhs) <= 1e-5 * gy.abs().sum().item()
    del gy, y
    _, b = _grad(mod, x, g)
    assert torch.equal(a, b)
    del b
    _, part = _grad(mod, x[37:42].clone(), g[37:42].clone())
    assert torch.equal(part, a[37:42])
    _, one = _grad(mod, x[1000:1001].clone(), g[1000:1001].clone())
    assert torch.equal(one, a[1000:1001])
    assert torch.isfinite(a).all()


@pytest.mark.parametrize("kw", [dict(orig_freq=44100, new_freq=16000), dict(orig_freq=16000, new_freq=8000),
                                dict(orig_freq=16000, new_freq=44100), dict(orig_freq=2003, new_freq=1999)],
                         ids=["44k1_16k", "16k_8k", "16k_44k1", "direct"])
def test_shift_covariance(kw):
    """Shifting g by n' outputs (one frame) shifts the interior gradient by o' samples, bit for bit."""
    mod = T.Resample(**kw).to(DEV)
    o, n = mod.orig_freq // mod.gcd, mod.new_freq // mod.gcd
    length = max(20000, 12 * o)
    out_len = O.resample_len(length, o, n)
    gen = torch.Generator().manual_seed(4)
    x = torch.randn(2, length, generator=gen).to(DEV)
    g1 = torch.randn(2, out_len, generator=gen).to(DEV)
    g2 = torch.randn(2, out_len, generator=gen).to(DEV)
    g2[:, n:] = g1[:, :-n]
    a = _grad(mod, x, g1)[1]
    b = _grad(mod, x, g2)[1]
    margin = 2 * (2 * mod.width + o)
    assert torch.equal(b[:, margin + o:length - margin], a[:, margin:length - margin - o])


def test_resample_mel_chain():
    """48 kHz leaf -> Resample(48000, 16000) -> MelSpectrogram -> L1, against the numpy composition of resample_vjp and
    mel_spectrogram_vjp (the mel VJP evaluated at the waveform the GPU produced)."""
    gen = torch.Generator().manual_seed(21)
    length = 48000
    x = (torch.randn(2, length, generator=gen) * 0.3).to(DEV).requires_grad_()
    rs = T.Resample(48000, 16000).to(DEV)
    mel = T.MelSpectrogram(16000, n_fft=512, hop_length=128, n_mels=64).to(DEV)
    with audio_b200.differentiable(resample=True):
        y = rs(x)
        m = mel(y)
        target = torch.rand(m.shape, generator=gen).to(DEV)
        loss = (m - target).abs().mean()
        loss.backward()
    gm = (torch.sign(m - target) / m.numel()).detach().double().cpu().numpy()
    gy = GV.mel_spectrogram_vjp(y.detach().double().cpu().numpy(), gm, 16000, n_fft=512, hop_length=128, n_mels=64,
                                fb=mel.mel_scale.fb.double().cpu().numpy())
    close(x.grad, _vjp(rs, torch.from_numpy(gy), length))


def test_kernel_edited_after_forward():
    gen = torch.Generator().manual_seed(6)
    x = torch.randn(2, 9000, generator=gen).to(DEV)
    mod = T.Resample(44100, 16000).to(DEV)
    g = torch.randn(2, O.resample_len(9000, 441, 160), generator=gen).to(DEV)
    _, ref = _grad(mod, x, g)
    with audio_b200.differentiable(resample=True):
        xt = x.clone().requires_grad_()
        y = mod(xt)
        with torch.no_grad():
            mod.kernel.mul_(3.0)
        mod(xt)  # a forward in between rebuilds both workspaces
        y.backward(g)
    assert torch.equal(xt.grad, ref)


def test_empty_batch():
    mod = T.Resample(44100, 16000).to(DEV)
    with audio_b200.differentiable(resample=True):
        x = torch.randn(0, 1000, device=DEV, requires_grad=True)
        y = mod(x)
        assert tuple(y.shape) == (0, O.resample_len(1000, 441, 160))
        y.sum().backward()
    assert x.grad.shape == x.shape


def test_what_still_raises():
    x = torch.randn(2, 8000, device=DEV)
    with audio_b200.differentiable():  # without the keyword the resampler stays forward-only
        with pytest.raises(RuntimeError, match=r"forward-only.*differentiable\(resample=True\)"):
            T.Resample(16000, 8000).to(DEV)(x.clone().requires_grad_())
    with audio_b200.differentiable(inverse=True):
        with pytest.raises(RuntimeError, match="forward-only"):
            T.Speed(16000, 1.1).to(DEV)(x.clone().requires_grad_())
    spec = T.Spectrogram(n_fft=512, power=None).to(DEV)(x)
    with audio_b200.differentiable(resample=True):
        for fn in (
            lambda: T.PitchShift(16000, 4).to(DEV)(x.clone().requires_grad_()),
            lambda: F.pitch_shift(x.clone().requires_grad_(), 16000, 4),
            lambda: T.TimeStretch(n_freq=257, fixed_rate=1.3).to(DEV)(spec.clone().requires_grad_()),
        ):
            with pytest.raises(RuntimeError, match="forward-only"):
                fn()
        mod = T.Resample(16000, 8000).to(DEV)
        mod.kernel.requires_grad_()
        with pytest.raises(RuntimeError, match="kernel requires grad"):
            mod(x.clone().requires_grad_())
    with pytest.raises(RuntimeError, match="forward-only"):  # switched off again
        T.Resample(16000, 8000).to(DEV)(x.clone().requires_grad_())


def test_double_backward_raises():
    with audio_b200.differentiable(resample=True):
        x = torch.randn(2, 8000, device=DEV, requires_grad=True)
        y = T.Resample(16000, 8000).to(DEV)(x)
        (gx,) = torch.autograd.grad(y.pow(2).sum(), x, create_graph=True)
        with pytest.raises(RuntimeError):
            gx.abs().sum().backward()
