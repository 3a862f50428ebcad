"""Spectrogram gradients of F.phase_vocoder / TimeStretch and waveform gradients of F.pitch_shift / PitchShift on the
GPU, inside audio_b200.differentiable(vocoder=True), against the float64 oracle with the kernels' float32 time grid.

phase_vocoder_backward_kernel walks each (row, bin) backwards once; PitchShift chains the adjoints of crop / pad, the
resampler, the inverse STFT, the phase vocoder and the complex STFT."""
import math
import os

import numpy as np
import pytest
import torch

import audio_b200
import audio_b200.functional as F
import audio_b200.transforms as T

import vocoder_grad_oracle as V
from istft_grad_oracle import inverse_spectrogram_vjp

try:
    import torchaudio.functional as TAF
except Exception:  # noqa: BLE001
    TAF = None

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "vocoder_ref_cases.npz")
RATES = (0.5, 0.7, 0.8, 0.9, 1.3, 2.0, 3.1)


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def _pa(bins, hop=128, device=DEV):
    return torch.linspace(0, math.pi * hop, bins, device=device)[..., None]


def _bar(got, exp, rel=1e-4):
    got = got.detach().cpu().numpy().astype(np.complex128)
    assert got.shape == exp.shape
    assert np.isfinite(got).all()
    err = np.abs(got - exp).max()
    assert err <= rel * np.abs(exp).max(), f"max err {err:.3e} vs max |e| {np.abs(exp).max():.3e}"


def _rand_complex(shape, gen):
    return torch.complex(torch.randn(shape, generator=gen), torch.randn(shape, generator=gen))


def _stretcher(bins, rate, module=False):
    if module:
        return T.TimeStretch(hop_length=128, n_freq=bins, fixed_rate=rate).to(DEV)
    pa = _pa(bins)
    return lambda x: F.phase_vocoder(x, rate, pa)


def _stretch_grad(spec, rate, g, fn=None):
    """(output, spectrogram gradient) of one TimeStretch / F.phase_vocoder call on a leaf copy of ``spec``."""
    fn = _stretcher(spec.shape[-2], rate) if fn is None else fn
    with audio_b200.differentiable(vocoder=True):
        x = spec.detach().clone().requires_grad_() if spec.is_contiguous() else spec.detach().requires_grad_()
        y = fn(x)
        y.backward(g)
    return y, x.grad


def _oracle(spec, g, rate):
    pa = np.linspace(0, math.pi * 128, spec.shape[-2])[:, None]
    return V.phase_vocoder_vjp(spec.detach().cpu().numpy(), g.detach().cpu().numpy(), rate, phase_advance=pa,
                               grid=np.float32)


@pytest.mark.parametrize("rate", RATES)
@pytest.mark.parametrize("layout", ["freq_major", "frame_major"])
def test_time_stretch_grad_golden(golden, rate, layout):
    spec_np = golden["spec"]
    if layout == "freq_major":  # the reference's layout: (rows, freq, frames) contiguous
        spec = torch.from_numpy(spec_np).to(DEV)
    else:  # what Spectrogram(power=None) returns: a transposed view of a frame-major buffer
        spec = torch.from_numpy(np.ascontiguousarray(np.swapaxes(spec_np, -1, -2))).to(DEV).transpose(-1, -2)
    frames_out = int(math.ceil(spec.shape[-1] / rate))
    g = _rand_complex((2, 257, frames_out), torch.Generator().manual_seed(int(rate * 10))).to(DEV)
    fn = _stretcher(257, rate, module=(layout == "freq_major"))
    y, gx = _stretch_grad(spec, rate, g, fn)
    with torch.no_grad():
        assert torch.equal(y, fn(spec))  # the grad path's forward is the no-grad one, bit for bit
    _bar(gx, _oracle(spec, g, rate))


@pytest.mark.parametrize("rate", [0.8, 1.3])
@pytest.mark.parametrize("lead", [(), (2, 3)], ids=["2d", "4d"])
def test_random_spectrogram_and_leading_dims(rate, lead):
    gen = torch.Generator().manual_seed(len(lead))
    spec = _rand_complex(lead + (129, 301), gen).to(DEV)
    frames_out = int(math.ceil(301 / rate))
    g = _rand_complex(lead + (129, frames_out), gen).to(DEV)
    _, gx = _stretch_grad(spec, rate, g)
    assert gx.shape == spec.shape
    _bar(gx, _oracle(spec, g, rate))


@pytest.mark.parametrize("kind", ["expanded", "strided", "conj"])
def test_expanded_and_non_contiguous_grads(golden, kind):
    spec = torch.from_numpy(golden["spec"]).to(DEV)
    rate = 0.8
    frames_out = int(math.ceil(spec.shape[-1] / rate))
    gen = torch.Generator().manual_seed(3)
    if kind == "expanded":
        g = _rand_complex((1, 257, 1), gen).to(DEV).expand(2, 257, frames_out)
    elif kind == "strided":
        g = _rand_complex((2, 257, 2 * frames_out), gen).to(DEV)[..., ::2]
    else:
        g = _rand_complex((2, 257, frames_out), gen).to(DEV).conj()
    _, gx = _stretch_grad(spec, rate, g)
    _bar(gx, _oracle(spec, g.resolve_conj(), rate))


@pytest.mark.parametrize("rate", [0.7, 1.3, 3.1])
def test_exact_zeros_give_exact_zero(rate):
    gen = torch.Generator().manual_seed(11)
    spec = _rand_complex((2, 65, 80), gen)
    spec[0, 3, 4] = 0
    spec[1, :, 0] = 0
    spec[0, :, 20:31] = 0
    spec = spec.to(DEV)
    g = _rand_complex((2, 65, int(math.ceil(80 / rate))), gen).to(DEV)
    _, gx = _stretch_grad(spec, rate, g)
    assert torch.isfinite(torch.view_as_real(gx)).all()
    assert gx[0, 3, 4] == 0 and (gx[1, :, 0] == 0).all() and (gx[0, :, 20:31] == 0).all()
    _bar(gx, _oracle(spec, g, rate))


def test_rate_one_returns_the_input():
    spec = _rand_complex((1, 33, 10), torch.Generator().manual_seed(0)).to(DEV).requires_grad_()
    with audio_b200.differentiable(vocoder=True):
        assert F.phase_vocoder(spec, 1.0, _pa(33)) is spec


@pytest.fixture(scope="module")
def full_size():
    gen = torch.Generator().manual_seed(1251)
    spec = _rand_complex((256, 1251, 257), gen).to(DEV).transpose(1, 2)  # frame-major, as Spectrogram returns it
    return spec


@pytest.mark.parametrize("rate", [0.8, 1.3])
def test_full_size_bitwise_properties(full_size, rate):
    spec = full_size
    frames_out = int(math.ceil(1251 / rate))
    g = _rand_complex((256, 257, frames_out), torch.Generator().manual_seed(int(rate * 10))).to(DEV)
    fn = _stretcher(257, rate)
    y1, g1 = _stretch_grad(spec, rate, g, fn)
    y2, g2 = _stretch_grad(spec, rate, g, fn)
    with torch.no_grad():
        assert torch.equal(y1, fn(spec))
    assert torch.equal(g1, g2)  # no atomics: reruns are bit-identical
    for r in (0, 97, 255):  # a row alone gives its gradient in the batch bit for bit
        _, gr = _stretch_grad(spec[r:r + 1], rate, g[r:r + 1], fn)
        assert torch.equal(gr[0], g1[r])
    _bar(g1[:32], _oracle(spec[:32], g[:32], rate))


def _torch_f32_pitch_grad(wave, g, sr, steps):
    """The float32 CPU torchaudio run's waveform gradient (the reference's own round-off), or None."""
    if TAF is None:
        return None
    x = torch.from_numpy(wave).float().requires_grad_()
    y = TAF.pitch_shift(x, sr, steps)
    y.backward(torch.from_numpy(g).float())
    return x.grad.double().numpy()


def _pitch_bar(got, exp, ref):
    got = got.detach().double().cpu().numpy()
    assert got.shape == exp.shape and np.isfinite(got).all()
    scale = np.abs(exp).max()
    err = np.abs(got - exp).max() / scale
    rel_l2 = np.linalg.norm(got - exp) / np.linalg.norm(exp)
    ref_err = None if ref is None else np.abs(ref - exp).max() / scale
    ok = (ref_err is not None and err <= 2 * ref_err) or (rel_l2 <= 5e-3 and err <= 2e-2)
    assert ok, f"max err {err:.3e} (float32 reference run: {ref_err}), rel L2 {rel_l2:.3e}"


PITCH = {"up12": (16000, 12), "down12": (16000, -12), "up7_1k": (1000, 7), "down5_1k": (1000, -5), "up4": (16000, 4),
         "down3": (16000, -3)}


@pytest.mark.parametrize("tag", list(PITCH))
def test_pitch_shift_grad(golden, tag):
    sr, steps = PITCH[tag]
    wave = golden["wave"]
    g = np.random.default_rng(len(tag)).standard_normal(wave.shape).astype(np.float32)
    x = torch.from_numpy(wave).to(DEV)
    gt = torch.from_numpy(g).to(DEV)
    mod = T.PitchShift(sr, steps).to(DEV)
    with audio_b200.differentiable(vocoder=True):
        xf = x.clone().requires_grad_()
        yf = F.pitch_shift(xf, sr, steps, window=mod.window)  # the module's window, to the last bit
        yf.backward(gt)
        xm = x.clone().reshape(1, 2, -1).requires_grad_()
        ym = mod(xm)
        ym.backward(gt.reshape(1, 2, -1))
        assert audio_b200.is_vocoder_differentiable() and not audio_b200.is_inverse_differentiable()
    with torch.no_grad():
        assert torch.equal(yf, F.pitch_shift(x, sr, steps, window=mod.window))
    exp = V.pitch_shift_vjp(wave, g, sr, steps, grid=np.float32)
    _pitch_bar(xf.grad, exp, _torch_f32_pitch_grad(wave, g, sr, steps))
    assert torch.equal(xm.grad.reshape(2, -1), xf.grad)  # the module and the function: the same gradient


def test_pitch_shift_large_batch():
    wave = torch.randn(64, 48000, generator=torch.Generator().manual_seed(5)).to(DEV)
    g = torch.randn(64, 48000, generator=torch.Generator().manual_seed(6)).to(DEV)
    with audio_b200.differentiable(vocoder=True):
        x = wave.clone().requires_grad_()
        F.pitch_shift(x, 16000, 4).backward(g)
        x2 = wave[5:6].clone().requires_grad_()
        F.pitch_shift(x2, 16000, 4).backward(g[5:6])
    assert torch.isfinite(x.grad).all()
    exp = V.pitch_shift_vjp(wave[:2].cpu().numpy(), g[:2].cpu().numpy(), 16000, 4, grid=np.float32)
    _pitch_bar(x.grad[:2], exp, None)
    assert torch.equal(x2.grad[0], x.grad[5])


def test_stretch_then_inverse_chain():
    """A leaf complex spectrogram -> TimeStretch -> InverseSpectrogram -> L1 loss, against the numpy composition."""
    gen = torch.Generator().manual_seed(9)
    wave = torch.randn(2, 8000, generator=gen).to(DEV)
    spec = T.Spectrogram(n_fft=512, hop_length=128, power=None).to(DEV)(wave)
    rate = 1.3
    with audio_b200.differentiable(inverse=True, vocoder=True):
        z = spec.detach().clone().requires_grad_()
        y = T.InverseSpectrogram(n_fft=512, hop_length=128).to(DEV)(
            T.TimeStretch(hop_length=128, n_freq=257, fixed_rate=rate).to(DEV)(z))
        y.abs().sum().backward()
    frames_out = int(math.ceil(spec.shape[-1] / rate))
    g_y = inverse_spectrogram_vjp(torch.sign(y).detach().cpu().numpy(), frames_out, None, 0,
                                  torch.hann_window(512).double().numpy(), 512, 128, 512)
    exp = _oracle(spec, torch.from_numpy(g_y), rate)
    _bar(z.grad, exp)


def test_what_raises_and_what_works(golden):
    spec = torch.from_numpy(golden["spec"]).to(DEV)
    x = torch.from_numpy(golden["wave"]).to(DEV)
    with audio_b200.differentiable(vocoder=True):
        z = spec.clone().requires_grad_()
        (gz,) = torch.autograd.grad(F.phase_vocoder(z, 1.3, _pa(257)).abs().sum(), z, create_graph=True)
        with pytest.raises(RuntimeError):  # double backward
            gz.abs().sum().backward()
        pa = _pa(257).requires_grad_()
        with pytest.raises(RuntimeError, match="phase_advance requires grad"):
            F.phase_vocoder(spec.clone().requires_grad_(), 1.3, pa)
        with pytest.raises(RuntimeError, match="forward-only"):
            T.GriffinLim(n_fft=512, n_iter=2).to(DEV)(spec.abs().clone().requires_grad_())
        with pytest.raises(RuntimeError, match="forward-only"):  # the inverse alone needs inverse=True
            T.InverseSpectrogram(n_fft=512, hop_length=128).to(DEV)(spec.clone().requires_grad_())
        with pytest.raises(RuntimeError, match="forward-only"):  # the resampler alone needs resample=True
            T.Resample(16000, 8000).to(DEV)(x.clone().requires_grad_())
        # an in-place edit of the saved input, or of the output, before backward
        leaf = spec.clone().requires_grad_()
        inp = leaf * 1
        y = F.phase_vocoder(inp, 1.3, _pa(257))
        inp.mul_(2)
        with pytest.raises(RuntimeError):
            y.abs().sum().backward()
        with pytest.raises(RuntimeError):
            y = F.phase_vocoder(spec.clone().requires_grad_(), 1.3, _pa(257))
            y.mul_(2)
            y.abs().sum().backward()
        # an empty batch works
        e = torch.zeros(0, 257, 47, dtype=torch.complex64, device=DEV).requires_grad_()
        F.phase_vocoder(e, 1.3, _pa(257)).abs().sum().backward()
        assert e.grad.shape == e.shape
    with pytest.raises(RuntimeError, match=r"forward-only.*differentiable\(vocoder=True\)"):  # switched off again
        T.TimeStretch(hop_length=128, n_freq=257, fixed_rate=1.3).to(DEV)(spec.clone().requires_grad_())
