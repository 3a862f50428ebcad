"""Spectrogram gradients of phase_vocoder and waveform gradients of pitch_shift without a GPU: the float64 oracle VJPs
against torch.autograd through torchaudio (or, where it does not import, a torch restatement of the reference's op
sequence), the ABI validation of b200a_phase_vocoder_backward, and the vocoder switch."""
import ctypes
import math
import threading

import numpy as np
import pytest
import torch

from oracle import frontend_oracle as O

import vocoder_grad_oracle as V

try:
    import torchaudio.functional as TAF
except Exception:  # noqa: BLE001 -- any import failure means "use the restatement"
    TAF = None

RATES = (0.5, 0.7, 0.8, 0.9, 1.3, 2.0, 3.1)
# the pitch cases of the forward tests (tests/test_inverse.py), plus 16 kHz +4 steps and no shift at all
PITCH_CASES = {"up12": (16000, 12), "down12": (16000, -12), "up7_1k": (1000, 7), "down5_1k": (1000, -5),
               "up4": (16000, 4), "zero": (16000, 0)}


def _torch_phase_vocoder(spec, rate, pa):
    """The reference's phase vocoder as torch ops (time grid in the spectrogram's real dtype): neighbours by
    truncation of the grid and of grid + 1, interpolated magnitudes, wrapped phase differences, cumulative phase."""
    if rate == 1.0:
        return spec
    shape = spec.size()
    spec = spec.reshape((-1,) + tuple(shape[-2:]))
    grid = torch.arange(0, spec.size(-1), rate, dtype=spec.real.dtype)
    padded = torch.nn.functional.pad(spec, [0, 2])
    z0, z1 = padded.index_select(-1, grid.long()), padded.index_select(-1, (grid + 1).long())
    dphi = z1.angle() - z0.angle() - pa
    dphi = dphi - 2 * math.pi * torch.round(dphi / (2 * math.pi)) + pa
    phase = torch.cumsum(torch.cat([spec[..., :1].angle(), dphi[..., :-1]], dim=-1), -1)
    alpha = grid % 1.0
    out = torch.polar(alpha * z1.abs() + (1 - alpha) * z0.abs(), phase)
    return out.reshape(shape[:-2] + out.shape[1:])


def phase_vocoder_ref(spec, rate, pa):
    return TAF.phase_vocoder(spec, rate, pa) if TAF is not None else _torch_phase_vocoder(spec, rate, pa)


def _torch_resample(x, orig, new):
    gcd = math.gcd(orig, new)
    o, n = orig // gcd, new // gcd
    kernel, width = O.sinc_resample_kernel(orig, new, gcd)
    k = torch.tensor(kernel).reshape(n, -1)
    rows, length = x.shape
    w = torch.nn.functional.pad(x, (width, width + o))
    y = torch.nn.functional.conv1d(w[:, None], k[:, None, :], stride=o).transpose(1, 2).reshape(rows, -1)
    return y[..., :O.resample_len(length, o, n)]


def pitch_shift_ref(x, sr, n_steps, window):
    """F.pitch_shift in float64 torch: torchaudio's where it imports, else its op sequence restated."""
    if TAF is not None:
        return TAF.pitch_shift(x, sr, n_steps, window=window)
    n_fft, hop = 512, 128
    rate = 2.0 ** (-float(n_steps) / 12)
    spec = torch.stft(x, n_fft, hop, n_fft, window, center=True, pad_mode="reflect", return_complex=True)
    pa = torch.linspace(0, math.pi * hop, spec.shape[-2], dtype=x.dtype)[..., None]
    len_stretch = int(round(x.shape[-1] / rate))
    y = torch.istft(_torch_phase_vocoder(spec, rate, pa), n_fft, hop, n_fft, window, length=len_stretch)
    orig = int(sr / rate)
    y = _torch_resample(y, orig, sr) if orig != sr else y
    n = y.shape[-1]
    return y[..., :x.shape[-1]] if n > x.shape[-1] else torch.nn.functional.pad(y, [0, x.shape[-1] - n])


def torch_grid(frames, rate):
    """The float64 time steps the reference's run takes: torch.arange's own, which its vectorised fill rounds
    differently from rate * t at some steps (enough to move a neighbour at rate 0.7)."""
    return torch.arange(0, frames, rate, dtype=torch.float64).numpy()


def _spec(rng, lead, bins, frames):
    return rng.standard_normal(lead + (bins, frames)) + 1j * rng.standard_normal(lead + (bins, frames))


def _check_vocoder(spec, rate, seed=0):
    bins, frames = spec.shape[-2:]
    rng = np.random.default_rng(seed)
    pa = np.linspace(0, math.pi * 4, bins)[:, None]
    x = torch.tensor(spec, requires_grad=True)
    y = phase_vocoder_ref(x, rate, torch.tensor(pa))
    assert y.shape[-1] == int(math.ceil(frames / rate))
    g = rng.standard_normal(tuple(y.shape)) + 1j * rng.standard_normal(tuple(y.shape))
    (exp,) = torch.autograd.grad(y, x, grad_outputs=torch.tensor(g))
    exp = exp.numpy()
    got = V.phase_vocoder_vjp(spec, g, rate, phase_advance=pa, grid=torch_grid(frames, rate))
    assert got.shape == exp.shape
    assert np.isfinite(got).all()
    np.testing.assert_allclose(got, exp, rtol=0, atol=1e-10 * np.abs(exp).max())
    return got


@pytest.mark.parametrize("rate", RATES)
@pytest.mark.parametrize("lead", [(), (3,), (2, 2)], ids=["2d", "3d", "4d"])
def test_phase_vocoder_vjp(rate, lead):
    _check_vocoder(_spec(np.random.default_rng(len(lead)), lead, 9, 23), rate, seed=int(rate * 10))


@pytest.mark.parametrize("rate", [0.7, 1.0 + 1e-9, 1.3, 3.1])
def test_zeros_and_silence(rate):
    spec = _spec(np.random.default_rng(5), (2,), 9, 30)
    spec[0, 3, 4] = 0  # an exact zero element
    spec[1, :, 0] = 0  # an all-zero first frame
    spec[0, :, 10:16] = 0  # a silent stretch
    got = _check_vocoder(spec, rate, seed=3)
    assert (got[0, 3, 4] == 0) and (got[1, :, 0] == 0).all() and (got[0, :, 10:16] == 0).all()


def test_untouched_frames_get_zero():
    got = _check_vocoder(_spec(np.random.default_rng(6), (), 5, 40), 3.1)
    i0, i1, _ = V.time_grid(40, 3.1, torch_grid(40, 3.1))
    untouched = sorted(set(range(40)) - set(i0) - set(i1) - {0})
    assert untouched and (got[:, untouched] == 0).all()


@pytest.mark.parametrize("rate", [0.7, 0.8, 0.9, 1.3])
def test_reference_non_zero_inputs(rate):
    """The reference's test_timestretch_non_zero input: a two-channel white-noise spectrogram at n_fft 16 with every
    element within 2e-2 of the origin pushed out to 2e-2."""
    wave = np.random.default_rng(40).uniform(-1, 1, (2, 40))
    spec = O.stft(wave, 16, 4, O.hann_window(16), center=True, pad_mode="reflect")
    close = np.abs(spec) < 2e-2
    spec[close] = 2e-2 * spec[close] / np.maximum(np.abs(spec[close]), 1e-300)
    spec[close & (spec == 0)] = 2e-2
    _check_vocoder(spec, rate, seed=7)


def test_float32_grid_picks_other_neighbours():
    """At rate 0.7 the float32 grid (the GPU kernels') and the float64 grid disagree on neighbours, and in float32
    trunc(ts + 1) is sometimes i0 + 2: the oracle follows whichever grid it is given."""
    i0_32, i1_32, _ = V.time_grid(501, 0.7, np.float32)
    i0_64, i1_64, _ = V.time_grid(501, 0.7, np.float64)
    assert (i0_32 != i0_64).any() or (i1_32 != i1_64).any()
    assert (i1_32 - i0_32 >= 1).all() and (i1_32 - i0_32 <= 2).all()
    i0, i1, _ = V.time_grid(3, 1.0, np.array([0.0, 2.0 - 2.0**-23], dtype=np.float32))  # 2.9999999 rounds to 3
    assert list(i0) == [0, 1] and list(i1) == [1, 3]


@pytest.mark.parametrize("tag", list(PITCH_CASES))
def test_pitch_shift_vjp(tag):
    sr, steps = PITCH_CASES[tag]
    rng = np.random.default_rng(len(tag))
    wave = rng.standard_normal((2, 6000)) * np.hanning(6000)
    window = torch.hann_window(512, dtype=torch.float64)
    x = torch.tensor(wave, requires_grad=True)
    y = pitch_shift_ref(x, sr, steps, window)
    assert y.shape == x.shape
    g = rng.standard_normal(tuple(y.shape))
    (exp,) = torch.autograd.grad(y, x, grad_outputs=torch.tensor(g))
    exp = exp.numpy()
    rate = 2.0 ** (-float(steps) / 12)
    got = V.pitch_shift_vjp(wave, g, sr, steps, window=window.numpy(), grid=torch_grid(1 + 6000 // 128, rate))
    np.testing.assert_allclose(got, exp, rtol=0, atol=1e-9 * np.abs(exp).max())


# ---- ABI validation (host only: every rejected call returns before touching a pointer) -------------------------------
def _lib_or_skip():
    from audio_b200 import _lib

    try:
        return _lib, _lib.lib()
    except ImportError:
        pytest.skip("libb200audio.so is not built")


def test_phase_vocoder_backward_validation():
    L, lib = _lib_or_skip()
    fake = ctypes.c_void_p(0x1000)

    def call(rows=2, bins=257, frames_in=100, rate=1.3, frames_out=77, gs=(257 * 77, 77, 1), ptrs=(True,) * 4):
        p = [fake if ok else None for ok in ptrs]
        return lib.b200a_phase_vocoder_backward(p[0], bins * frames_in, frames_in, 1, rows, bins, frames_in, rate, p[1],
                                                p[2], gs[0], gs[1], gs[2], p[3], frames_out, None)

    assert call(rows=-1) == L.EINVAL
    assert call(bins=0) == L.EINVAL
    assert call(frames_in=0) == L.EINVAL
    assert call(frames_out=0) == L.EINVAL
    assert call(rate=0.0) == L.EINVAL
    assert call(rate=-1.3) == L.EINVAL
    assert call(rate=float("nan")) == L.EINVAL
    for i in range(3):
        assert call(gs=tuple(-1 if j == i else s for j, s in enumerate((257 * 77, 77, 1)))) == L.EINVAL
    for i in range(4):
        assert call(ptrs=tuple(j != i for j in range(4))) == L.EINVAL
    assert call(rows=0, ptrs=(False,) * 4) == L.OK  # empty batch: no pointer is read
    assert call(rows=65536) == L.EUNSUPPORTED  # one grid row per batch row, as the forward


# ---- the vocoder switch ----------------------------------------------------------------------------------------------
def test_vocoder_switch_is_thread_local_opt_in_and_independent():
    import audio_b200 as A

    def others():
        return (A.is_inverse_differentiable(), A.is_resample_differentiable(), A.is_feature_differentiable(),
                A.is_kaldi_differentiable())

    assert not A.is_vocoder_differentiable()
    with A.differentiable(vocoder=True):
        assert A.is_vocoder_differentiable() and A.is_differentiable()
        assert others() == (False,) * 4
        seen = []
        t = threading.Thread(target=lambda: seen.append(A.is_vocoder_differentiable()))
        t.start()
        t.join()
        assert seen == [False]
        with A.differentiable():  # the plain switch keeps its meaning
            assert not A.is_vocoder_differentiable()
        assert A.is_vocoder_differentiable()
    assert not A.is_vocoder_differentiable()
    with A.differentiable(False, vocoder=True):  # needs the switch itself on
        assert not A.is_vocoder_differentiable()
    with A.differentiable(inverse=True, resample=True, features=True, kaldi=True):
        assert not A.is_vocoder_differentiable() and others() == (True,) * 4
    with A.differentiable(inverse=True, resample=True, features=True, kaldi=True, vocoder=True):
        assert A.is_vocoder_differentiable() and others() == (True,) * 4
    A.set_differentiable(True, vocoder=True)
    try:
        assert A.is_vocoder_differentiable()
    finally:
        A.set_differentiable(False)
    assert not A.is_vocoder_differentiable()


def test_vocoder_chain_turns_the_stages_on_for_one_call_only():
    import audio_b200 as A
    from audio_b200._plans import vocoder_chain

    x = torch.zeros(4, requires_grad=True)
    with A.differentiable(vocoder=True, features=True):
        with vocoder_chain(x):
            assert A.is_differentiable() and A.is_inverse_differentiable() and A.is_resample_differentiable()
            assert A.is_feature_differentiable() and A.is_vocoder_differentiable()
        assert not (A.is_inverse_differentiable() or A.is_resample_differentiable())
        with vocoder_chain(x.detach()):  # nothing to differentiate: the switches stay as they are
            assert not A.is_inverse_differentiable()
        with torch.no_grad(), vocoder_chain(x):
            assert not A.is_inverse_differentiable()
    with A.differentiable(inverse=True, resample=True):  # without vocoder=True the chain changes nothing
        with vocoder_chain(x):
            assert not A.is_vocoder_differentiable() and A.is_inverse_differentiable()


def test_forward_only_message_names_the_vocoder_keyword():
    from audio_b200._plans import _no_autograd

    with pytest.raises(RuntimeError, match=r"forward-only.*differentiable\(kaldi=True\).*differentiable\(vocoder=True\)"):
        _no_autograd(torch.zeros(2, requires_grad=True))
