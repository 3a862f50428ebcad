"""Waveform gradients without a GPU: the float64 oracle VJPs against torch.autograd through torch.stft, and the ABI
validation of b200a_frontend_backward / b200a_frontend_backward_scratch_bytes."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import frontend_oracle as O

import grad_oracle as V


def _torch_spectrogram(x, pad, window, n_fft, hop, win_length, power, normalized, center, pad_mode, onesided):
    """torchaudio.functional.spectrogram's composition in float64 torch (the autograd reference)."""
    if pad > 0:
        x = torch.nn.functional.pad(x, (pad, pad), "constant")
    shape = x.size()
    x = x.reshape(-1, shape[-1])
    fl_norm, win_norm = O._spec_norms(normalized)
    spec = torch.stft(x, n_fft=n_fft, hop_length=hop, win_length=win_length, window=window, center=center,
                      pad_mode=pad_mode, normalized=fl_norm, onesided=onesided, return_complex=True)
    spec = spec.reshape(shape[:-1] + spec.shape[-2:])
    if win_norm:
        spec = spec / window.pow(2.0).sum().sqrt()
    if power is None:
        return spec
    return spec.abs() if power == 1.0 else spec.abs().pow(power)


def _torch_vjp(x, g, **kw):
    xt = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    window = torch.tensor(kw.pop("window"), dtype=torch.float64)
    y = _torch_spectrogram(xt, window=window, **kw)
    gt = torch.tensor(g, dtype=y.dtype)
    (dx,) = torch.autograd.grad(y, xt, grad_outputs=gt)
    return dx.numpy()


def _case(seed, shape, n_fft, hop, win_length=None, pad=0, power=2.0, normalized=False, center=True,
          pad_mode="reflect", onesided=True):
    rng = np.random.default_rng(seed)
    win_length = n_fft if win_length is None else win_length
    x = rng.standard_normal(shape)
    window = O.hann_window(win_length) + 0.1 * rng.random(win_length)  # no exact zeros at the window's ends
    kw = dict(pad=pad, window=window, n_fft=n_fft, hop=hop, win_length=win_length, power=power, normalized=normalized,
              center=center, pad_mode=pad_mode, onesided=onesided)
    y = O.spectrogram(x, **{k: v for k, v in kw.items()})
    g = rng.standard_normal(y.shape)
    if power is None:
        g = g + 1j * rng.standard_normal(y.shape)
    return x, g, kw


def _check(x, g, kw):
    exp = _torch_vjp(x, g, **dict(kw))
    got = V.spectrogram_vjp(x, g, **kw)
    assert got.shape == x.shape
    np.testing.assert_allclose(got, exp, rtol=0, atol=1e-10 * max(1.0, np.abs(exp).max()))


@pytest.mark.parametrize("pad_mode", ["reflect", "constant", "replicate", "circular"])
@pytest.mark.parametrize("center", [True, False])
def test_pad_modes(pad_mode, center):
    _check(*_case(1, (2, 1500), 256, 64, pad_mode=pad_mode, center=center))


@pytest.mark.parametrize("pad_mode", ["reflect", "replicate", "circular", "constant"])
def test_pre_pad_and_short_window(pad_mode):
    _check(*_case(2, (2, 1300), 256, 100, win_length=200, pad=37, pad_mode=pad_mode))


@pytest.mark.parametrize("normalized", [False, True, "window", "frame_length"])
@pytest.mark.parametrize("onesided", [True, False])
def test_normalized_and_onesided(normalized, onesided):
    _check(*_case(3, (1, 2000), 400, 160, normalized=normalized, onesided=onesided))


@pytest.mark.parametrize("power", [None, 0.5, 1.0, 2.0, 3.0])
def test_powers(power):
    _check(*_case(4, (2, 1800), 256, 64, power=power))


@pytest.mark.parametrize("n_fft,hop", [(256, 64), (400, 100), (77, 20), (2048, 512)])
@pytest.mark.parametrize("power", [None, 1.0, 2.0])
def test_sizes(n_fft, hop, power):
    _check(*_case(5, (2, 6000), n_fft, hop, power=power, onesided=power is not None))


def test_odd_size_two_sided_and_3d():
    _check(*_case(6, (2, 2, 900), 77, 30, power=None, onesided=False))
    _check(*_case(7, (2, 2, 900), 77, 30, power=1.0, pad_mode="circular"))


@pytest.mark.parametrize("mel_scale,norm", [("htk", None), ("slaney", "slaney")])
@pytest.mark.parametrize("power", [1.0, 2.0])
def test_mel(mel_scale, norm, power):
    rng = np.random.default_rng(8)
    x = rng.standard_normal((2, 4000))
    fb = O.melscale_fbanks(257, 0.0, 8000.0, 40, 16000, norm, mel_scale)
    y = O.mel_spectrogram(x, n_fft=512, hop_length=128, power=power, fb=fb)
    g = rng.standard_normal(y.shape)
    got = V.mel_spectrogram_vjp(x, g, n_fft=512, hop_length=128, power=power, fb=fb)
    xt = torch.tensor(x, requires_grad=True)
    spec = _torch_spectrogram(xt, 0, torch.tensor(O.hann_window(512)), 512, 128, 512, power, False, True, "reflect", True)
    mel = torch.matmul(spec.transpose(-1, -2), torch.tensor(fb)).transpose(-1, -2)
    (exp,) = torch.autograd.grad(mel, xt, grad_outputs=torch.tensor(g))
    np.testing.assert_allclose(got, exp.numpy(), rtol=0, atol=1e-10 * max(1.0, np.abs(exp.numpy()).max()))


@pytest.mark.parametrize("power,expect_nan", [(0.5, True), (1.0, False), (2.0, False)])
def test_zero_input(power, expect_nan):
    """torch's float64 backward at X = 0: NaN everywhere for p < 1, zero for p >= 1; the oracle agrees."""
    x = np.zeros((1, 2048))
    kw = dict(pad=0, window=O.hann_window(256), n_fft=256, hop=64, win_length=256, power=power, normalized=False,
              center=True, pad_mode="reflect", onesided=True)
    g = np.ones(O.spectrogram(x, **kw).shape)
    exp = _torch_vjp(x, g, **dict(kw))
    got = V.spectrogram_vjp(x, g, **kw)
    if expect_nan:
        assert np.isnan(exp).all() and np.isnan(got).all()
    else:
        assert (exp == 0).all() and (got == 0).all()


# ---- ABI validation (host only: every rejected call returns before touching a pointer) -------------------------------
def _lib_or_skip():
    from audio_b200 import _lib

    try:
        return _lib, _lib.lib()
    except ImportError:
        pytest.skip("libb200audio.so is not built")


def _desc(n_fft=512, n_mels=0, power=2.0, **kw):
    from audio_b200._plans import FrontendPlan

    d = FrontendPlan.make_desc(n_fft, n_fft, n_fft // 4, 0, True, "reflect", True, False, False, power, n_mels)
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def test_backward_abi_validation():
    L, lib = _lib_or_skip()
    fake = ctypes.c_void_p(0x1000)  # never dereferenced: every case below fails validation first

    def call(d, stage, rows=2, length=4000, row_stride=4000, grad_row_stride=4000, ptrs=True):
        p = fake if ptrs else None
        return lib.b200a_frontend_backward(d, p, stage, p, rows, length, row_stride, p, 0, 0, 0, p, p, grad_row_stride,
                                           None)

    assert call(_desc(), L.STAGE_FEAT) == L.EUNSUPPORTED
    assert call(_desc(), 7) == L.EINVAL
    assert call(_desc(), -1) == L.EINVAL
    assert call(_desc(), L.STAGE_MEL) == L.EINVAL  # no filterbank in the descriptor
    assert call(_desc(power=0.0), L.STAGE_POWER) == L.EINVAL
    assert call(_desc(), L.STAGE_POWER, ptrs=False) == L.EINVAL
    assert call(_desc(), L.STAGE_POWER, rows=0, ptrs=False) == L.OK
    assert call(_desc(), L.STAGE_POWER, row_stride=100) == L.EINVAL
    assert call(_desc(), L.STAGE_POWER, grad_row_stride=100) == L.EINVAL
    assert call(_desc(), L.STAGE_POWER, length=200, row_stride=200, grad_row_stride=200) == L.ESHORT
    assert call(_desc(hop=0), L.STAGE_POWER) == L.EINVAL
    assert call(_desc(n_fft=16384), L.STAGE_POWER) == L.EUNSUPPORTED


def test_backward_scratch_bytes():
    L, lib = _lib_or_skip()
    T = lib.b200a_num_frames(4000, 512, 128, 1, 0)
    # register-FFT sizes: the frame gradients only
    assert lib.b200a_frontend_backward_scratch_bytes(_desc(), L.STAGE_POWER, 3, 4000) >= 3 * T * 512 * 4
    assert lib.b200a_frontend_backward_scratch_bytes(_desc(), L.STAGE_POWER, 3, 4000) < 3 * T * 512 * 4 + 4096
    # other sizes also hold the complex spectrum and a flag per frame
    d = _desc(n_fft=400)
    T4 = lib.b200a_num_frames(4000, 400, 100, 1, 0)
    assert lib.b200a_frontend_backward_scratch_bytes(d, L.STAGE_COMPLEX, 3, 4000) >= 3 * T4 * (400 + 2 * 201 + 1) * 4
    assert lib.b200a_frontend_backward_scratch_bytes(_desc(), L.STAGE_FEAT, 3, 4000) == 0
    assert lib.b200a_frontend_backward_scratch_bytes(_desc(), L.STAGE_POWER, 3, 100) == 0
    assert lib.b200a_frontend_backward_scratch_bytes(None, L.STAGE_POWER, 3, 4000) == 0


def test_switch_is_thread_local_and_off_by_default():
    import threading

    import audio_b200

    assert not audio_b200.is_differentiable()
    seen = []
    with audio_b200.differentiable():
        assert audio_b200.is_differentiable()
        t = threading.Thread(target=lambda: seen.append(audio_b200.is_differentiable()))
        t.start()
        t.join()
        with audio_b200.differentiable(False):
            assert not audio_b200.is_differentiable()
        assert audio_b200.is_differentiable()
    assert seen == [False]
    assert not audio_b200.is_differentiable()
    audio_b200.set_differentiable(True)
    try:
        assert audio_b200.is_differentiable()
    finally:
        audio_b200.set_differentiable(False)
