"""Spectrogram gradients of inverse_spectrogram without a GPU: the float64 oracle VJP against torch.autograd through
torch.istft, the ABI validation of b200a_istft_backward / b200a_istft_backward_scratch_bytes, and the inverse switch."""
import ctypes
import threading
import warnings

import numpy as np
import pytest
import torch

from oracle import frontend_oracle as O

import istft_grad_oracle as V


def _torch_inverse(spec, length, pad, window, n_fft, hop, win_length, normalized, center):
    """torchaudio.functional.inverse_spectrogram's composition in float64 torch (the autograd reference)."""
    fl_norm, win_norm = O._spec_norms(normalized)
    if win_norm:
        spec = spec * window.pow(2.0).sum().sqrt()
    shape = spec.size()
    spec = spec.reshape(-1, shape[-2], shape[-1])
    y = torch.istft(spec, n_fft=n_fft, hop_length=hop, win_length=win_length, window=window, center=center,
                    normalized=fl_norm, onesided=True, length=length + 2 * pad if length is not None else None,
                    return_complex=False)
    if length is not None and pad > 0:
        y = y[:, pad:-pad]
    return y.reshape(shape[:-2] + y.shape[-1:])


def _check(seed, lead, n_fft, hop, frames, length=None, pad=0, win_length=None, normalized=False, center=True):
    rng = np.random.default_rng(seed)
    win_length = n_fft if win_length is None else win_length
    window = O.hann_window(win_length) + 0.1 * rng.random(win_length)  # no exact zeros: the envelope is positive
    shape = lead + (n_fft // 2 + 1, frames)
    z = torch.tensor(rng.standard_normal(shape) + 1j * rng.standard_normal(shape), requires_grad=True)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")  # torch.istft warns when `length` exceeds what the frames cover
        y = _torch_inverse(z, length, pad, torch.tensor(window), n_fft, hop, win_length, normalized, center)
    g = rng.standard_normal(tuple(y.shape))
    (exp,) = torch.autograd.grad(y, z, grad_outputs=torch.tensor(g))
    exp = exp.numpy()
    got = V.inverse_spectrogram_vjp(g, frames, length, pad, window, n_fft, hop, win_length, normalized, center)
    assert got.shape == exp.shape
    np.testing.assert_allclose(got, exp, rtol=0, atol=1e-10 * max(1.0, np.abs(exp).max()))
    assert (got[..., 0, :].imag == 0).all()


@pytest.mark.parametrize("center", [True, False])
@pytest.mark.parametrize("length", [None, 1000, 2000], ids=["none", "short", "long"])
def test_center_and_length(center, length):
    _check(1, (2,), 256, 64, 24, length=length, center=center)  # expected = 1728 samples


@pytest.mark.parametrize("length", [None, 1000, 1300])
def test_pre_pad_and_short_window(length):
    _check(2, (2,), 256, 100, 14, length=length, pad=37, win_length=200)


@pytest.mark.parametrize("normalized", [False, True, "window", "frame_length"])
def test_normalized(normalized):
    _check(3, (1,), 400, 160, 12, normalized=normalized)


@pytest.mark.parametrize("n_fft,hop", [(256, 64), (400, 100), (77, 20), (2048, 512)])
@pytest.mark.parametrize("center", [True, False])
def test_sizes(n_fft, hop, center):
    _check(4, (2,), n_fft, hop, 9, center=center, length=None if center else 5 * hop + n_fft // 2)


def test_3d_and_pad_with_long_length():
    _check(5, (2, 2), 256, 64, 10, length=900, pad=20)


# ---- ABI validation (host only: every rejected call returns before touching a pointer) -------------------------------
def _lib_or_skip():
    from audio_b200 import _lib

    try:
        return _lib, _lib.lib()
    except ImportError:
        pytest.skip("libb200audio.so is not built")


def _desc(n_fft=512, **kw):
    from audio_b200._plans import FrontendPlan

    d = FrontendPlan.make_desc(n_fft, n_fft, n_fft // 4, 0, True, "reflect", True, False, False, 2.0)
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def test_istft_backward_abi_validation():
    L, lib = _lib_or_skip()
    fake = ctypes.c_void_p(0x1000)  # never dereferenced: every case below fails validation first

    def call(d, rows=2, g_row_stride=4000, start=256, g_len=4000, frames=30, ptrs=True, scratch=True):
        p = fake if ptrs else None
        return lib.b200a_istft_backward(d, p, p, rows, g_row_stride, start, g_len, frames, p if scratch else None, p, None)

    assert call(_desc(onesided=0)) == L.EUNSUPPORTED
    assert call(_desc(hop=0)) == L.EINVAL
    assert call(_desc(n_fft=16384)) == L.EUNSUPPORTED
    assert call(_desc(), rows=-1) == L.EINVAL
    assert call(_desc(), frames=0) == L.EINVAL
    assert call(_desc(), g_row_stride=-1) == L.EINVAL
    assert call(_desc(), start=-1) == L.EINVAL
    assert call(_desc(), g_len=-1) == L.EINVAL
    assert call(_desc(), ptrs=False) == L.EINVAL
    assert call(_desc(), rows=0, ptrs=False) == L.OK
    assert call(_desc(n_fft=400), scratch=False) == L.EINVAL  # the composition path needs its scratch
    assert call(None) == L.EINVAL


def test_istft_backward_scratch_bytes():
    L, lib = _lib_or_skip()
    # register-FFT sizes need none; every other size holds g / env for the n_fft + hop (frames - 1) samples of each row
    assert lib.b200a_istft_backward_scratch_bytes(_desc(), 3, 30) == 0
    assert lib.b200a_istft_backward_scratch_bytes(_desc(n_fft=400), 3, 30) >= 3 * (400 + 100 * 29) * 4
    assert lib.b200a_istft_backward_scratch_bytes(_desc(n_fft=400), 3, 30) < 3 * (400 + 100 * 29) * 4 + 256
    assert lib.b200a_istft_backward_scratch_bytes(_desc(n_fft=77), 1, 5) >= (77 + 19 * 4) * 4
    assert lib.b200a_istft_backward_scratch_bytes(_desc(onesided=0), 3, 30) == 0
    assert lib.b200a_istft_backward_scratch_bytes(_desc(), 3, 0) == 0
    assert lib.b200a_istft_backward_scratch_bytes(None, 3, 30) == 0


def test_inverse_switch_is_thread_local_and_off_by_default():
    import audio_b200

    assert not audio_b200.is_differentiable() and not audio_b200.is_inverse_differentiable()
    seen = []
    with audio_b200.differentiable(inverse=True):
        assert audio_b200.is_differentiable() and audio_b200.is_inverse_differentiable()
        t = threading.Thread(target=lambda: seen.append((audio_b200.is_differentiable(),
                                                         audio_b200.is_inverse_differentiable())))
        t.start()
        t.join()
        with audio_b200.differentiable():  # the plain switch keeps its meaning: waveform gradients only
            assert audio_b200.is_differentiable() and not audio_b200.is_inverse_differentiable()
        assert audio_b200.is_inverse_differentiable()
        with audio_b200.differentiable(False, inverse=True):  # inverse gradients need the switch itself on
            assert not audio_b200.is_differentiable() and not audio_b200.is_inverse_differentiable()
        assert audio_b200.is_differentiable() and audio_b200.is_inverse_differentiable()
    assert seen == [(False, False)]
    assert not audio_b200.is_differentiable() and not audio_b200.is_inverse_differentiable()
    audio_b200.set_differentiable(True, inverse=True)
    try:
        assert audio_b200.is_inverse_differentiable()
    finally:
        audio_b200.set_differentiable(False)
    assert not audio_b200.is_differentiable() and not audio_b200.is_inverse_differentiable()


def test_forward_only_message_names_the_keyword():
    from audio_b200._plans import _no_autograd

    with pytest.raises(RuntimeError, match=r"forward-only.*differentiable\(inverse=True\)"):
        _no_autograd(torch.zeros(2, requires_grad=True))
