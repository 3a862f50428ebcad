"""Waveform gradients of the resampler without a GPU: the float64 oracle VJP against torch.autograd through the
reference's op sequence (F.pad, conv1d, transpose, reshape, slice), the ABI validation of the three backward entry
points, and the resample switch."""
import ctypes
import math
import threading

import numpy as np
import pytest
import torch
from golden_cases import RESAMPLE

from oracle import frontend_oracle as O

import resample_grad_oracle as V

RATIOS = {key: (kw["orig_freq"], kw["new_freq"], kw.get("resampling_method", "sinc_interp_hann"),
                kw.get("lowpass_filter_width", 6), kw.get("rolloff", 0.99), cut)
          for key, (cut, kw) in RESAMPLE.items()}
RATIOS.update({"16k_8k": (16000, 8000, "sinc_interp_hann", 6, 0.99, None),
               "8k_16k": (8000, 16000, "sinc_interp_hann", 6, 0.99, None),
               "2003_1999": (2003, 1999, "sinc_interp_hann", 6, 0.99, None)})


def _torch_resample(x, o, n, kernel, width):
    """_apply_sinc_resample_kernel's composition in float64 torch (the autograd reference)."""
    shape = x.size()
    w = x.reshape(-1, shape[-1])
    rows, length = w.shape
    w = torch.nn.functional.pad(w, (width, width + o))
    y = torch.nn.functional.conv1d(w[:, None], kernel[:, None, :], stride=o)
    y = y.transpose(1, 2).reshape(rows, -1)
    y = y[..., :O.resample_len(length, o, n)]
    return y.reshape(shape[:-1] + y.shape[-1:])


def _check(seed, lead, length, orig, new, method="sinc_interp_hann", lpw=6, rolloff=0.99):
    gcd = math.gcd(orig, new)
    o, n = orig // gcd, new // gcd
    kernel, width = O.sinc_resample_kernel(orig, new, gcd, lpw, rolloff, method)
    rng = np.random.default_rng(seed)
    x = torch.tensor(rng.standard_normal(lead + (length,)), requires_grad=True)
    y = _torch_resample(x, o, n, torch.tensor(kernel), width)
    assert y.shape[-1] == O.resample_len(length, o, n)
    g = rng.standard_normal(tuple(y.shape))
    (exp,) = torch.autograd.grad(y, x, grad_outputs=torch.tensor(g))
    exp = exp.numpy()
    got = V.resample_vjp(g, orig, new, gcd, kernel, width, length)
    assert got.shape == exp.shape
    np.testing.assert_allclose(got, exp, rtol=0, atol=1e-10 * max(1.0, np.abs(exp).max()))
    return got


@pytest.mark.parametrize("key", sorted(RATIOS))
def test_every_ratio(key):
    orig, new, method, lpw, rolloff, cut = RATIOS[key]
    length = cut if cut is not None else 3001
    _check(len(key), (2,), length, orig, new, method, lpw, rolloff)


def test_short_signal():
    got = _check(1, (2,), 7, 44100, 16000)  # rs_short: 7 samples give 3 outputs, every sample still gets a value
    assert np.abs(got).min() > 0


@pytest.mark.parametrize("length,mid_frame", [(441 * 7, False), (441 * 7 + 100, True), (160 * 3, True)])
def test_out_len_on_and_off_frame_boundaries(length, mid_frame):
    out_len = O.resample_len(length, 441, 160)
    assert (out_len % 160 != 0) == mid_frame
    _check(2, (1,), length, 44100, 16000, "sinc_interp_kaiser")


@pytest.mark.parametrize("lead", [(), (3,), (2, 2)], ids=["1d", "2d", "3d"])
def test_leading_dims(lead):
    _check(3, lead, 1234, 48000, 16000)


# ---- ABI validation (host only: every rejected call returns before touching a pointer) -------------------------------
def _lib_or_skip():
    from audio_b200 import _lib

    try:
        return _lib, _lib.lib()
    except ImportError:
        pytest.skip("libb200audio.so is not built")


def test_resample_backward_workspace_bytes():
    L, lib = _lib_or_skip()
    assert lib.b200a_resample_backward_workspace_bytes(0, 160, 17) == 0
    assert lib.b200a_resample_backward_workspace_bytes(441, 0, 17) == 0
    assert lib.b200a_resample_backward_workspace_bytes(441, 160, -1) == 0
    for o, n, w in ((441, 160, 17), (1, 2, 7), (2, 1, 13), (2003, 1999, 7), (2003, 1000, 13)):
        taps = 2 * w + o
        tables = 64 + 8 * n + 8 * taps + 4 * taps * n  # header, supports, tap ranges, transposed taps
        got = lib.b200a_resample_backward_workspace_bytes(o, n, w)
        assert got >= tables, (o, n, w)
        # the mma kernel's fragments are bounded by every tap group spanning every phase group
        assert got <= tables + 6 * 256 + 16 * ((taps + 7) // 8) + 512 * ((taps + 7) // 8) * ((n + 7) // 8), (o, n, w)
    # ratios the mma kernel cannot take (new' > 1024 phases) carry no fragments
    o, n, w = 2003, 1999, 7
    assert lib.b200a_resample_backward_workspace_bytes(o, n, w) < 64 + 8 * n + 8 * (2 * w + o) + 4 * (2 * w + o) * n + 6 * 256


def test_resample_backward_prepare_validation():
    L, lib = _lib_or_skip()
    fake = ctypes.c_void_p(0x1000)
    need = lib.b200a_resample_backward_workspace_bytes(441, 160, 17)
    assert lib.b200a_resample_backward_prepare(None, 441, 160, 17, fake, need, None) == L.EINVAL
    assert lib.b200a_resample_backward_prepare(fake, 441, 160, 17, None, need, None) == L.EINVAL
    assert lib.b200a_resample_backward_prepare(fake, 0, 160, 17, fake, need, None) == L.EINVAL
    assert lib.b200a_resample_backward_prepare(fake, 441, 0, 17, fake, need, None) == L.EINVAL
    assert lib.b200a_resample_backward_prepare(fake, 441, 160, -1, fake, need, None) == L.EINVAL
    assert lib.b200a_resample_backward_prepare(fake, 441, 160, 17, fake, need - 1, None) == L.EWORKSPACE


def test_resample_backward_validation():
    L, lib = _lib_or_skip()
    fake = ctypes.c_void_p(0x1000)
    length = 22050
    out_len = lib.b200a_resample_len(length, 441, 160)

    def call(o=441, n=160, w=17, rows=2, g_row_stride=out_len, out_len=out_len, length=length, grad_row_stride=length,
             ptrs=True):
        p = fake if ptrs else None
        return lib.b200a_resample_backward(p, o, n, w, p, rows, g_row_stride, out_len, p, length, grad_row_stride, None)

    assert call(o=0) == L.EINVAL
    assert call(n=0) == L.EINVAL
    assert call(w=-1) == L.EINVAL
    assert call(rows=-1) == L.EINVAL
    assert call(length=-1) == L.EINVAL
    assert call(g_row_stride=-1) == L.EINVAL
    assert call(out_len=-1) == L.EINVAL
    assert call(out_len=out_len + 1) == L.EINVAL  # must be b200a_resample_len(length, o', n')
    assert call(out_len=out_len - 1) == L.EINVAL
    assert call(ptrs=False) == L.EINVAL
    assert call(grad_row_stride=length - 1) == L.EINVAL
    assert call(rows=0, ptrs=False) == L.OK  # empty batch: no pointer is read


# ---- the resample switch ---------------------------------------------------------------------------------------------
def test_resample_switch_is_thread_local_and_off_by_default():
    import audio_b200

    def state():
        return (audio_b200.is_differentiable(), audio_b200.is_inverse_differentiable(),
                audio_b200.is_resample_differentiable())

    assert state() == (False, False, False)
    seen = []
    with audio_b200.differentiable(resample=True):
        assert state() == (True, False, True)
        t = threading.Thread(target=lambda: seen.append(state()))
        t.start()
        t.join()
        with audio_b200.differentiable():  # the plain switch keeps its meaning: front-end waveform gradients only
            assert state() == (True, False, False)
        with audio_b200.differentiable(inverse=True):  # independent of the inverse keyword
            assert state() == (True, True, False)
        with audio_b200.differentiable(inverse=True, resample=True):
            assert state() == (True, True, True)
        with audio_b200.differentiable(False, resample=True):  # resample gradients need the switch itself on
            assert state() == (False, False, False)
        assert state() == (True, False, True)
    assert seen == [(False, False, False)]
    assert state() == (False, False, False)
    audio_b200.set_differentiable(True, resample=True)
    try:
        assert audio_b200.is_resample_differentiable()
    finally:
        audio_b200.set_differentiable(False)
    assert state() == (False, False, False)


def test_forward_only_message_names_the_resample_keyword():
    from audio_b200._plans import _no_autograd

    with pytest.raises(RuntimeError, match=r"forward-only.*differentiable\(inverse=True\).*differentiable\(resample=True\)"):
        _no_autograd(torch.zeros(2, requires_grad=True))
