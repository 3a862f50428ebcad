"""Input gradients of MFCC, LFCC, AmplitudeToDB, MelScale and SpectralCentroid without a GPU: the float64 oracle VJPs
against torch.autograd through the reference's op sequence (restated in float64 torch), including the top_db clamp's
ties; the ABI validation of the new entry points; and the feature switch."""
import ctypes
import threading

import numpy as np
import pytest
import torch

from oracle import frontend_oracle as O

import feature_grad_oracle as V
from feature_grad_oracle import torch_amplitude_to_db as _torch_amplitude_to_db
from feature_grad_oracle import torch_mfcc as _torch_mfcc
from feature_grad_oracle import torch_spectrogram as _torch_spectrogram


def _grad(fn, x, g):
    xt = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    y = fn(xt)
    (dx,) = torch.autograd.grad(y, xt, grad_outputs=torch.tensor(g, dtype=torch.float64))
    return dx.numpy()


def _close(got, exp):
    assert got.shape == exp.shape
    np.testing.assert_allclose(got, exp, rtol=0, atol=1e-10 * max(1.0, np.abs(exp).max()))


# ---- AmplitudeToDB -----------------------------------------------------------------------------------------------
def _db_input(shape, seed):
    """Positive values over 160 dB with exact zeros (below amin), exact amin values, and duplicated rows (ties)."""
    rng = np.random.default_rng(seed)
    x = 10.0 ** rng.uniform(-12, 4, shape)
    flat = x.reshape(-1, shape[-1])
    flat[0, :3] = 0.0
    flat[0, 3] = 1e-10
    flat[-1] = flat[0]  # the group maxima may tie
    return x


@pytest.mark.parametrize("shape", [(6, 9), (2, 5, 7), (3, 2, 4, 6), (2, 2, 2, 3, 5)], ids=["2d", "3d", "4d", "5d"])
@pytest.mark.parametrize("multiplier", [10.0, 20.0], ids=["power", "magnitude"])
@pytest.mark.parametrize("top_db", [None, 80.0, 0.0])
def test_amplitude_to_db(shape, multiplier, top_db):
    x = _db_input(shape, len(shape))
    g = np.random.default_rng(1).standard_normal(shape)
    exp = _grad(lambda t: _torch_amplitude_to_db(t, multiplier, 1e-10, 0.0, top_db), x, g)
    _close(V.amplitude_to_db_vjp(x, g, multiplier, 1e-10, 0.0, top_db), exp)


def test_amplitude_to_db_ties_and_clamped_rows():
    """A tie of two group maxima (count 2), elements exactly at the threshold (top_db 0 ties every maximum with it), a
    row 100 dB below a loud one (clamped), an all-zero row (below amin: zero gradient) and an offset (ref != 1)."""
    x = np.array([[4.0, 1.0, 4.0, 2.0], [1e-8, 2e-8, 3e-8, 1e-8], [0.0, 0.0, 0.0, 0.0]])
    g = np.array([[1.0, -2.0, 3.0, 0.5], [0.25, -1.0, 2.0, 4.0], [1.0, 1.0, 1.0, 1.0]])
    for top_db in (0.0, 80.0, 150.0):
        for db_multiplier in (0.0, 0.5):
            exp = _grad(lambda t: _torch_amplitude_to_db(t, 10.0, 1e-10, db_multiplier, top_db), x, g)
            got = V.amplitude_to_db_vjp(x, g, 10.0, 1e-10, db_multiplier, top_db)
            _close(got, exp)
            assert (got[2] == 0).all()
    # the two tied maxima share the routed sum: both receive it, the other loud elements do not
    exp = _grad(lambda t: _torch_amplitude_to_db(t, 10.0, 1e-10, 0.0, 0.0), x, g)
    assert exp[0, 0] != 0 and exp[0, 2] != 0 and exp[0, 1] == 0 and exp[0, 3] == 0


def test_amplitude_to_db_external_decisions():
    """With the forward's own d / maxima supplied, the oracle gives the same gradient as without."""
    x = _db_input((2, 3, 4, 5), 9)
    g = np.random.default_rng(2).standard_normal(x.shape)
    d = 10.0 * np.log10(np.maximum(x, 1e-10))
    gmax = d.reshape(2, -1).max(axis=1)
    exp = V.amplitude_to_db_vjp(x, g, 10.0, 1e-10, 0.0, 0.0)
    got = V.amplitude_to_db_vjp(x, g, 10.0, 1e-10, 0.0, 0.0, d=d.astype(np.float32).astype(np.float64),
                                gmax=gmax.astype(np.float32))
    assert np.isfinite(got).all() and got.shape == exp.shape


# ---- MFCC / LFCC -------------------------------------------------------------------------------------------------
def _waves(lead, length, seed, sr=16000, silence=True):
    """Tones + noise with a quiet row, a silent stretch and (2-D) a duplicated row, so that the clamp fires and the
    batch maximum ties."""
    rng = np.random.default_rng(seed)
    t = np.arange(length) / sr
    x = np.sin(2 * np.pi * rng.uniform(200, 3000, lead + (1,)) * t) + 0.01 * rng.standard_normal(lead + (length,))
    flat = x.reshape(-1, length)
    flat[-1] *= 1e-5
    if silence:
        flat[0, length // 3 : length // 2] = 0.0
    if flat.shape[0] >= 3:
        flat[1] = flat[0]
    return x


@pytest.mark.parametrize("lead", [(), (3,), (2, 3)], ids=["1d", "2d", "3d"])
@pytest.mark.parametrize("log_mels", [False, True])
@pytest.mark.parametrize("n_fft,mel_scale,norm", [(400, "htk", None), (256, "slaney", "slaney"), (77, "htk", None)])
def test_mfcc(lead, log_mels, n_fft, mel_scale, norm):
    hop = n_fft // 4
    n_mels, n_mfcc = 24, 13
    x = _waves(lead, 1600, n_fft)
    fb = O.melscale_fbanks(n_fft // 2 + 1, 0.0, 8000.0, n_mels, 16000, norm, mel_scale)
    dct = O.create_dct(n_mfcc, n_mels, "ortho")
    melkwargs = dict(n_fft=n_fft, hop_length=hop, n_mels=n_mels, norm=norm, mel_scale=mel_scale)
    y = O.mfcc(x, 16000, n_mfcc, "ortho", log_mels, melkwargs, fb=fb, dct=dct)
    g = np.random.default_rng(3).standard_normal(y.shape)
    exp = _grad(_torch_mfcc(fb, dct, n_fft, hop, log_mels), x, g)
    _close(V.mfcc_vjp(x, g, 16000, n_mfcc, "ortho", log_mels, melkwargs, fb=fb, dct=dct), exp)


def test_mfcc_duplicated_rows_tie_and_silent_batch():
    """2-D batch: the loudest row duplicated (count_g = 2); then an all-zero batch (every mel below amin)."""
    n_fft, hop, n_mels, n_mfcc = 256, 64, 20, 10
    fb = O.melscale_fbanks(129, 0.0, 8000.0, n_mels, 16000, None, "htk")
    dct = O.create_dct(n_mfcc, n_mels, "ortho")
    melkwargs = dict(n_fft=n_fft, hop_length=hop, n_mels=n_mels)
    for x in (_waves((3,), 1024, 4), np.zeros((2, 1024))):
        y = O.mfcc(x, 16000, n_mfcc, "ortho", False, melkwargs, fb=fb, dct=dct)
        g = np.random.default_rng(5).standard_normal(y.shape)
        exp = _grad(_torch_mfcc(fb, dct, n_fft, hop, False), x, g)
        _close(V.mfcc_vjp(x, g, 16000, n_mfcc, "ortho", False, melkwargs, fb=fb, dct=dct), exp)
    assert (exp == 0).all()


@pytest.mark.parametrize("lead", [(2,), (2, 2)], ids=["2d", "3d"])
@pytest.mark.parametrize("log_lf", [False, True])
def test_lfcc(lead, log_lf):
    n_fft, n_filter, n_lfcc = 256, 32, 12
    x = _waves(lead, 1500, 6)
    filter_mat = O.linear_fbanks(n_fft // 2 + 1, 0.0, 8000.0, n_filter, 16000)
    dct = O.create_dct(n_lfcc, n_filter, "ortho")
    speckwargs = dict(n_fft=n_fft)
    y = O.lfcc(x, 16000, n_filter, n_lfcc=n_lfcc, log_lf=log_lf, speckwargs=speckwargs, filter_mat=filter_mat, dct=dct)
    g = np.random.default_rng(7).standard_normal(y.shape)
    exp = _grad(_torch_mfcc(filter_mat, dct, n_fft, n_fft // 2, log_lf), x, g)
    got = V.lfcc_vjp(x, g, 16000, n_filter, n_lfcc=n_lfcc, log_lf=log_lf, speckwargs=speckwargs, filter_mat=filter_mat,
                     dct=dct)
    _close(got, exp)


# ---- MelScale / SpectralCentroid -----------------------------------------------------------------------------------
def test_melscale_strided():
    rng = np.random.default_rng(8)
    fb = O.melscale_fbanks(201, 0.0, 8000.0, 40, 16000, "slaney", "slaney")
    big = torch.tensor(rng.random((2, 3, 201, 40)), requires_grad=True)
    spec = big[..., ::2]  # non-contiguous spectrogram
    y = torch.matmul(spec.transpose(-1, -2), torch.tensor(fb)).transpose(-1, -2)
    g = rng.standard_normal(tuple(y.shape))
    (exp,) = torch.autograd.grad(y, spec, grad_outputs=torch.tensor(g))
    _close(V.melscale_vjp(g, fb), exp.numpy())


@pytest.mark.parametrize("n_fft,hop", [(400, 200), (256, 64)])
def test_spectral_centroid_tones(n_fft, hop):
    x = _waves((2,), 2000, 10, silence=False)  # a silent frame has D = 0: NaN, as in the reference
    window = O.hann_window(n_fft)
    y = O.spectral_centroid(x, 16000, 0, window, n_fft, hop, n_fft)
    g = np.random.default_rng(11).standard_normal(y.shape)
    wt = torch.tensor(window)

    def fn(t):
        spec = _torch_spectrogram(t, 0, wt, n_fft, hop, n_fft, 1.0)
        freqs = torch.linspace(0, 8000, steps=1 + n_fft // 2, dtype=torch.float64).reshape((-1, 1))
        return (freqs * spec).sum(dim=-2) / spec.sum(dim=-2)

    _close(V.spectral_centroid_vjp(x, g, 16000, 0, window, n_fft, hop, n_fft), _grad(fn, x, g))


# ---- ABI validation (host only: every rejected call returns before touching a pointer) -------------------------------
def _lib_or_skip():
    from audio_b200 import _lib

    try:
        return _lib, _lib.lib()
    except ImportError:
        pytest.skip("libb200audio.so is not built")


def _desc(n_mels=40, n_mfcc=13, log_mels=False, **kw):
    from audio_b200._plans import FrontendPlan

    d = FrontendPlan.make_desc(512, 512, 128, 0, True, "reflect", True, False, False, 2.0, n_mels, n_mfcc, log_mels)
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def test_mfcc_backward_validation():
    L, lib = _lib_or_skip()
    fake = ctypes.c_void_p(0x1000)

    def call(d=None, rows=2, frames=50, rpg=2, top_db=80.0, gs=(1, 1, 1), ptrs=True, feat=True, gmax=True, scratch=True):
        p = fake if ptrs else None
        return lib.b200a_mfcc_backward(_desc() if d is None else d, p, p, *gs, fake if feat else None, p,
                                       fake if gmax else None, rows, frames, rpg, top_db, fake if scratch else None, p, None)

    assert call(d=_desc(hop=0)) == L.EINVAL
    assert call(d=_desc(n_mfcc=0)) == L.EINVAL
    assert call(d=_desc(n_mels=0)) == L.EINVAL
    assert call(rows=-1) == L.EINVAL
    assert call(frames=-1) == L.EINVAL
    assert call(gs=(-1, 1, 1)) == L.EINVAL
    assert call(rpg=0) == L.EINVAL
    assert call(ptrs=False) == L.EINVAL
    assert call(feat=False) == L.EINVAL  # the clamp's masks read the forward's features
    assert call(scratch=False) == L.EINVAL
    assert call(rows=0, ptrs=False, feat=False, scratch=False) == L.OK
    # n_mels x n_mfcc past the shared-memory limit
    assert call(d=_desc(n_mels=512, n_mfcc=400)) == L.EUNSUPPORTED
    # scratch: per-tile partials of 64 frames + one float per group, each table 256-byte aligned
    assert lib.b200a_mfcc_backward_scratch_bytes(_desc(), 4, 100, 2) == 256 + 256
    assert lib.b200a_mfcc_backward_scratch_bytes(_desc(), 256, 626, 256) == 20224 + 256
    assert lib.b200a_mfcc_backward_scratch_bytes(_desc(), 4, 100, 0) == 0
    assert lib.b200a_mfcc_backward_scratch_bytes(_desc(n_mfcc=0), 4, 100, 2) == 0


def test_amplitude_to_db_backward_validation():
    L, lib = _lib_or_skip()
    fake = ctypes.c_void_p(0x1000)

    def call(groups=2, elems=100, g_stride=1, top_db=80.0, ptrs=True, gmax=True, scratch=True):
        p = fake if ptrs else None
        return lib.b200a_amplitude_to_db_backward(p, p, g_stride, groups, elems, 10.0, 1e-10, 0.0, top_db,
                                                  fake if gmax else None, fake if scratch else None, p, None)

    assert call(groups=-1) == L.EINVAL
    assert call(elems=-1) == L.EINVAL
    assert call(g_stride=2) == L.EINVAL
    assert call(ptrs=False) == L.EINVAL
    assert call(scratch=False) == L.EINVAL
    assert call(groups=0, ptrs=False, scratch=False) == L.OK
    assert lib.b200a_amplitude_to_db_backward_scratch_bytes(3, 5000) == 256 + 256
    assert lib.b200a_amplitude_to_db_backward_scratch_bytes(-1, 5000) == 0


def test_apply_fbank_and_ratio_backward_validation():
    L, lib = _lib_or_skip()
    fake = ctypes.c_void_p(0x1000)
    f = lib.b200a_apply_fbank_backward
    assert f(fake, 2, 0, 10, 1, 1, 1, fake, 201, fake, None) == L.EINVAL
    assert f(fake, 2, 40, 10, 1, 1, 1, fake, 0, fake, None) == L.EINVAL
    assert f(fake, -1, 40, 10, 1, 1, 1, fake, 201, fake, None) == L.EINVAL
    assert f(fake, 2, 40, 10, -1, 1, 1, fake, 201, fake, None) == L.EINVAL
    assert f(None, 2, 40, 10, 1, 1, 1, fake, 201, fake, None) == L.EINVAL
    assert f(None, 0, 40, 10, 1, 1, 1, None, 201, None, None) == L.OK
    assert f(fake, 70000, 40, 10, 1, 1, 1, fake, 201, fake, None) == L.EUNSUPPORTED
    r = lib.b200a_ratio_backward
    assert r(fake, fake, -1, 10, 1, 1, fake, None) == L.EINVAL
    assert r(fake, fake, 2, 10, -1, 1, fake, None) == L.EINVAL
    assert r(None, fake, 2, 10, 1, 1, fake, None) == L.EINVAL
    assert r(None, None, 0, 10, 1, 1, None, None) == L.OK


# ---- the feature switch ---------------------------------------------------------------------------------------------
def test_feature_switch_is_thread_local_and_off_by_default():
    import audio_b200

    def state():
        return (audio_b200.is_differentiable(), audio_b200.is_inverse_differentiable(),
                audio_b200.is_resample_differentiable(), audio_b200.is_feature_differentiable())

    assert state() == (False, False, False, False)
    seen = []
    with audio_b200.differentiable(features=True):
        assert state() == (True, False, False, True)
        t = threading.Thread(target=lambda: seen.append(state()))
        t.start()
        t.join()
        with audio_b200.differentiable():  # the plain switch keeps its meaning
            assert state() == (True, False, False, False)
        with audio_b200.differentiable(inverse=True, resample=True):  # independent of the other keywords
            assert state() == (True, True, True, False)
        with audio_b200.differentiable(resample=True, features=True):
            assert state() == (True, False, True, True)
        with audio_b200.differentiable(False, features=True):  # feature gradients need the switch itself on
            assert state() == (False, False, False, False)
        assert state() == (True, False, False, True)
    assert seen == [(False, False, False, False)]
    assert state() == (False, False, False, False)
    audio_b200.set_differentiable(True, features=True)
    try:
        assert audio_b200.is_feature_differentiable()
    finally:
        audio_b200.set_differentiable(False)
    assert state() == (False, False, False, False)


def test_forward_only_message_names_the_features_keyword():
    from audio_b200._plans import _no_autograd

    with pytest.raises(RuntimeError, match=r"forward-only.*differentiable\(inverse=True\).*differentiable\(resample=True\)"
                                           r".*differentiable\(features=True\)"):
        _no_autograd(torch.zeros(2, requires_grad=True))
