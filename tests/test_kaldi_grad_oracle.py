"""CPU checks of the Kaldi feature gradients: the float64 numpy VJPs of tests/kaldi_grad_oracle.py against torch.autograd
of the reference's op sequence on every argument set of the Kaldi goldens and on the edge cases of the framing, the
log floor and the energy floor; the C ABI's validation of b200a_kaldi_backward without a GPU; the kaldi= switch."""
import json
import os
import threading

import numpy as np
import pytest
import torch

from kaldi_grad_oracle import kaldi_vjp, torch_vjp

KINDS = ("spectrogram", "fbank", "mfcc")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _cases(fixture, kind):
    return [json.loads(str(a)) for a in fixture[f"{kind}_args"]]


def _grad_for(kind, wave, kw, seed):
    out = torch_vjp_shape(kind, wave, kw)
    return np.random.default_rng(seed).standard_normal(out)


def torch_vjp_shape(kind, wave, kw):
    from kaldi_grad_oracle import torch_kaldi

    return tuple(torch_kaldi(kind, torch.tensor(np.asarray(wave).reshape(-1), dtype=torch.float64), **kw).shape)


def _check(kind, wave, kw, seed=0, tol=1e-10):
    g = _grad_for(kind, wave, kw, seed)
    exp = torch_vjp(kind, wave, g, **kw)
    got = kaldi_vjp(kind, wave, g, **kw)
    scale = max(np.abs(exp).max(), 1e-300)
    assert np.abs(got - exp).max() <= tol * scale, (kind, kw, np.abs(got - exp).max() / scale)


@pytest.mark.parametrize("kind", KINDS)
def test_vjp_matches_autograd_on_kaldi_goldens(kind):
    fx = np.load(os.path.join(GOLDEN, "kaldi_goldens.npz"))
    wave = fx["wave"][0].astype(np.float64)
    cases = _cases(fx, kind)
    assert len(cases) > 50
    for i, kw in enumerate(cases):
        _check(kind, wave, kw, seed=i)


@pytest.mark.parametrize("kind", KINDS)
def test_vjp_matches_autograd_on_long_signals(kind):
    fx = np.load(os.path.join(GOLDEN, "kaldi_ref_cases.npz"))
    wave = fx["wave"][0].astype(np.float64)
    for i, kw in enumerate(_cases(fx, kind)):
        _check(kind, wave, kw, seed=100 + i)


EDGE = [
    # shift > win: a negative mirror lead; signals barely longer than one frame
    dict(frame_length=2.0, frame_shift=3.0, sample_frequency=8000.0, snip_edges=False),
    dict(frame_length=2.0, frame_shift=3.0, sample_frequency=8000.0, snip_edges=True),
    dict(frame_length=4.0, frame_shift=1.0, sample_frequency=8000.0, snip_edges=False, round_to_power_of_two=False),
    dict(frame_length=4.0, frame_shift=1.0, sample_frequency=8000.0, snip_edges=True, raw_energy=False),
    dict(energy_floor=0.0, snip_edges=False, frame_length=2.0, frame_shift=1.0, sample_frequency=8000.0),
    dict(energy_floor=1e6, frame_length=2.0, frame_shift=1.0, sample_frequency=8000.0),  # floor hit
    dict(energy_floor=1e-6, frame_length=2.0, frame_shift=1.0, sample_frequency=8000.0, raw_energy=False),  # missed
]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", range(len(EDGE)))
@pytest.mark.parametrize("signal", ["noise", "silent", "constant"])
def test_vjp_edge_cases(kind, case, signal):
    kw = dict(EDGE[case])
    if kind != "spectrogram":
        kw.update(num_mel_bins=5, low_freq=0.0)
        if kind == "fbank":
            kw.update(use_energy=True)
        else:
            kw.update(num_ceps=4)
    n = {0: 17, 1: 17, 2: 33, 3: 33}.get(case, 24)
    rng = np.random.default_rng(case)
    wave = {"noise": rng.standard_normal(n), "silent": np.zeros(n), "constant": np.full(n, 0.25)}[signal]
    _check(kind, wave, kw, seed=case)


def test_energy_floor_tie_gets_half():
    """Rectangular window, no DC removal, no pre-emphasis, a constant frame whose E equals energy_floor: the floor's
    maximum ties and each side gets half of the gradient."""
    kw = dict(window_type="rectangular", remove_dc_offset=False, preemphasis_coefficient=0.0, energy_floor=16.0,
              frame_length=2.0, frame_shift=2.0, sample_frequency=8000.0, use_energy=True, num_mel_bins=4, low_freq=0.0)
    wave = np.full(16, 1.0)  # 16-sample frames of ones: E = 16
    g = np.zeros(torch_vjp_shape("fbank", wave, kw))
    g[:, 0] = 1.0  # the energy column only
    exp = torch_vjp("fbank", wave, g, **kw)
    got = kaldi_vjp("fbank", wave, g, **kw)
    assert np.abs(got - exp).max() <= 1e-12
    # d log(E)/dx = 2 x / E = 1/8 per sample, halved by the tie
    assert np.allclose(got, 0.5 / 8.0)


def test_torchaudio_agrees_where_importable():
    ta = pytest.importorskip("torchaudio.compliance.kaldi")
    fx = np.load(os.path.join(GOLDEN, "kaldi_ref_cases.npz"))
    wave = fx["wave"][0, :4000].astype(np.float64)
    for kind in KINDS:
        for kw in _cases(fx, kind)[:4]:
            x = torch.tensor(wave[None], requires_grad=True)
            out = getattr(ta, kind)(x, **kw)
            g = np.random.default_rng(1).standard_normal(tuple(out.shape))
            out.backward(torch.from_numpy(g))
            got = kaldi_vjp(kind, wave, g, **kw)
            # the reference builds its mel banks in float32 whatever the waveform's dtype: ~1e-7 relative apart
            assert np.abs(got - x.grad[0].numpy()).max() <= 1e-5 * np.abs(got).max()


# ---- the C ABI without a GPU ---------------------------------------------------------------------------------------
def test_kaldi_backward_status_codes():
    from audio_b200 import _lib
    from audio_b200._plans import FrontendPlan

    lib = _lib.lib()
    d = FrontendPlan.make_desc(512, 512, 160, 0, False, "reflect", True, False, False, 2.0, n_mels=23)
    k = _lib.KaldiDesc()
    k.window_size, k.window_shift, k.padded_size, k.snip_edges, k.remove_dc_offset = 400, 160, 512, 1, 1
    k.preemphasis, k.energy_mode, k.energy_floor, k.energy_col, k.out_width, k.out_col0, k.use_log = 0.97, 1, 1.0, 0, 24, 1, 1
    n = lib.b200a_kaldi_backward_scratch_bytes(k, d, _lib.STAGE_MEL, 2, 16000)
    frames = 1 + (16000 - 400) // 160
    # padded 512: the fused kernel -- pre-log rows and frame gradients, no complex spectrum
    assert 2 * frames * 512 * 4 + 2 * frames * 24 * 4 <= n < 2 * frames * 512 * 4 + 2 * frames * 257 * 8
    d400 = FrontendPlan.make_desc(400, 400, 160, 0, False, "reflect", True, False, False, 2.0, n_mels=23)
    k.padded_size = 400
    assert lib.b200a_kaldi_backward_scratch_bytes(k, d400, _lib.STAGE_MEL, 2, 16000) >= (
        2 * frames * 400 * 4 + 2 * frames * 201 * 8)  # composition: the complex spectrum as well
    k.padded_size = 512
    assert lib.b200a_kaldi_backward_scratch_bytes(k, d, _lib.STAGE_COMPLEX, 2, 16000) == 0
    assert lib.b200a_kaldi_backward_scratch_bytes(k, d, _lib.STAGE_MEL, -1, 16000) == 0
    assert lib.b200a_kaldi_backward_scratch_bytes(k, d, _lib.STAGE_MEL, 2, 399) == 0
    assert lib.b200a_kaldi_backward_scratch_bytes(None, d, _lib.STAGE_MEL, 2, 16000) == 0
    args = lambda **a: [a.get("kd", k), d, 1, _lib.STAGE_MEL, 1, 2, a.get("length", 16000), 16000, a.get("g", 1), 24, 24 * frames,
                        1, a.get("scratch", 1), a.get("gw", 1), 16000, None]
    assert lib.b200a_kaldi_backward(*args(kd=None)) == _lib.EINVAL
    assert lib.b200a_kaldi_backward(*args(g=None)) == _lib.EINVAL
    assert lib.b200a_kaldi_backward(*args(scratch=None)) == _lib.EINVAL
    assert lib.b200a_kaldi_backward(*args(gw=None)) == _lib.EINVAL
    assert lib.b200a_kaldi_backward(*args(length=399)) == _lib.ESHORT
    bad = args()
    bad[3] = _lib.STAGE_FEAT
    assert lib.b200a_kaldi_backward(*bad) == _lib.EINVAL
    neg = args()
    neg[10] = -1
    assert lib.b200a_kaldi_backward(*neg) == _lib.EINVAL
    empty = args(g=None, scratch=None, gw=None)
    empty[5] = 0
    assert lib.b200a_kaldi_backward(*empty) == _lib.OK
    k.energy_mode = 3
    assert lib.b200a_kaldi_backward(*args()) == _lib.EINVAL


# ---- the switch ----------------------------------------------------------------------------------------------------
def test_kaldi_switch_is_thread_local_opt_in_and_independent():
    import audio_b200 as A

    assert not A.is_kaldi_differentiable()
    with A.differentiable(kaldi=True):
        assert A.is_kaldi_differentiable() and A.is_differentiable()
        assert not (A.is_inverse_differentiable() or A.is_resample_differentiable() or A.is_feature_differentiable())
        seen = []
        t = threading.Thread(target=lambda: seen.append(A.is_kaldi_differentiable()))
        t.start()
        t.join()
        assert seen == [False]
    assert not A.is_kaldi_differentiable()
    with A.differentiable(False, kaldi=True):
        assert not A.is_kaldi_differentiable()
    with A.differentiable(inverse=True, resample=True, features=True):
        assert not A.is_kaldi_differentiable()
    A.set_differentiable(True, kaldi=True)
    try:
        assert A.is_kaldi_differentiable()
    finally:
        A.set_differentiable(False)
    assert not A.is_kaldi_differentiable()
