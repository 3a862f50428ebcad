"""Inverse path (SURVEY.md 8f.3): F.inverse_spectrogram / T.InverseSpectrogram over the istft kernels.

CPU: the oracle's torch.istft restatement against outputs of the reference (tests/golden/make_istft_golden.py).
GPU: the product against the same fixtures and the oracle, and the reference's own round-trip property
(transforms/transforms_test_impl.py:84-110: spectrogram -> inverse spectrogram returns the signal)."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import frontend_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def istft_ref():
    return np.load(os.path.join(GOLDEN, "istft_ref_cases.npz"))


def _cases(fx):
    return [(i, json.loads(str(c))) for i, c in enumerate(fx["cases"])]


def _stable(c, frames, out_len):
    """Mask of output positions whose window envelope is not vanishing (float32 y/env is noise where env ~ 1e-8)."""
    w = np.zeros(c["n_fft"])
    left = (c["n_fft"] - c["win"]) // 2
    w[left:left + c["win"]] = np.hanning(c["win"] + 1)[:-1] if c["center"] else np.hamming(c["win"] + 1)[:-1]
    expected = c["n_fft"] + c["hop"] * (frames - 1)
    env = np.zeros(max(expected, (c["n_fft"] // 2 if c["center"] else 0) + out_len + 2 * c["pad"]))
    for t in range(frames):
        env[t * c["hop"]:t * c["hop"] + c["n_fft"]] += w * w
    start = (c["n_fft"] // 2 if c["center"] else 0) + c["pad"]
    seg = env[start:start + out_len]
    return (seg > 1e-3 * env.max()) | (seg == 0)


def test_oracle_istft_matches_reference(istft_ref):
    for i, c in _cases(istft_ref):
        exp = istft_ref[f"out_{i}"]
        got = O.inverse_spectrogram(istft_ref[f"spec_{i}"], c["length"], c["pad"], istft_ref[f"window_{i}"], c["n_fft"],
                                    c["hop"], c["win"], c["normalized"], c["center"])
        assert got.shape == exp.shape
        ok = _stable(c, istft_ref[f"spec_{i}"].shape[-1], exp.shape[-1])
        assert np.abs(got - exp)[..., ok].max() <= 5e-6 * max(np.abs(exp).max(), 1.0), i
    # a consistent STFT inverts exactly
    x = np.random.default_rng(0).standard_normal((2, 4000))
    w = O.hann_window(400)
    spec = O.spectrogram(x, 0, w, 400, 100, 400, None, False)
    y = O.inverse_spectrogram(spec, 4000, 0, w, 400, 100, 400)
    assert np.abs(y - x).max() < 1e-9


def test_inverse_module_surface_cpu():
    import audio_b200.transforms as T

    inv = T.InverseSpectrogram(n_fft=512)
    assert (inv.n_fft, inv.win_length, inv.hop_length, inv.pad, inv.center, inv.onesided) == (512, 512, 256, 0, True, True)
    assert set(inv.state_dict()) == {"window"}
    with pytest.raises(ValueError, match="complex dtype"):
        inv(torch.zeros(2, 257, 10))
    with pytest.raises(RuntimeError, match="no CPU or ATen fallback"):
        inv(torch.zeros(2, 257, 10, dtype=torch.complex64))


@pytest.mark.gpu
def test_gpu_inverse_matches_reference_and_oracle(istft_ref):
    import audio_b200.functional as F

    for i, c in _cases(istft_ref):
        spec = torch.from_numpy(istft_ref[f"spec_{i}"]).cuda()
        window = torch.from_numpy(istft_ref[f"window_{i}"]).cuda()
        with pytest.warns(UserWarning) if i == 5 else _nullcontext():
            got = F.inverse_spectrogram(spec, c["length"], c["pad"], window, c["n_fft"], c["hop"], c["win"], c["normalized"],
                                        c["center"])
        exp = istft_ref[f"out_{i}"]
        assert tuple(got.shape) == exp.shape
        ok = _stable(c, spec.shape[-1], exp.shape[-1])
        ora = O.inverse_spectrogram(istft_ref[f"spec_{i}"], c["length"], c["pad"], istft_ref[f"window_{i}"], c["n_fft"], c["hop"],
                                    c["win"], c["normalized"], c["center"])
        scale = max(np.abs(exp).max(), 1.0)
        g = got.cpu().numpy()
        assert np.abs(g - ora)[..., ok].max() <= 1e-5 * scale, i
        assert np.abs(g - exp)[..., ok].max() <= 1e-5 * scale, i
        # the transposed (frame-major) layout our own forward produces is accepted as is
        got_t = F.inverse_spectrogram(spec.transpose(-1, -2).contiguous().transpose(-1, -2), c["length"], c["pad"], window,
                                      c["n_fft"], c["hop"], c["win"], c["normalized"], c["center"]) if i != 5 else got
        assert torch.equal(got_t, got)


class _nullcontext:
    def __enter__(self):
        return None

    def __exit__(self, *a):
        return False


@pytest.mark.gpu
@pytest.mark.parametrize("n_fft,hop,win", [(400, 100, 400), (512, 128, 512), (1024, 256, 1024), (600, 150, 400),
                                           (2048, 512, 2048), (401, 100, 401)])
def test_gpu_round_trip(n_fft, hop, win):
    """Spectrogram(power=None) -> InverseSpectrogram returns the waveform (reference transforms_test_impl.py:84-110)."""
    import audio_b200.transforms as T

    x = torch.randn(2, 3, 12000, generator=torch.Generator().manual_seed(n_fft)).cuda()
    fwd = T.Spectrogram(n_fft=n_fft, hop_length=hop, win_length=win, power=None).cuda()
    inv = T.InverseSpectrogram(n_fft=n_fft, hop_length=hop, win_length=win).cuda()
    y = inv(fwd(x), 12000)
    assert tuple(y.shape) == (2, 3, 12000)
    assert (y - x).abs().max().item() < 2e-5
    with pytest.raises(RuntimeError, match="window overlap add min"):
        T.InverseSpectrogram(n_fft=n_fft, hop_length=win, win_length=win // 2).cuda()(fwd(x)[..., :5], None)


# ---- Griffin-Lim --------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gl_goldens():
    return np.load(os.path.join(GOLDEN, "griffinlim_goldens.npz"))


@pytest.mark.parametrize("tag,momentum", [("0", 0.0), ("0_99", 0.99)])
def test_oracle_griffinlim_matches_librosa(gl_goldens, tag, momentum):
    """The reference's own golden test (functional/librosa_compatibility_test_impl.py:16-54): float64, atol 5e-5."""
    got = O.griffinlim(gl_goldens["specgram"], O.hann_window(400), 400, 100, 400, 1, 8, momentum, 16000)
    np.testing.assert_allclose(got[0], gl_goldens[f"librosa_{tag}"], atol=5e-5, rtol=1e-7)
    assert np.abs(got - gl_goldens[f"ref_{tag}"]).max() < 1e-4  # the reference ran with a float32-built window


def test_griffinlim_surface_cpu():
    import audio_b200.transforms as T

    gl = T.GriffinLim()
    assert (gl.n_fft, gl.n_iter, gl.win_length, gl.hop_length, gl.power, gl.momentum, gl.length, gl.rand_init) == (
        400, 32, 400, 200, 2.0, 0.99, None, True)
    with pytest.raises(ValueError, match="momentum must be in the range"):
        T.GriffinLim(momentum=1.0)
    import audio_b200.functional as F

    with pytest.raises(ValueError, match="momentum must be in range"):
        F.griffinlim(torch.zeros(1, 201, 10), torch.hann_window(400), 400, 100, 400, 1, 8, 1.5, None, False)


@pytest.mark.gpu
@pytest.mark.parametrize("tag,momentum", [("0", 0.0), ("0_99", 0.99)])
def test_gpu_griffinlim_matches_librosa(gl_goldens, tag, momentum):
    """Same case in float32 on the GPU: 8 iterations of istft / stft round-off stay within 1e-3 of the float64 golden
    (signal amplitude ~1); the reference's float32 run sits at the same distance."""
    import audio_b200.functional as F

    spec = torch.from_numpy(gl_goldens["specgram"]).float().cuda()
    got = F.griffinlim(spec, torch.hann_window(400).cuda(), 400, 100, 400, 1, 8, momentum, 16000, False)
    assert tuple(got.shape) == (1, 16000)
    assert np.abs(got.cpu().numpy()[0] - gl_goldens[f"librosa_{tag}"]).max() < 1e-3


@pytest.mark.gpu
def test_gpu_griffinlim_module_defaults(gl_goldens):
    import audio_b200.transforms as T

    spec = torch.from_numpy(gl_goldens["power_spec_512"]).cuda()
    gl = T.GriffinLim(n_fft=512, hop_length=128, length=6000, rand_init=False).cuda()
    got = gl(spec).cpu().numpy()
    assert got.shape == (2, 6000)
    oracle = O.griffinlim(gl_goldens["power_spec_512"], O.hann_window(512), 512, 128, 512, 2.0, 32, 0.99, 6000)
    # 32 momentum iterations amplify float32 round-off; the reference's own float32 run differs from float64 by 2e-3
    assert np.abs(got - oracle).max() < 2e-2 * np.abs(oracle).max()
    assert np.abs(got - gl_goldens["ref_512"]).max() < 2e-2 * np.abs(oracle).max()
    # the recovered signal's magnitude spectrogram is close to the target (what Griffin-Lim optimises)
    rebuilt = T.Spectrogram(n_fft=512, hop_length=128, power=2.0).cuda()(torch.from_numpy(got).cuda())
    rel = (rebuilt - spec).norm() / spec.norm()
    assert rel.item() < 0.35
    # random initial phase: runs, is reproducible under torch.manual_seed, and converges about as well
    gl_r = T.GriffinLim(n_fft=512, hop_length=128, length=6000).cuda()
    torch.manual_seed(1)
    a = gl_r(spec)
    torch.manual_seed(1)
    b = gl_r(spec)
    assert torch.equal(a, b)
    rel_r = (T.Spectrogram(n_fft=512, hop_length=128, power=2.0).cuda()(a) - spec).norm() / spec.norm()
    assert rel_r.item() < 0.35


# ---- phase vocoder / TimeStretch / PitchShift (SURVEY.md 8f.4) -----------------------------------------------------
@pytest.fixture(scope="module")
def vocoder_ref():
    return np.load(os.path.join(GOLDEN, "vocoder_ref_cases.npz"))


PITCH_CASES = {"up12": (16000, 12), "down12": (16000, -12), "up7_1k": (1000, 7), "down5_1k": (1000, -5)}


def test_oracle_vocoder_matches_reference(vocoder_ref):
    """float64 oracle vs the reference's float32 run: the reference accumulates thousands of radians of phase in
    float32 (~1e-3 rad of round-off), which bounds the agreement at ~1e-3 of the largest magnitude."""
    import math

    pa = np.linspace(0, math.pi * 128, 257)
    for rate in (0.8, 1.3, 2.0):
        got, exp = O.phase_vocoder(vocoder_ref["spec"], rate, pa), vocoder_ref[f"pv_{rate}"]
        assert got.shape == exp.shape
        assert np.abs(got - exp).max() <= 2e-3 * np.abs(exp).max()
        assert np.abs(np.abs(got) - np.abs(exp)).max() <= 1e-5 * np.abs(exp).max()  # magnitudes carry no phase round-off
    for tag, (sr, steps) in PITCH_CASES.items():
        got, exp = O.pitch_shift(vocoder_ref["wave"], sr, steps), vocoder_ref[f"ps_{tag}"]
        assert got.shape == exp.shape and np.abs(got - exp).max() <= 2e-3 * np.abs(exp).max(), tag


def test_vocoder_surface_cpu():
    import audio_b200.transforms as T

    ts = T.TimeStretch(hop_length=128, n_freq=257, fixed_rate=1.3)
    assert tuple(ts.phase_advance.shape) == (257, 1) and set(ts.state_dict()) == {"phase_advance"}
    with pytest.raises(ValueError, match="must pass a valid rate"):
        T.TimeStretch()(torch.zeros(1, 201, 5, dtype=torch.complex64))
    ps = T.PitchShift(16000, 4)
    assert (ps.n_fft, ps.win_length, ps.hop_length, ps.orig_freq, ps.gcd) == (512, 512, 128, 20158, 2)
    x = torch.zeros(1, 257, 5, dtype=torch.complex64)
    assert T.TimeStretch(fixed_rate=1.0, n_freq=257)(x) is x  # rate 1: returned as is, like the reference


@pytest.mark.gpu
def test_gpu_phase_vocoder_and_time_stretch(vocoder_ref):
    import math

    import audio_b200.transforms as T

    spec = torch.from_numpy(vocoder_ref["spec"]).cuda()
    pa = np.linspace(0, math.pi * 128, 257)
    for rate in (0.8, 1.3, 2.0):
        got = T.TimeStretch(hop_length=128, n_freq=257, fixed_rate=rate).cuda()(spec)
        exp, ora = vocoder_ref[f"pv_{rate}"], O.phase_vocoder(vocoder_ref["spec"], rate, pa)
        assert tuple(got.shape) == exp.shape and got.dtype == torch.complex64
        g = got.cpu().numpy()
        scale = np.abs(ora).max()
        assert np.abs(g - ora).max() <= 1e-4 * scale, rate   # phase carried in double: closer to float64 than the reference
        assert np.abs(g - exp).max() <= 2e-3 * scale, rate   # the reference's own float32 phase round-off
    got = T.TimeStretch(n_freq=257).cuda()(spec.reshape(1, 2, 257, -1), 1.3)
    assert tuple(got.shape) == (1, 2, 257, 37)


@pytest.mark.gpu
@pytest.mark.parametrize("tag", list(PITCH_CASES))
def test_gpu_pitch_shift(vocoder_ref, tag):
    import audio_b200.functional as F
    import audio_b200.transforms as T

    sr, steps = PITCH_CASES[tag]
    x = torch.from_numpy(vocoder_ref["wave"]).cuda()
    exp = vocoder_ref[f"ps_{tag}"]
    ora = O.pitch_shift(vocoder_ref["wave"], sr, steps)
    scale = np.abs(ora).max()
    got = F.pitch_shift(x, sr, steps).cpu().numpy()
    assert got.shape == exp.shape
    assert np.abs(got - ora).max() <= 1e-3 * scale and np.abs(got - exp).max() <= 2e-3 * scale
    mod = T.PitchShift(sr, steps).cuda()
    got_m = mod(x.reshape(1, 2, -1)).cpu().numpy()
    assert got_m.shape == (1, 2, 6000) and np.abs(got_m[0] - got).max() <= 1e-5 * scale
