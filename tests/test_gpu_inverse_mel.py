"""InverseMelScale on the GPU: parity with the reference's outputs (tests/golden/make_inverse_mel_golden.py) and the
float64 oracle, layouts, errors, plan reuse, the opt-in mel gradient, and the mel -> linear -> Griffin-Lim chain."""
import os

import numpy as np
import pytest
import torch

from conftest import scaled_tol_close
from inverse_mel_oracle import inverse_mel_scale, inverse_mel_scale_vjp
from oracle import frontend_oracle as O

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# name: (n_stft, n_mels, sample_rate, f_min, f_max, norm, mel_scale), as in the fixture's generator
CONFIGS = {
    "c201_64_8k": (201, 64, 8000, 0.0, None, None, "htk"),
    "c513_128_16k": (513, 128, 16000, 0.0, None, None, "htk"),
    "c513_80_16k": (513, 80, 16000, 0.0, None, None, "htk"),
    "c1025_128_22k_slaney": (1025, 128, 22050, 0.0, None, "slaney", "slaney"),
    "c257_40_16k_band": (257, 40, 16000, 20.0, 7600.0, None, "htk"),
    "c201_40_16k": (201, 40, 16000, 0.0, None, None, "htk"),
}


@pytest.fixture(scope="module")
def inv_ref():
    with np.load(os.path.join(GOLDEN, "inverse_mel_ref_cases.npz")) as z:
        return {k: z[k] for k in z.files}


def _module(name, inv_ref, driver="gels"):
    import audio_b200.transforms as T

    n_stft, n_mels, sr, f_min, f_max, norm, scale = CONFIGS[name]
    mod = T.InverseMelScale(n_stft, n_mels, sr, f_min, f_max, norm, scale, driver).cuda()
    assert np.array_equal(mod.fb.cpu().numpy(), inv_ref[f"{name}_fb"])  # the same filterbank as the reference's
    return mod


def _dist(a, e):
    e = np.asarray(e, dtype=np.float64)
    return float(np.max(np.abs(np.asarray(a, np.float64) - e) / (np.abs(e) + np.sqrt(np.mean(e ** 2)))))


@pytest.mark.parametrize("name", list(CONFIGS))
@pytest.mark.parametrize("driver", ["gels", "gelsd"])
def test_parity_with_reference_and_oracle(inv_ref, name, driver):
    mod = _module(name, inv_ref, driver)
    for kind in ("speech", "rand"):
        x = inv_ref[f"{name}_{kind}_in"]
        got = mod(torch.from_numpy(x).cuda()).cpu().numpy()
        exp, orc = inv_ref[f"{name}_{kind}_out"], inverse_mel_scale(x, inv_ref[f"{name}_fb"])
        scaled_tol_close(got, exp, 1e-4, f"{name} {kind} vs reference ({_dist(got, exp):.3g})")
        scaled_tol_close(got, orc, 1e-5, f"{name} {kind} vs oracle ({_dist(got, orc):.3g})")


def _expected_strides(lead, n_stft, frames):
    # the reference's layout: a contiguous (..., T, n_stft) tensor seen as (..., n_stft, T)
    return torch.empty(lead + (frames, n_stft)).transpose(-1, -2).stride()


def test_layouts_and_strides(inv_ref):
    import audio_b200.transforms as T

    mod = _module("c513_80_16k", inv_ref)
    spec = T.MelSpectrogram(16000, n_fft=1024, hop_length=256, n_mels=80, power=1.0).cuda()
    mel = spec(torch.randn(3, 16000, device="cuda"))
    assert mel.stride()[-2] == 1  # frame-major
    frames = mel.shape[-1]
    mod(mel)  # builds the plan (one device-to-host copy of fb)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU]) as prof:
        a = mod(mel)
    names = {e.key for e in prof.key_averages()}
    assert not names & {"aten::copy_", "aten::clone", "aten::contiguous"}, names  # the frame-major input is read in place
    assert a.shape == (3, 513, frames) and a.stride() == _expected_strides((3,), 513, frames)
    b = mod(mel.contiguous())
    assert b.stride() == a.stride() and torch.equal(a, b)  # both input layouts give the same bits
    c = mod(mel[1])
    assert c.shape == (513, frames) and c.stride() == (1, 513) and torch.equal(c, a[1])
    m4 = mel.reshape(1, 3, 80, frames).expand(2, 3, 80, frames)
    d = mod(m4)
    assert d.shape == (2, 3, 513, frames) and d.stride() == _expected_strides((2, 3), 513, frames)
    assert torch.equal(d[1, 2], a[2])
    with pytest.raises(RuntimeError, match="0 elements"):  # the reference's view(-1, n_mels, 0) raises the same
        mod(mel[..., :0])


def test_rank_deficient_and_tall_banks(inv_ref):
    import audio_b200.transforms as T

    for n_stft, key in ((201, "s201_128_16k"), (65, "s65_128_16k")):
        m = torch.rand(1, 128, 3, device="cuda")
        with pytest.warns(UserWarning):
            mod = T.InverseMelScale(n_stft, 128, 16000).cuda()
        with pytest.raises(torch.linalg.LinAlgError, match="does not have full rank"):
            mod(m)
        assert "does not have full rank" in str(inv_ref[f"{key}_gels"])
        for drv in ("gelsy", "gelsd", "gelss"):
            with pytest.warns(UserWarning):
                mod = T.InverseMelScale(n_stft, 128, 16000, driver=drv).cuda()
            with pytest.raises(RuntimeError, match="not supported"):
                mod(m)


def test_plan_is_rebuilt_only_when_fb_changes(inv_ref):
    mod = _module("c201_64_8k", inv_ref)
    x = torch.from_numpy(inv_ref["c201_64_8k_rand_in"]).cuda()
    a = mod(x)
    plan = mod._plan._plan
    b = mod(x)
    assert mod._plan._plan is plan and torch.equal(a, b)
    mod.fb.mul_(2.0)  # x = fb G^-1 m halves
    c = mod(x)
    assert mod._plan._plan is not plan
    scaled_tol_close(c.cpu().numpy(), 0.5 * a.cpu().numpy(), 1e-5, "fb * 2")


@pytest.mark.parametrize("name", list(CONFIGS))
def test_gradient(inv_ref, name):
    import audio_b200

    mod = _module(name, inv_ref)
    fb = inv_ref[f"{name}_fb"]
    x = torch.from_numpy(inv_ref[f"{name}_grad_in"]).cuda()
    up = torch.from_numpy(inv_ref[f"{name}_grad_up"]).cuda()
    with torch.no_grad():
        plain = mod(x)
    with audio_b200.differentiable(features=True):
        xg = x.clone().requires_grad_()
        out = mod(xg)
        assert torch.equal(out.detach(), plain)  # the forward is bit-identical with and without grad
        (g1,) = torch.autograd.grad(out, xg, up)
        (g2,) = torch.autograd.grad(mod(xg), xg, up)
    assert torch.equal(g1, g2)  # no atomics: reruns are bit-identical
    got = g1.cpu().numpy()
    mask = plain.cpu().numpy() > 0
    orc = inverse_mel_scale_vjp(inv_ref[f"{name}_grad_in"], fb, inv_ref[f"{name}_grad_up"], mask)
    scaled_tol_close(got, orc, 1e-5, f"{name} grad vs oracle ({_dist(got, orc):.3g})")
    exp = inv_ref[f"{name}_grad"]
    scaled_tol_close(got, exp, 1e-4, f"{name} grad vs reference ({_dist(got, exp):.3g})")
    # a non-contiguous, expanded upstream gradient reads through its strides
    with audio_b200.differentiable(features=True):
        (g3,) = torch.autograd.grad(mod(xg), xg, torch.ones(()).cuda().expand(out.shape))
        (g4,) = torch.autograd.grad(mod(xg), xg, torch.ones_like(out))
    assert torch.equal(g3, g4)


def test_gradient_switches(inv_ref):
    import audio_b200

    mod = _module("c201_64_8k", inv_ref)
    x = torch.from_numpy(inv_ref["c201_64_8k_grad_in"]).cuda().requires_grad_()
    with pytest.raises(RuntimeError, match=r"forward-only.*InverseMelScale"):
        mod(x)
    with audio_b200.differentiable(inverse=True, resample=True, kaldi=True, vocoder=True):
        with pytest.raises(RuntimeError, match="forward-only"):
            mod(x)
    with audio_b200.differentiable(features=True):
        mod.fb.requires_grad_()
        with pytest.raises(RuntimeError, match="fb requires grad"):
            mod(x)


def test_mel_to_audio_chain_stays_on_device_and_matches_oracle():
    """MelSpectrogram(power=1) -> InverseMelScale -> GriffinLim(rand_init=False, n_iter=8): the reference's mel -> audio
    recipe, against the float64 oracle of the last two stages fed the same mel spectrogram (the GriffinLim bar of
    tests/test_inverse.py)."""
    import audio_b200.transforms as T

    g = torch.Generator().manual_seed(7)
    wave = (0.3 * torch.randn(2, 8000, generator=g)).cuda()
    mel = T.MelSpectrogram(8000, n_fft=400, hop_length=100, n_mels=64, power=1.0).cuda()(wave)
    inv = T.InverseMelScale(201, 64, 8000).cuda()
    gl = T.GriffinLim(n_fft=400, hop_length=100, power=1.0, n_iter=8, length=8000, rand_init=False).cuda()
    lin = inv(mel)
    out = gl(lin)
    assert out.is_cuda and lin.is_cuda and out.shape == (2, 8000)
    lin_o = inverse_mel_scale(mel.cpu().numpy(), inv.fb.cpu().numpy())
    scaled_tol_close(lin.cpu().numpy(), lin_o, 1e-5, "linear spectrogram")
    out_o = O.griffinlim(lin_o, O.hann_window(400), 400, 100, 400, 1.0, 8, 0.99, 8000)
    assert np.abs(out.cpu().numpy() - out_o).max() < 1e-3 * max(1.0, np.abs(out_o).max())


def test_reference_quality_gauge():
    """transforms_test_impl.py:21-60 of the reference: |Spectrogram| -> MelScale -> InverseMelScale against the
    spectrogram, 8 kHz white noise, n_fft 400, 64 mels; shares of elements within 1e-1 / 1e-3 / 1e-5 relative."""
    import audio_b200.transforms as T

    g = torch.Generator().manual_seed(0)
    noise = (torch.rand(2, 8000, generator=g) * 2 - 1).cuda()
    expected = T.Spectrogram(n_fft=400, power=1).cuda()(noise)
    mel = T.MelScale(n_mels=64, sample_rate=8000, n_stft=201).cuda()(expected)
    result = T.InverseMelScale(201, n_mels=64, sample_rate=8000).cuda()(mel)
    rel = torch.abs((result - expected) / (expected + 1e-60))
    assert (rel < 1e-1).float().mean().item() > 0.2
    assert (rel < 1e-3).float().mean().item() > 5e-3
    assert (rel < 1e-5).float().mean().item() > 1e-5


def test_reference_switch_picks_up_inverse_mel_scale():
    """B200A_REFERENCE=1 routes InverseMelScale through ``__all__`` like every other transform."""
    import subprocess
    import sys

    pytest.importorskip("torchaudio")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = r"""
import sys, warnings
sys.path.insert(0, sys.argv[1])
import torch
warnings.simplefilter("ignore")
import audio_b200.transforms as T
import torchaudio.transforms as R
m = torch.rand(2, 40, 6, generator=torch.Generator().manual_seed(0))
assert torch.equal(T.InverseMelScale(201, 40)(m), R.InverseMelScale(201, 40)(m))
print("ok")
"""
    out = subprocess.run([sys.executable, "-c", code, root], env=dict(os.environ, B200A_REFERENCE="1"),
                         capture_output=True, text=True)
    assert out.returncode == 0 and "ok" in out.stdout, out.stderr[-2000:]
