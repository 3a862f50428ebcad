"""The RNN-T feature extractors on the GPU (audio_b200.pipelines.RNNTFeatureExtractor, b200audio::rnnt_features).

Forward bars.  On one launch the features equal the float64 chain evaluated on the kernel's own mel values with the
kernel's float32 decisions to 1e-6 max(1, |y|).  Against the reference's float32 fixture and the float64 oracle, the
forward bar 1e-4 |e| + 1e-4 rms(e) holds wherever the reference's own float32 run meets it, and elsewhere the error is
at most 2x that run's; elements whose float32 and float64 decisions fall on different pieces are excluded, counted, and
must be under 0.1 %.

Gradient bar, against the float64 VJP.  The relative L2 error is at most 2x that of the same op sequence run in float32
torch on the CPU (plus 2e-7, a few float32 ulps, so that the bar does not hinge on the CPU's vector width); measured on
an H100: 3.7e-7 / 4.3e-7 / 3.1e-7 (1-D / 2-D / expanded upstream gradient) against the CPU's 2.5e-7 / 2.5e-7 / 1.8e-7.
The largest error does not meet 2x the CPU's: it was measured at 1.1e-6 to 1.5e-6 of the gradient's largest magnitude
against the CPU's 1.8e-7 to 2.6e-7.  Its cause is upstream of the chain: the Stockham FFT's absolute round-off is larger
than the CPU's float32 FFT's (both inside the forward's 1e-4 bar), and the chain's d log(x) = dx / x passes a quiet
band's share of it on relative to the band.  That bound is pinned at 1e-5 of the gradient's largest magnitude, well
inside the ceiling of DESIGN.md 3.8 (relative L2 <= 5e-3, largest error <= 2e-2), which is asserted too.
"""
import json
import math
import os
import time

import numpy as np
import pytest
import torch

import audio_b200
from audio_b200 import _ops
from audio_b200.pipelines import RNNTFeatureExtractor, _gain

import rnnt_grad_oracle as R

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LENGTHS = (201, 3200, 16000, 37920)


@pytest.fixture(scope="module")
def fx():
    with np.load(os.path.join(GOLDEN, "rnnt_ref_cases.npz")) as z:
        return {k: z[k] for k in z.files}


def _stats_path(tmp_path_factory, fx, name):
    path = tmp_path_factory.mktemp(name) / "global_stats.json"
    path.write_text(json.dumps({"mean": fx[f"stats_{name}_mean"].tolist(),
                                "invstddev": fx[f"stats_{name}_invstddev"].tolist()}))
    return str(path)


@pytest.fixture(scope="module")
def libri(tmp_path_factory, fx):
    return _stats_path(tmp_path_factory, fx, "librispeech")


@pytest.fixture(scope="module")
def ted(tmp_path_factory, fx):
    return _stats_path(tmp_path_factory, fx, "tedlium3")


def _np(t):
    return t.detach().double().cpu().numpy()


def _input(fx, n, i):
    return torch.from_numpy(fx[f"base_{n}"] * fx["levels"][i])


def _launch(e, waves, lengths=None, out_frames=None):
    """One b200audio::rnnt_features launch with mel_out: (features, mel values)."""
    mel_mod = e.pipeline["0"]
    plan = mel_mod._fused_plan()
    ws = plan.workspace(mel_mod.spectrogram.window, mel_mod.mel_scale.fb, None)
    flat = waves.contiguous()
    frames = plan.frames(flat.shape[1]) if out_frames is None else out_frames
    desc_i, desc_f = plan._packed_desc()
    lens = None if lengths is None else torch.tensor(lengths, dtype=torch.int64, device=DEV)
    return _ops.rnnt_features(flat, ws, desc_i, desc_f, lens, e._packed_stats(ws.device), _gain, frames, 0,
                              flat.shape[1], True)


def _stats(fx, name="librispeech"):
    return fx[f"stats_{name}_mean"], fx[f"stats_{name}_invstddev"]


def _fill(fx, name):
    mean, invstd = _stats(fx, name)
    return (np.float32(0) - mean) * invstd


# ---- forward --------------------------------------------------------------------------------------------------------
def test_chain_exact_on_the_kernels_own_mel(fx, libri):
    e = RNNTFeatureExtractor(libri).to(DEV)
    mean, invstd = _stats(fx)
    seen = set()
    for n in LENGTHS:
        waves = torch.stack([_input(fx, n, i) for i in range(3)]).to(DEV)
        out, mel = _launch(e, waves)
        m = mel.cpu().numpy()
        p = R.pieces32(m)
        seen |= set(np.unique(p).tolist())
        exp = R.chain(m, mean, invstd, p)
        err = np.abs(_np(out) - exp)
        assert (err <= 1e-6 * np.maximum(1.0, np.abs(exp))).all(), f"n={n}: worst {err.max():.3e}"
    assert seen == {1, 2, 3}


def _check_against_reference(got, ref, orc, flip, what):
    rms = float(np.sqrt(np.mean(orc**2)))
    tol = 1e-4 * np.abs(orc) + 1e-4 * rms
    e_gpu, e_ref = np.abs(got - orc), np.abs(ref - orc)
    ok = ~flip
    meets = (e_ref <= tol) & ok
    assert (e_gpu[meets] <= tol[meets]).all(), f"{what}: worst {(e_gpu[meets] / tol[meets]).max():.3f} of the bar"
    rest = ~(e_ref <= tol) & ok
    assert (e_gpu[rest] <= 2.0 * e_ref[rest]).all(), f"{what}: beyond 2x the reference's own error"


@pytest.mark.parametrize("n", LENGTHS)
def test_extractors_against_reference_and_oracle(fx, libri, n):
    full = RNNTFeatureExtractor(libri).to(DEV)
    stream = RNNTFeatureExtractor(libri, right_padding=0).to(DEV)
    mean, invstd = _stats(fx)
    flips = total = 0
    for i in range(3):
        x = _input(fx, n, i)
        f, lf = full(x.to(DEV))
        s, ls = stream(x.to(DEV))
        t = 1 + n // 160
        assert f.shape == (t + 4, 80) and f.stride() == (80, 1) and f.is_contiguous() and f.dtype == torch.float32
        assert lf.dtype == torch.int64 and lf.device.type == "cpu" and lf.tolist() == [t + 4]
        assert ls.tolist() == [t] and s.shape == (t, 80)
        assert torch.equal(f[:t], s) and (f[t:] == 0).all() and not torch.signbit(f[t:]).any()
        mel64 = np.swapaxes(R.mel_spectrogram(x.numpy().astype(np.float64), **R.MEL_ARGS), -1, -2)
        flip = R.pieces32(mel64) != R.pieces64(mel64)
        flips += int(flip.sum())
        total += flip.size
        orc = R.chain(mel64, mean, invstd)
        _check_against_reference(_np(s), fx[f"stream_{n}_{i}"].astype(np.float64), orc, flip, f"n={n} level {i}")
        assert np.array_equal(fx[f"full_{n}_{i}"][:t], fx[f"stream_{n}_{i}"])
    assert flips <= 1e-3 * total, f"{flips} of {total} elements on a breakpoint"


def test_ragged_batch_against_recipe_and_streaming_extractor(fx, ted):
    e = RNNTFeatureExtractor(ted, right_padding=0).to(DEV)
    base = fx["base_37920"]
    lens, levels = fx["batch_lengths"].tolist(), fx["batch_levels"]
    total = max(lens) + 37  # the batch buffer is longer than its longest row
    waves = torch.zeros(len(lens), total)
    for r, (n, lv) in enumerate(zip(lens, levels)):
        waves[r, :n] = torch.from_numpy(base[:n] * lv)
        waves[r, n:] = 7.0  # samples past a row's length are never read
    out, frames = e.forward_batch(waves.to(DEV), torch.tensor(lens))
    assert frames.dtype == torch.int32 and frames.device.type == "cpu"
    assert frames.tolist() == fx["batch_frames"].tolist()
    exp = fx["batch_feats"]
    assert out.shape == exp.shape
    fill = _fill(fx, "tedlium3")
    mean, invstd = _stats(fx, "tedlium3")
    got = out.cpu().numpy()
    for r, n in enumerate(lens):
        t = int(frames[r])
        alone, _ = e(waves[r, :n].to(DEV))
        assert torch.equal(out[r, :t].cpu(), alone.cpu()), f"row {r} differs from the extractor on its own"
        assert (got[r, t:] == fill).all(), f"row {r}: fill frames are not (0 - mean) * invstddev"
        mel64 = np.zeros((exp.shape[1], 80))
        mel64[:t] = np.swapaxes(R.mel_spectrogram((base[:n] * levels[r]).astype(np.float64), **R.MEL_ARGS), -1, -2)
        flip = R.pieces32(mel64) != R.pieces64(mel64)
        _check_against_reference(got[r].astype(np.float64), exp[r].astype(np.float64), R.chain(mel64, mean, invstd),
                                 flip, f"row {r}")
    # a sequence works as well as a CPU tensor; bad lengths raise the reference's errors
    out2, _ = e.forward_batch(waves.to(DEV), lens)
    assert torch.equal(out, out2)
    with pytest.raises(RuntimeError, match="padding size"):
        e.forward_batch(waves.to(DEV), [100] + lens[1:])
    with pytest.raises(ValueError):
        e.forward_batch(waves.to(DEV), [total + 1] + lens[1:])
    with pytest.raises(ValueError):
        e.forward_batch(waves.to(DEV), torch.tensor(lens, device=DEV))


def test_silence_padding_and_determinism(fx, libri):
    full = RNNTFeatureExtractor(libri).to(DEV)
    f, _ = full(torch.zeros(16000, device=DEV))
    assert (f[-4:] == 0).all()
    assert (f[:-4].cpu().numpy() == _fill(fx, "librispeech")).all()
    x = _input(fx, 37920, 1).to(DEV)
    a, _ = full(x)
    b, _ = full(x)
    assert torch.equal(a, b)


def test_batch_rows_alone_equal_their_batch_rows(libri):
    e = RNNTFeatureExtractor(libri, right_padding=0).to(DEV)
    g = torch.Generator().manual_seed(3)
    waves = (0.1 * torch.randn(256, 160000, generator=g)).to(DEV)
    out, frames = e.forward_batch(waves)
    assert out.shape == (256, 1001, 80) and frames.tolist() == [1001] * 256
    out2, _ = e.forward_batch(waves)
    assert torch.equal(out, out2)
    for r in (0, 1, 77, 255):
        alone, _ = e(waves[r])
        assert torch.equal(out[r], alone)


def test_only_library_kernels_and_no_host_sync(fx, libri):
    e = RNNTFeatureExtractor(libri).to(DEV)
    x = _input(fx, 16000, 0).to(DEV)
    e(x)  # builds the workspace and the packed statistics
    # a profiler session now and then comes back without some of its kernel records, more often for short sessions late
    # in a long test run (as test_gpu_generic_fft.launched_kernels): the session is padded with 20 ms of idle time at
    # both ends, and the deterministic call runs again, up to ten sessions, until both expected kernels were recorded
    for _ in range(10):
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            time.sleep(0.02)
            e(x)
            torch.cuda.synchronize()
            time.sleep(0.02)
        names = {ev.name for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA}
        if any("stft_rnnt_kernel" in n for n in names) and any("fill_kernel" in n for n in names):
            break
    kernels = {n for n in names if "Memcpy" not in n and "Memset" not in n}
    assert kernels and all("stft_rnnt_kernel" in n or "fill_kernel" in n for n in kernels), kernels
    assert any("stft_rnnt_kernel" in n for n in kernels) and any("fill_kernel" in n for n in kernels)
    assert not any("Memcpy" in n for n in names), names
    waves = torch.stack([_input(fx, 16000, i) for i in range(3)]).to(DEV)
    e.forward_batch(waves, [16000, 9000, 4000])  # warm the pinned-memory pool
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        e(x)
        e.forward_batch(waves)
        e.forward_batch(waves, [16000, 9000, 4000])
        e.forward_batch(waves, torch.tensor([16000, 12000, 201]))
    finally:
        torch.cuda.set_sync_debug_mode(0)


# ---- gradients ------------------------------------------------------------------------------------------------------
def _grad_input(fx):
    """2.37 s with a silent middle fifth, its thirds at levels 1, 1e-3 and 1e-5: all three pieces and silence."""
    base = fx["base_37920"].copy()
    n = base.shape[0]
    base[n // 3 : 2 * n // 3] *= np.float32(1e-3)
    base[2 * n // 3 :] *= np.float32(1e-5)
    return base


def _cpu_float32_grad(x, g, fb, mean, invstd, right_padding):
    """The reference op sequence in float32 torch on the CPU: torch.stft, |.|^2, the mel matrix, the chain, the pad."""
    xt = torch.tensor(x, requires_grad=True)
    spec = torch.stft(xt, 400, 160, window=torch.hann_window(400), center=True, pad_mode="reflect",
                      return_complex=True).abs().pow(2.0)
    mel = torch.matmul(spec.transpose(-1, -2), fb)
    y = mel * _gain
    y[y > math.e] = torch.log(y[y > math.e])
    y[y <= math.e] = y[y <= math.e] / math.e
    y = (y - torch.from_numpy(mean)) * torch.from_numpy(invstd)
    if right_padding:
        y = torch.nn.functional.pad(y, (0, 0, 0, right_padding))
    (y * torch.from_numpy(g)).sum().backward()
    return xt.grad.double().numpy()


def _check_grad(got, exp, f32, what):
    err, err32 = np.abs(got - exp), np.abs(f32 - exp)
    scale = float(np.abs(exp).max())
    rel = float(np.sqrt((err**2).sum() / (exp**2).sum()))
    rel32 = float(np.sqrt((err32**2).sum() / (exp**2).sum()))
    print(f"{what}: gpu relative L2 {rel:.3e} max {err.max() / scale:.3e}; "
          f"float32 cpu relative L2 {rel32:.3e} max {err32.max() / scale:.3e}")
    assert rel <= 5e-3 and err.max() <= 2e-2 * scale, f"{what}: relative L2 {rel:.3e}, max {err.max() / scale:.3e}"
    assert rel <= 2.0 * rel32 + 2e-7, f"{what}: relative L2 {rel:.3e} against float32 cpu {rel32:.3e}"
    assert err.max() <= 1e-5 * scale, f"{what}: largest error {err.max() / scale:.3e} of the largest magnitude"


def test_gradient_1d_and_uniform_batch(fx, libri):
    mean, invstd = _stats(fx)
    full = RNNTFeatureExtractor(libri).to(DEV)
    fb = full.pipeline["0"].mel_scale.fb.cpu()
    fb64 = fb.double().numpy()
    x = _grad_input(fx)
    mel64 = np.swapaxes(R.mel_spectrogram(x.astype(np.float64), fb=fb64, **R.MEL_ARGS), -1, -2)
    p = R.pieces32(mel64)
    assert {1, 2, 3} <= set(np.unique(p).tolist()) and (mel64 == 0).all(axis=1).any()
    rng = np.random.default_rng(9)
    t = mel64.shape[0]
    g = rng.standard_normal((t + 4, 80)).astype(np.float32)
    xd = torch.from_numpy(x).to(DEV).requires_grad_(True)
    with audio_b200.differentiable(features=True):
        f, _ = full(xd)
        (f * torch.from_numpy(g).to(DEV)).sum().backward()
    with torch.no_grad():
        f0, _ = full(xd)
    assert torch.equal(f, f0)  # the forward with grad is the no-grad forward, bit for bit
    exp = R.features_vjp(x, g, mean, invstd, fb64, pieces=p)
    _check_grad(_np(xd.grad), exp, _cpu_float32_grad(x, g, fb, mean, invstd, 4), "1-D")

    stream = RNNTFeatureExtractor(libri, right_padding=0).to(DEV)
    waves = np.stack([x, x[::-1].copy() * np.float32(0.01)])
    g2 = rng.standard_normal((2, t, 80)).astype(np.float32)
    wd = torch.from_numpy(waves).to(DEV).requires_grad_(True)
    with audio_b200.differentiable(features=True):
        out, frames = stream.forward_batch(wd)
        (out * torch.from_numpy(g2).to(DEV)).sum().backward()
    assert frames.tolist() == [t, t]
    mel2 = np.swapaxes(R.mel_spectrogram(waves.astype(np.float64), fb=fb64, **R.MEL_ARGS), -1, -2)
    exp2 = R.features_vjp(waves, g2, mean, invstd, fb64, pieces=R.pieces32(mel2))
    _check_grad(_np(wd.grad), exp2, _cpu_float32_grad(waves, g2, fb, mean, invstd, 0), "2-D")
    # an expanded (stride 0) upstream gradient
    xe = torch.from_numpy(x).to(DEV).requires_grad_(True)
    with audio_b200.differentiable(features=True):
        f, _ = full(xe)
        f.sum().backward()
    ge = np.ones((t + 4, 80), np.float32)
    _check_grad(_np(xe.grad), R.features_vjp(x, ge, mean, invstd, fb64, pieces=p),
                _cpu_float32_grad(x, ge, fb, mean, invstd, 4), "expanded")


def test_gradient_raises(fx, libri):
    full = RNNTFeatureExtractor(libri).to(DEV)
    x = _input(fx, 16000, 0).to(DEV).requires_grad_(True)
    with pytest.raises(RuntimeError, match=r"forward-only.*features=True"):
        full(x)
    with audio_b200.differentiable():  # the plain switch does not cover the feature chain
        with pytest.raises(RuntimeError, match="forward-only"):
            full(x)
    with audio_b200.differentiable(features=True):
        with pytest.raises(RuntimeError, match="ragged"):
            full.forward_batch(x[None].expand(2, -1), [16000, 9000])
        for name in ("mean", "invstddev"):
            buf = getattr(full.pipeline["3"], name)
            buf.requires_grad_(True)
            try:
                with pytest.raises(RuntimeError, match=name):
                    full(x)
            finally:
                buf.requires_grad_(False)
        for mod, name in ((full.pipeline["0"].spectrogram, "window"), (full.pipeline["0"].mel_scale, "fb")):
            buf = getattr(mod, name)
            buf.requires_grad_(True)
            try:
                with pytest.raises(RuntimeError, match=name):
                    full(x)
            finally:
                buf.requires_grad_(False)
        f, _ = full(x)
        (g,) = torch.autograd.grad(f.sum(), x, create_graph=True)
        with pytest.raises(RuntimeError):
            g.sum().backward()
        f, _ = full(x)
        with torch.no_grad():
            full.pipeline["3"].mean.add_(0.0)  # an in-place edit of a saved buffer
        with pytest.raises(RuntimeError, match="modified by an inplace operation"):
            f.sum().backward()
