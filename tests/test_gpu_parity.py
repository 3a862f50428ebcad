"""GPU parity tests: the CUDA product (through the C ABI) vs
  * the golden fixtures (librosa vectors of the reference's tests + the reference's own outputs),
  * the CPU oracle on seeded inputs,
  * size-independent properties at BASELINE.json's full sizes.
Floating-point bar (BASELINE.json north_star): 1e-4 relative to the reference CPU path, stated
as |a-e| <= 1e-4*|e| + 1e-4*rms(e) (SURVEY.md 8c); integer bookkeeping / shapes / strides exact.
"""
import math

import numpy as np
import pytest
import torch
from conftest import assert_close, scaled_tol_close
from golden_cases import LIBROSA_FRAMES, MELSPECTROGRAM, MFCC, RESAMPLE, SPECTROGRAM, SPEC_VARIANTS

import audio_b200.functional as F
import audio_b200.transforms as T
from oracle import frontend_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def host(t):
    if t.is_complex():
        return t.cpu().numpy()
    return t.float().cpu().numpy()


def spec_module(window=None, **kw):
    if window == "hamming":
        kw["window_fn"] = torch.hamming_window
    return T.Spectrogram(**kw).to(DEV)


# ---------------- librosa goldens of the reference's own tests ---------------------------------
@pytest.mark.parametrize("i", range(len(SPECTROGRAM)))
def test_spectrogram_librosa(librosa_transforms, i):
    got = spec_module(**SPECTROGRAM[i])(dev(librosa_transforms["whitenoise"]))[0]
    assert_close(host(got)[..., LIBROSA_FRAMES], librosa_transforms[f"spectrogram_{i}"], rtol=1e-4, atol=1e-4)


def test_spectrogram_complex_librosa(librosa_transforms):
    got = spec_module(n_fft=400, hop_length=200, power=None)(dev(librosa_transforms["whitenoise"]))[0]
    assert got.dtype == torch.complex64
    assert_close(host(got.abs())[..., LIBROSA_FRAMES], librosa_transforms["spectrogram_complex"], rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("i", range(len(MELSPECTROGRAM)))
def test_melspectrogram_librosa(librosa_transforms, i):
    m = T.MelSpectrogram(sample_rate=16000, window_fn=torch.hann_window, **MELSPECTROGRAM[i]).to(DEV)
    got = m(dev(librosa_transforms["sinusoid"]))[0]
    assert_close(host(got)[..., LIBROSA_FRAMES], librosa_transforms[f"melspectrogram_{i:02d}"], rtol=1e-5, atol=5e-4)


@pytest.mark.parametrize("i", range(len(MFCC)))
def test_mfcc_librosa(librosa_transforms, i):
    cfg = dict(MFCC[i])
    n_mfcc = cfg.pop("n_mfcc")
    m = T.MFCC(sample_rate=16000, n_mfcc=n_mfcc, norm="ortho", melkwargs=cfg).to(DEV)
    got = m(dev(librosa_transforms["whitenoise"]))[0]
    # the reference asserts atol=5e-4 in float64; in float32 the dB of near-floor bins moves by
    # ~1e-3 (its own CPU fp32 run differs from this golden by the same amount)
    assert_close(host(got)[..., LIBROSA_FRAMES], librosa_transforms[f"mfcc_{i}"], rtol=1e-4, atol=5e-3)


def test_amplitude_to_db_librosa(librosa_transforms):
    spec = spec_module(n_fft=400, hop_length=100)(dev(librosa_transforms["whitenoise"]))
    got = T.AmplitudeToDB("power", 80.0)(spec)[0]
    assert_close(host(got)[..., LIBROSA_FRAMES], librosa_transforms["power_to_db"], rtol=1e-3, atol=1e-3)
    got = T.AmplitudeToDB("magnitude", 80.0)(spec)[0]
    assert_close(host(got)[..., LIBROSA_FRAMES], librosa_transforms["magnitude_to_db"], rtol=1e-3, atol=1e-3)


# ---------------- the reference's own outputs (tests/golden/ref_cases.npz) ---------------------
def test_config1_spectrogram(ref_cases):
    got = spec_module(n_fft=512, hop_length=256)(dev(ref_cases["c1_in"]))
    assert tuple(got.shape) == (1, 257, 63)
    assert got.stride() == (257 * 63, 1, 257)  # frame-major memory, as torch.stft returns it
    scaled_tol_close(host(got), ref_cases["c1_out"], what="config 1")


@pytest.mark.parametrize("name", sorted(SPEC_VARIANTS))
def test_spectrogram_variants(ref_cases, name):
    got = spec_module(**SPEC_VARIANTS[name])(dev(ref_cases["spec_in"]))
    scaled_tol_close(host(got), ref_cases[f"spec_{name}"], what=name)


@pytest.mark.parametrize("n_fft,hop,key", [(400, 200, "spec_complex400"), (1024, 256, "spec_complex1024")])
def test_spectrogram_complex(ref_cases, n_fft, hop, key):
    got = spec_module(n_fft=n_fft, hop_length=hop, power=None)(dev(ref_cases["spec_in"]))
    ref = ref_cases[key][..., 0] + 1j * ref_cases[key][..., 1]
    scaled_tol_close(host(got), ref, what=key)


def test_functional_spectrogram_matches_module(ref_cases):
    x = dev(ref_cases["spec_in"])
    w = torch.hann_window(400, device=DEV)
    got = F.spectrogram(x, 0, w, 400, 200, 400, 2.0, False)
    scaled_tol_close(host(got), ref_cases["spec_default400"])
    got = F.spectrogram(x.reshape(1, 1, 1600), 0, w, 400, 200, 400, 2.0, False)  # leading dims are packed
    assert tuple(got.shape) == (1, 1, 201, 9)


MEL_CASES = {
    "mel_c2_out": dict(sample_rate=16000, n_fft=1024, hop_length=256, n_mels=80),
    "mel_default_out": dict(sample_rate=16000),
    "mel_rnnt_out": dict(sample_rate=16000, n_fft=400, hop_length=160, n_mels=80),
    "mel_slaney2048_out": dict(sample_rate=22050, n_fft=2048, hop_length=512, n_mels=128, norm="slaney", mel_scale="slaney", f_max=8000.0),
    "mel_512_p1_out": dict(sample_rate=16000, n_fft=512, hop_length=128, n_mels=40, power=1.0),
    "mel_256_out": dict(sample_rate=16000, n_fft=256, hop_length=64, n_mels=80),
}


@pytest.mark.parametrize("key", sorted(MEL_CASES))
def test_melspectrogram_reference(ref_cases, key):
    import warnings

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = T.MelSpectrogram(**MEL_CASES[key]).to(DEV)
    got = m(dev(ref_cases["mel_in"]))
    scaled_tol_close(host(got), ref_cases[key], what=key)


def test_melspectrogram_scaled_rows_and_strides(ref_cases):
    m = T.MelSpectrogram(16000, n_fft=1024, hop_length=256, n_mels=80).to(DEV)
    got = m(dev(ref_cases["mel_scaled_in"]))
    assert tuple(got.shape) == (4, 80, 8) and got.stride() == (80 * 8, 1, 80)
    g, ref = host(got), ref_cases["mel_scaled_out"]
    for r in range(4):  # loud (x1000), quiet (x1e-3), silent, unit rows
        scaled_tol_close(g[r], ref[r], what=f"row {r}")
    assert np.all(g[2] == 0.0)


def test_mfcc_reference_batch_coupling(ref_cases):
    """MFCC against the reference's own outputs under the stated rule |a-e| <= 1e-4 |e| + 1e-4 rms(e) (SURVEY.md 8c).
    The slack is pinned, not asserted: tests/test_oracle_golden.py::test_mfcc_tolerance_is_pinned shows the
    reference's fp32 CPU run itself sits within 6 % of that bound from the fp64 oracle on these very cases."""
    kw = dict(n_fft=1024, hop_length=256, n_mels=80)
    mf = T.MFCC(16000, n_mfcc=40, melkwargs=kw).to(DEV)
    x, xs = dev(ref_cases["mel_in"]), dev(ref_cases["mel_scaled_in"])
    scaled_tol_close(host(mf(x)), ref_cases["mfcc_x_out"], what="mfcc_x")
    scaled_tol_close(host(mf(xs)), ref_cases["mfcc_2d_out"], what="mfcc_2d")  # ONE cut-off for the batch
    scaled_tol_close(host(mf(xs[:, None, :])), ref_cases["mfcc_3d_out"], what="mfcc_3d")  # per-item cut-off
    scaled_tol_close(host(mf(xs[0])), ref_cases["mfcc_1d_out"], what="mfcc_1d")
    mfl = T.MFCC(16000, n_mfcc=13, log_mels=True, melkwargs=dict(n_fft=400, hop_length=160, n_mels=23)).to(DEV)
    scaled_tol_close(host(mfl(x)), ref_cases["mfcc_log_out"], what="mfcc_log")
    mfn = T.MFCC(16000, n_mfcc=20, norm=None, melkwargs=dict(n_fft=512, hop_length=256, n_mels=64)).to(DEV)
    scaled_tol_close(host(mfn(x)), ref_cases["mfcc_nonorm_out"], what="mfcc_nonorm")
    scaled_tol_close(host(T.MFCC().to(DEV)(x)), ref_cases["mfcc_default_out"], what="mfcc_default")


def test_amplitude_to_db_reference(ref_cases):
    p = dev(ref_cases["db_in"])
    assert_close(host(T.AmplitudeToDB("power", 80.0)(p)), ref_cases["db_power_top80_3d"], rtol=1e-5, atol=2e-4)
    assert_close(host(T.AmplitudeToDB("power", 80.0)(p[:, None])), ref_cases["db_power_top80_4d"], rtol=1e-5, atol=2e-4)
    assert_close(host(T.AmplitudeToDB("magnitude")(p)), ref_cases["db_mag_none"], rtol=1e-5, atol=2e-4)


def test_melscale_standalone(ref_cases):
    x = dev(ref_cases["mel_in"])
    spec = spec_module(n_fft=1024, hop_length=256)(x)  # (4, 513, 8) transposed view
    got = T.MelScale(80, 16000, n_stft=513).to(DEV)(spec)
    scaled_tol_close(host(got), ref_cases["mel_c2_out"])
    got = T.MelScale(80, 16000, n_stft=513).to(DEV)(spec.contiguous())  # other strides, same answer
    scaled_tol_close(host(got), ref_cases["mel_c2_out"])


@pytest.mark.parametrize("key", sorted(RESAMPLE))
def test_resample_reference(ref_cases, key):
    cut, kw = RESAMPLE[key]
    x = ref_cases["rs_in"] if cut is None else ref_cases["rs_in"][:, :cut]
    got = host(T.Resample(**kw).to(DEV)(dev(x)))
    ref = ref_cases[key]
    assert got.shape == ref.shape
    assert np.abs(got - ref).max() <= 1e-4 * np.abs(ref).max(), key


def test_resample_functional_and_layout(ref_cases):
    x = dev(ref_cases["rs_in"])
    got = F.resample(x, 44100, 16000, resampling_method="sinc_interp_kaiser")
    assert np.abs(host(got) - ref_cases["rs_func_kaiser"]).max() <= 1e-4 * np.abs(ref_cases["rs_func_kaiser"]).max()
    got = F.resample(x, 3, 2)
    assert np.abs(host(got) - ref_cases["rs_func_hann_3_2"]).max() <= 1e-4
    r = T.Resample(44100, 16000).to(DEV)
    y = r(x.reshape(1, 1, -1))
    assert tuple(y.shape) == (1, 1, 1600)
    # 3 Hz cosine known-answer test of the reference (functional_impl.py:22-49)
    for up, down in [(2, 1), (1, 2), (3, 2), (8, 5)]:
        sr, sr2 = 1000 * down, 1000 * up
        t = torch.arange(0, 2, 1 / sr, dtype=torch.float64)
        t2 = torch.arange(0, 2, 1 / sr2, dtype=torch.float64)
        wav = torch.cos(2 * math.pi * 3 * t).float()[None].to(DEV)
        est = F.resample(wav, sr, sr2)[0].cpu()
        ref = torch.cos(2 * math.pi * 3 * t2).float()
        assert est.shape[-1] == math.ceil(sr2 * wav.shape[-1] / sr)
        n = min(est.shape[-1], ref.shape[-1])
        assert torch.allclose(est[20 : n - 20], ref[20 : n - 20], atol=1e-1, rtol=1e-4)


# ---------------- seeded inputs vs the CPU oracle ------------------------------------------------
@pytest.mark.parametrize("n_fft,hop,n_mels,rows,length", [
    (1024, 256, 80, 5, 9000), (512, 128, 80, 3, 5000), (256, 64, 40, 7, 3001), (2048, 512, 80, 2, 12345),
    (400, 160, 80, 3, 7777), (1024, 256, 80, 1, 513), (1024, 256, 80, 2, 1024), (1024, 100, 64, 2, 4099),
])
def test_melspectrogram_vs_oracle(n_fft, hop, n_mels, rows, length):
    g = torch.Generator().manual_seed(1000 + n_fft + rows)
    x = torch.randn(rows, length, generator=g)
    import warnings

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = T.MelSpectrogram(16000, n_fft=n_fft, hop_length=hop, n_mels=n_mels).to(DEV)
    got = host(m(x.to(DEV)))
    exp = O.mel_spectrogram(x.numpy(), sample_rate=16000, n_fft=n_fft, hop_length=hop, n_mels=n_mels,
                            fb=m.mel_scale.fb.cpu().numpy())
    scaled_tol_close(got, exp, what=f"mel n_fft={n_fft}")
    # every row is independent: batch == item by item (batch_consistency_test.py:102-107)
    one = host(m(x[:1].to(DEV)))
    assert np.array_equal(one[0], got[0])


def test_tonal_and_silent_rows_vs_oracle():
    sr, n = 16000, 16000
    t = torch.arange(n) / sr
    x = torch.stack([torch.sin(2 * math.pi * 300 * t), torch.zeros(n), 0.25 * torch.sin(2 * math.pi * 3000 * t) + 1e-3 * torch.randn(n)])
    m = T.MelSpectrogram(sr, n_fft=1024, hop_length=256, n_mels=80).to(DEV)
    got = host(m(x.to(DEV)))
    exp = O.mel_spectrogram(x.numpy(), sample_rate=sr, n_fft=1024, hop_length=256, n_mels=80, fb=m.mel_scale.fb.cpu().numpy())
    for r in range(3):
        scaled_tol_close(got[r], exp[r], what=f"row {r}")
    mf = T.MFCC(sr, n_mfcc=40, melkwargs=dict(n_fft=1024, hop_length=256, n_mels=80)).to(DEV)
    got = host(mf(x[:, None, :].to(DEV)))
    exp = O.mfcc(x[:, None, :].numpy(), sr, 40, "ortho", False, dict(n_fft=1024, hop_length=256, n_mels=80),
                 fb=m.mel_scale.fb.cpu().numpy(), dct=mf.dct_mat.cpu().numpy())
    assert_close(got, exp, rtol=1e-4, atol=2e-2)  # silent row sits exactly on the -100 dB floor
    assert np.allclose(got[1, 0, 1:], 0.0, atol=1e-3)  # constant -100 dB frame -> only c0 is non-zero


@pytest.mark.parametrize("orig,new,method", [(44100, 16000, "sinc_interp_kaiser"), (16000, 44100, "sinc_interp_hann"),
                                             (48000, 16000, "sinc_interp_hann"), (8000, 22050, "sinc_interp_kaiser")])
def test_resample_vs_oracle(orig, new, method):
    g = torch.Generator().manual_seed(orig + new)
    x = torch.randn(3, 6001, generator=g)
    r = T.Resample(orig, new, resampling_method=method).to(DEV)
    got = host(r(x.to(DEV)))
    exp = O.resample(x.numpy(), orig, new, resampling_method=method)
    assert got.shape == exp.shape
    assert np.abs(got - exp).max() <= 1e-4 * np.abs(exp).max()


# ---------------- error behaviour -----------------------------------------------------------------
def test_errors_on_gpu():
    with pytest.raises(RuntimeError, match="should be less than"):
        spec_module(n_fft=512)(torch.randn(1, 256, device=DEV))  # reflect pad needs n_fft//2 < L
    with pytest.raises(RuntimeError, match="too short"):
        spec_module(n_fft=512, center=False)(torch.randn(1, 100, device=DEV))
    with pytest.raises(TypeError, match="float32"):
        spec_module()(torch.randn(1, 4000, device=DEV, dtype=torch.float64))
    with pytest.raises(RuntimeError, match="forward-only"):
        spec_module()(torch.randn(1, 4000, device=DEV, requires_grad=True))
    with pytest.raises(TypeError, match="Expected floating point"):
        T.Resample(16000, 8000).to(DEV)(torch.zeros(1, 100, dtype=torch.int32, device=DEV))
    out = spec_module()(torch.randn(0, 4000, device=DEV))  # empty batch
    assert tuple(out.shape) == (0, 201, 21)


def test_window_update_invalidates_plan():
    m = spec_module(n_fft=256, hop_length=64)
    x = torch.randn(2, 2000, device=DEV)
    a = m(x).clone()
    m.window.fill_(1.0)  # in-place change of the buffer must be picked up (tensor version stamp)
    b = m(x)
    exp = O.spectrogram(x.cpu().numpy(), 0, np.ones(256), 256, 64, 256, 2.0)
    scaled_tol_close(host(b), exp)
    assert not torch.allclose(a, b)


# ---------------- BASELINE.json full sizes: properties -----------------------------------------
def test_config2_full_size_properties():
    """MelSpectrogram n_fft=1024 hop=256 n_mels=80 on 256 x 160000 (BASELINE config 2)."""
    B, L = 256, 160000
    g = torch.Generator(device=DEV).manual_seed(1234)
    x = torch.randn(B, L, device=DEV, generator=g)
    m = T.MelSpectrogram(16000, n_fft=1024, hop_length=256, n_mels=80).to(DEV)
    y = m(x)
    assert tuple(y.shape) == (B, 80, 626) and y.stride() == (80 * 626, 1, 80)
    assert torch.isfinite(y).all() and (y >= 0).all()
    # (1) rows are independent and the result does not depend on batch position
    idx = [0, 17, 255]
    assert torch.equal(m(x[idx]), y[idx])
    # (2) power is quadratic in the input: mel(2x) == 4 mel(x) exactly in binary fp
    assert torch.equal(m(2.0 * x[:8]), 4.0 * y[:8])
    # (3) interior frames are shift-covariant: dropping two hops of input shifts frames by two,
    #     bit for bit (frames are transformed in (even, odd) pairs, so an even shift keeps the pairing)
    z = m(x[:4, 512:])
    assert torch.equal(z[:, :, 2:600], y[:4, :, 4:602])
    z1 = m(x[:4, 256:])  # odd shift: same values up to the pair partner's round-off
    assert torch.allclose(z1[:, :, 2:600], y[:4, :, 3:601], rtol=5e-5, atol=1e-4)  # TF32x3 products: ~2^-21
    # (4) a sample of rows against the fp64 oracle
    exp = O.mel_spectrogram(x[idx].cpu().numpy(), sample_rate=16000, n_fft=1024, hop_length=256, n_mels=80,
                            fb=m.mel_scale.fb.cpu().numpy())
    scaled_tol_close(host(y[idx]), exp, what="config 2 rows")
    # (5) Parseval with the mel filters' partition of unity is not exact; check the plain power
    #     spectrogram instead: sum_k |X_k|^2 (two-sided) == n_fft * sum_n (w x)^2
    s = T.Spectrogram(n_fft=1024, hop_length=256, onesided=False).to(DEV)(x[:2])
    frames = torch.nn.functional.pad(x[:2, None], (512, 512), mode="reflect")[:, 0].unfold(-1, 1024, 256)
    energy = ((frames * m.spectrogram.window) ** 2).sum(-1).double() * 1024
    assert torch.allclose(s.sum(1).double(), energy, rtol=2e-5)


def test_config3_full_size_properties():
    """Resample 44.1k -> 16k kaiser on 1024 x 220500 (BASELINE config 3), in two halves to bound memory."""
    B, L = 1024, 220500
    r = T.Resample(44100, 16000, resampling_method="sinc_interp_kaiser").to(DEV)
    g = torch.Generator(device=DEV).manual_seed(4321)
    x = torch.randn(B, L, device=DEV, generator=g)
    y = r(x)
    assert tuple(y.shape) == (B, 80000) and y.stride() == (80160, 1)
    assert torch.isfinite(y).all()
    # linearity, row independence
    a = r(x[:4] * 3.0 - x[4:8])
    # (TF32 x 3 tensor-core kernel: ~2^-21 relative per product; north-star tolerance 1e-4 relative)
    assert torch.allclose(a, 3.0 * y[:4] - y[4:8], atol=1e-4)
    assert torch.equal(r(x[[5, 900]]), y[[5, 900]])
    # shifting the input by one polyphase period (441 samples) shifts the output by 160
    z = r(x[:2, 441:])
    assert torch.equal(z[:, 100:70000], y[:2, 260:70160])
    # a band-limited tone passes with unit gain (filter rows sum to 1)
    # (phases are formed in float64: 2 pi 1000 t reaches 3e4 rad, beyond float32 resolution)
    t = torch.arange(L, device=DEV, dtype=torch.float64) / 44100.0
    tone = torch.sin(2 * math.pi * 1000.0 * t).float()[None]
    out = r(tone)[0, 1000:-1000]
    t2 = torch.arange(80000, device=DEV, dtype=torch.float64)[1000:-1000] / 16000.0
    assert torch.allclose(out, torch.sin(2 * math.pi * 1000.0 * t2).float(), atol=2e-3)
    exp = O.resample(x[:2].cpu().numpy(), 44100, 16000, resampling_method="sinc_interp_kaiser")
    assert np.abs(host(y[:2]) - exp).max() <= 1e-4 * np.abs(exp).max()


def test_config4_mfcc_shard_consistency():
    """MFCC n_mfcc=40 (BASELINE config 4) on one shard of 256 x 160000: a 2-D batch shares one
    top_db cut-off; splitting the batch and supplying the global maximum reproduces it."""
    g = torch.Generator(device=DEV).manual_seed(99)
    x = torch.randn(64, 160000, device=DEV, generator=g)
    x[3] *= 1e-4  # a quiet utterance that the batch-global clamp will floor
    mf = T.MFCC(16000, n_mfcc=40, melkwargs=dict(n_fft=1024, hop_length=256, n_mels=80)).to(DEV)
    y = mf(x)
    assert tuple(y.shape) == (64, 40, 626) and torch.isfinite(y).all()
    y3 = mf(x[:, None, :])[:, 0]
    assert not torch.allclose(y[3], y3[3])  # per-item clamp differs for the quiet row
    assert torch.allclose(y[0], y3[0], atol=1e-3)
    exp = O.mfcc(x[:5].cpu().numpy()[:, None], 16000, 40, "ortho", False, dict(n_fft=1024, hop_length=256, n_mels=80),
                 fb=mf.MelSpectrogram.mel_scale.fb.cpu().numpy(), dct=mf.dct_mat.cpu().numpy())
    assert_close(host(y3[:5]), exp[:, 0], rtol=1e-4, atol=5e-3)


@pytest.mark.parametrize("n_fft", [256, 512, 2048])
def test_config5_sweep_sizes(n_fft):
    """Sweep sizes of BASELINE config 5 (hop = n_fft/4, n_mels=80, L=160000) at batch 64: shapes + oracle rows."""
    hop = n_fft // 4
    g = torch.Generator(device=DEV).manual_seed(n_fft)
    x = torch.randn(64, 160000, device=DEV, generator=g)
    import warnings

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = T.MelSpectrogram(16000, n_fft=n_fft, hop_length=hop, n_mels=80).to(DEV)
    y = m(x)
    assert tuple(y.shape) == (64, 80, 1 + 160000 // hop)
    exp = O.mel_spectrogram(x[:2].cpu().numpy(), sample_rate=16000, n_fft=n_fft, hop_length=hop, n_mels=80,
                            fb=m.mel_scale.fb.cpu().numpy())
    scaled_tol_close(host(y[:2]), exp, what=f"sweep n_fft={n_fft}")
