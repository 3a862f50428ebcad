"""LFCC and SpectralCentroid (SURVEY.md 8f.2): the MFCC kernels with a linear filterbank, and the
fused kernel with a weighted-sum epilogue.  CPU: oracle vs the reference's librosa goldens
(transforms/librosa_compatibility_test_impl.py:136-158) and the reference's own outputs; GPU: product
vs the same fixtures."""
import numpy as np
import pytest
import torch
from conftest import assert_close
from golden_cases import LIBROSA_FRAMES

from oracle import frontend_oracle as O

CENTROID = [dict(n_fft=400, hop_length=200), dict(n_fft=600, hop_length=100), dict(n_fft=200, hop_length=50)]


@pytest.mark.parametrize("i", range(3))
def test_oracle_spectral_centroid_librosa(librosa_transforms, i):
    c = CENTROID[i]
    got = O.spectral_centroid(librosa_transforms["whitenoise"], 16000, 0, O.hann_window(c["n_fft"]), c["n_fft"],
                              c["hop_length"], c["n_fft"])
    assert_close(got[..., LIBROSA_FRAMES], librosa_transforms[f"spectral_centroid_{i}"], rtol=1e-5, atol=5e-4)


def test_oracle_lfcc_and_centroid_reference(ref_cases):
    x = ref_cases["mel_in"]
    assert_close(O.linear_fbanks(257, 0.0, 8000.0, 64, 16000), ref_cases["lfcc_filter_mat"], rtol=1e-5, atol=1e-5)
    tol = dict(rtol=1e-4, atol=3e-3)
    assert_close(O.lfcc(x, 16000, 64, n_lfcc=20, speckwargs=dict(n_fft=512, hop_length=128)), ref_cases["lfcc_512_out"], **tol)
    assert_close(O.lfcc(x[:, None]), ref_cases["lfcc_default_out"], **tol)
    got = O.lfcc(x, 16000, 40, n_lfcc=13, log_lf=True, speckwargs=dict(n_fft=1024, hop_length=256))
    assert_close(got, ref_cases["lfcc_log_out"], rtol=1e-4, atol=1e-3)
    got = O.spectral_centroid(x, 16000, 0, O.hann_window(1024), 1024, 256, 1024)
    assert_close(got, ref_cases["centroid_1024_out"], rtol=2e-5, atol=1e-2)  # Hz, values ~4000
    got = O.spectral_centroid(x, 16000, 0, O.hann_window(400), 400, 200, 400)
    assert_close(got, ref_cases["centroid_default_out"], rtol=2e-5, atol=1e-2)


def test_module_surface_cpu():
    import audio_b200.transforms as T

    lf = T.LFCC()
    assert set(lf.state_dict()) == {"Spectrogram.window", "filter_mat", "dct_mat"}
    assert (lf.n_filter, lf.n_lfcc, lf.top_db, lf.log_lf, lf.f_max) == (128, 40, 80.0, False, 8000.0)
    with pytest.raises(ValueError, match="DCT type not supported"):
        T.LFCC(dct_type=1)
    with pytest.raises(ValueError, match="Cannot select more LFCC"):
        T.LFCC(n_lfcc=500)
    sc = T.SpectralCentroid(16000)
    assert (sc.n_fft, sc.win_length, sc.hop_length, sc.pad) == (400, 400, 200, 0)
    with pytest.raises(RuntimeError, match="no CPU or ATen fallback"):
        sc(torch.randn(1, 4000))


def test_filter_mat_bit_identical(ref_cases):
    import audio_b200.transforms as T

    lf = T.LFCC(16000, n_filter=64, n_lfcc=20, speckwargs=dict(n_fft=512, hop_length=128))
    assert np.array_equal(lf.filter_mat.numpy(), ref_cases["lfcc_filter_mat"])


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(3))
def test_gpu_spectral_centroid_librosa(librosa_transforms, i):
    import audio_b200.transforms as T

    x = torch.from_numpy(librosa_transforms["whitenoise"]).cuda()
    got = T.SpectralCentroid(sample_rate=16000, **CENTROID[i]).cuda()(x)
    assert tuple(got[..., LIBROSA_FRAMES].shape) == librosa_transforms[f"spectral_centroid_{i}"].shape
    # the reference asserts atol=5e-4 in float64; in float32 sums of ~200 magnitudes carry ~1e-3 Hz
    assert_close(got[..., LIBROSA_FRAMES].cpu().numpy(), librosa_transforms[f"spectral_centroid_{i}"], rtol=2e-6, atol=5e-3)


@pytest.mark.gpu
def test_gpu_lfcc_and_centroid_reference(ref_cases):
    import audio_b200.transforms as T

    x = torch.from_numpy(ref_cases["mel_in"]).cuda()
    tol = dict(rtol=1e-4, atol=5e-3)
    lf = T.LFCC(16000, n_filter=64, n_lfcc=20, speckwargs=dict(n_fft=512, hop_length=128)).cuda()
    assert_close(lf(x).cpu().numpy(), ref_cases["lfcc_512_out"], **tol)
    assert_close(T.LFCC().cuda()(x[:, None]).cpu().numpy(), ref_cases["lfcc_default_out"], **tol)
    lfl = T.LFCC(16000, n_filter=40, n_lfcc=13, log_lf=True, speckwargs=dict(n_fft=1024, hop_length=256)).cuda()
    assert_close(lfl(x).cpu().numpy(), ref_cases["lfcc_log_out"], rtol=1e-4, atol=2e-3)
    got = T.SpectralCentroid(16000, n_fft=1024, hop_length=256).cuda()(x)
    assert_close(got.cpu().numpy(), ref_cases["centroid_1024_out"], rtol=2e-5, atol=2e-2)
    got = T.SpectralCentroid(16000).cuda()(x.reshape(2, 2, -1))
    assert tuple(got.shape) == (2, 2, 11)
    assert_close(got.reshape(4, 11).cpu().numpy(), ref_cases["centroid_default_out"], rtol=2e-5, atol=2e-2)


def test_speed_surface_cpu():
    import audio_b200.transforms as T

    sp = T.Speed(16000, 1.1)
    assert (sp.source_sample_rate, sp.target_sample_rate) == (11, 10)
    assert (sp.resampler.orig_freq, sp.resampler.new_freq) == (11, 10)
    assert (T.Speed(44100, 0.9).source_sample_rate, T.Speed(44100, 0.9).target_sample_rate) == (9, 10)
    pert = T.SpeedPerturbation(16000, [0.9, 1.1, 1.0])
    assert len(pert.speeders) == 3


@pytest.mark.gpu
def test_gpu_speed_matches_oracle_resample():
    import audio_b200.functional as F
    import audio_b200.transforms as T

    x = torch.randn(3, 8000, generator=torch.Generator().manual_seed(3))
    lengths = torch.tensor([8000, 4001, 17])
    for factor, (src, dst) in ((1.1, (11, 10)), (0.9, (9, 10))):
        y, out_len = T.Speed(16000, factor).cuda()(x.cuda(), lengths.cuda())
        exp = O.resample(x.numpy(), src, dst)
        assert tuple(y.shape) == exp.shape
        assert np.abs(y.cpu().numpy() - exp).max() <= 1e-4 * np.abs(exp).max()
        assert out_len.cpu().tolist() == [int(np.ceil(n * dst / src)) for n in lengths.tolist()]
        y2, none = F.speed(x.cuda(), 16000, factor)
        assert none is None and np.abs(y2.cpu().numpy() - exp).max() <= 1e-4 * np.abs(exp).max()
    torch.manual_seed(0)
    pert = T.SpeedPerturbation(16000, [0.9, 1.1, 1.0]).cuda()
    y, _ = pert(x.cuda())
    assert y.shape[-1] in (8889, 7273, 8000)
