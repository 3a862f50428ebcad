"""Branch coverage of the register-FFT kernels (n_fft 256/512/1024/2048) and the tensor-pipe
resampler against the CPU oracle: staged (bulk copy) / plain-load / padding-gather input paths, aligned
and unaligned hops, one..few frames, odd frame counts, ragged batches, every output stage."""
import math
import warnings

import numpy as np
import pytest
import torch
from conftest import assert_close, scaled_tol_close

import audio_b200.functional as F
import audio_b200.transforms as T
from oracle import frontend_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def randn(rows, length, seed):
    return torch.randn(rows, length, generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("n_fft", [256, 512, 1024, 2048])
@pytest.mark.parametrize("hop_kind", ["quarter", "half", "odd", "tiny"])
def test_mel_hops_and_lengths(n_fft, hop_kind):
    hop = {"quarter": n_fft // 4, "half": n_fft // 2, "odd": n_fft // 4 + 3, "tiny": 20}[hop_kind]
    # lengths chosen to give 1, 2, 3 frames, an odd count, and a long ragged utterance
    base = n_fft // 2 + 1  # shortest signal reflect padding accepts
    for length in (base, base + hop, base + 2 * hop + 5, base + 7 * hop + 11, base + 40 * hop + 123):
        x = randn(3, length, n_fft + length)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            m = T.MelSpectrogram(16000, n_fft=n_fft, hop_length=hop, n_mels=40).to(DEV)
        got = m(x.to(DEV)).cpu().numpy()
        exp = O.mel_spectrogram(x.numpy(), sample_rate=16000, n_fft=n_fft, hop_length=hop, n_mels=40,
                                fb=m.mel_scale.fb.cpu().numpy())
        assert got.shape == exp.shape == (3, 40, 1 + length // hop)
        scaled_tol_close(got, exp, what=f"n_fft={n_fft} hop={hop} L={length}")


@pytest.mark.parametrize("n_fft", [256, 512, 1024, 2048])
def test_spectrogram_stage_options(n_fft):
    x = randn(2, 9 * n_fft + 17, n_fft)
    xd = x.to(DEV)
    for kw in (dict(power=1.0), dict(power=3.0), dict(win_length=n_fft - 56, hop_length=n_fft // 4),
               dict(center=False, hop_length=n_fft // 2), dict(pad=24, hop_length=n_fft // 4),
               dict(pad=13, hop_length=n_fft // 4), dict(pad_mode="constant"), dict(normalized=True)):
        win = kw.get("win_length", n_fft)
        hop = kw.get("hop_length", win // 2)
        got = T.Spectrogram(n_fft=n_fft, **kw).to(DEV)(xd).cpu().numpy()
        exp = O.spectrogram(x.numpy(), kw.get("pad", 0), O.hann_window(win), n_fft, hop, win, kw.get("power", 2.0),
                            kw.get("normalized", False), kw.get("center", True), kw.get("pad_mode", "reflect"))
        scaled_tol_close(got, exp, what=f"n_fft={n_fft} {kw}")


@pytest.mark.parametrize("n_fft", [256, 512, 1024, 2048])
def test_strided_and_offset_inputs(n_fft):
    """Row pitch > length and a base pointer that is not 16-byte aligned (bulk staging must stand down)."""
    big = randn(4, 6 * n_fft + 64, 3).to(DEV)
    view = big[:, 3 : 3 + 5 * n_fft + 1]  # offset 3 floats, pitch > length
    m = T.MelSpectrogram(16000, n_fft=n_fft, hop_length=n_fft // 4, n_mels=32).to(DEV)
    got = m(view).cpu().numpy()
    exp = O.mel_spectrogram(view.cpu().numpy(), sample_rate=16000, n_fft=n_fft, hop_length=n_fft // 4, n_mels=32,
                            fb=m.mel_scale.fb.cpu().numpy())
    scaled_tol_close(got, exp)
    assert np.array_equal(m(view.contiguous()).cpu().numpy(), got)  # same bits whichever input path ran


@pytest.mark.parametrize("n_fft,n_mels,n_mfcc", [(256, 40, 13), (512, 64, 20), (1024, 80, 40), (2048, 128, 40), (1024, 23, 23)])
def test_mfcc_all_sizes(n_fft, n_mels, n_mfcc):
    x = randn(5, 12 * n_fft, n_fft + n_mels)
    x[1] *= 1e-3
    kw = dict(n_fft=n_fft, hop_length=n_fft // 4, n_mels=n_mels)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        mf = T.MFCC(16000, n_mfcc=n_mfcc, melkwargs=kw).to(DEV)
    fb, dct = mf.MelSpectrogram.mel_scale.fb.cpu().numpy(), mf.dct_mat.cpu().numpy()
    got = mf(x.to(DEV)).cpu().numpy()
    exp = O.mfcc(x.numpy(), 16000, n_mfcc, "ortho", False, kw, fb=fb, dct=dct)
    assert_close(got, exp, rtol=1e-4, atol=5e-3, what="2-D (batch-global clamp)")
    got = mf(x[:, None].to(DEV)).cpu().numpy()
    exp = O.mfcc(x[:, None].numpy(), 16000, n_mfcc, "ortho", False, kw, fb=fb, dct=dct)
    assert_close(got, exp, rtol=1e-4, atol=5e-3, what="3-D (per-item clamp)")


def test_many_filters_take_the_generic_path():
    """> 512 mel filters exceed the contraction plan: the call must still be right (generic kernel)."""
    x = randn(2, 6000, 1)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = T.MelSpectrogram(16000, n_fft=1024, hop_length=256, n_mels=520).to(DEV)
    got = m(x.to(DEV)).cpu().numpy()
    exp = O.mel_spectrogram(x.numpy(), sample_rate=16000, n_fft=1024, hop_length=256, n_mels=520,
                            fb=m.mel_scale.fb.cpu().numpy())
    scaled_tol_close(got, exp)


def test_dense_filterbank_matrix():
    """A filterbank without band structure (every bin feeds every filter): fragments no longer fit in
    shared memory and are streamed from global memory, at every register-FFT size."""
    x = randn(3, 9000, 2)
    for n_fft in (256, 512, 1024, 2048):
        m = T.MelSpectrogram(16000, n_fft=n_fft, hop_length=n_fft // 4, n_mels=48).to(DEV)
        fb = torch.rand(n_fft // 2 + 1, 48, generator=torch.Generator().manual_seed(9))
        m.mel_scale.fb.copy_(fb.to(DEV))
        got = m(x.to(DEV)).cpu().numpy()
        exp = O.mel_spectrogram(x.numpy(), sample_rate=16000, n_fft=n_fft, hop_length=n_fft // 4, n_mels=48,
                                fb=fb.numpy())
        scaled_tol_close(got, exp, what=f"n_fft={n_fft}")


@pytest.mark.parametrize("orig,new", [(44100, 16000), (16000, 44100), (48000, 44100), (16000, 8000), (8000, 16000),
                                      (22050, 16000), (3, 2), (7, 5), (160, 161)])
@pytest.mark.parametrize("length", [1, 33, 1000, 12345])
def test_resample_ratios_and_lengths(orig, new, length):
    x = randn(3, length, orig + new + length)
    r = T.Resample(orig, new).to(DEV)
    got = r(x.to(DEV)).cpu().numpy()
    exp = O.resample(x.numpy(), orig, new)
    assert got.shape == exp.shape
    assert np.abs(got - exp).max() <= 1e-4 * max(np.abs(exp).max(), 1e-3)


def test_resample_unaligned_views():
    big = randn(5, 30011, 4).to(DEV)
    r = T.Resample(44100, 16000, resampling_method="sinc_interp_kaiser").to(DEV)
    for off in (0, 1, 2, 3, 5):
        view = big[:, off : off + 29000]
        got = r(view)
        ref = r(view.contiguous())
        assert torch.equal(got, ref), off  # any alignment takes the same arithmetic path
        exp = O.resample(view.cpu().numpy(), 44100, 16000, resampling_method="sinc_interp_kaiser")
        assert np.abs(got.cpu().numpy() - exp).max() <= 1e-4 * np.abs(exp).max()


def test_resample_large_prime_ratio_uses_fallback():
    x = randn(2, 5000, 8)
    # new' = 1999 > 1024 phases: the one-output-per-thread kernel.  (The transform builds its taps in
    # float64 like the reference; F.resample builds them in float32 on the device, also like the reference,
    # which at this ratio is itself only good to ~1e-3 -- so the oracle comparison uses the transform.)
    got = T.Resample(2003, 1999).to(DEV)(x.to(DEV)).cpu().numpy()
    exp = O.resample(x.numpy(), 2003, 1999)
    assert got.shape == exp.shape
    assert np.abs(got - exp).max() <= 1e-4 * np.abs(exp).max()
    fun = F.resample(x.to(DEV), 2003, 1999).cpu().numpy()
    assert fun.shape == exp.shape and np.abs(fun - exp).max() <= 5e-3 * np.abs(exp).max()


def test_mma_sync_contraction_against_oracle():
    """The fused mel stage contracts each power tile with the filterbank on mma.sync (TF32 hi/lo operands): every
    register-FFT size, narrow and wide filterbanks, against the fp64 oracle."""
    for n_fft, n_mels in ((256, 40), (512, 64), (1024, 80), (1024, 128)):
        x = torch.randn(5, 9000, generator=torch.Generator().manual_seed(n_fft + n_mels))
        got = T.MelSpectrogram(16000, n_fft=n_fft, hop_length=n_fft // 4, n_mels=n_mels).to(DEV)(x.to(DEV)).cpu().numpy()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            exp = O.mel_spectrogram(x.numpy(), sample_rate=16000, n_fft=n_fft, hop_length=n_fft // 4, n_mels=n_mels)
        scaled_tol_close(got, exp, what=f"mma {n_fft}/{n_mels}")
