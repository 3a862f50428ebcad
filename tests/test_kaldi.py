"""Kaldi-compatible features (SURVEY.md 8f.1): compliance.kaldi.{spectrogram, fbank, mfcc}.

CPU: the oracle against (a) the 311 outputs of the Kaldi binaries the reference's own tests hold
(compliance/kaldi/kaldi_compatibility_impl.py:20-48, same rtol / atol) and (b) the reference itself on realistic
signals; the host-side tables bit-identical to the reference's.  GPU: the product (one fused kernel through the C ABI)
against the same fixtures."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import kaldi_oracle as KO

KINDS = ("fbank", "mfcc", "spectrogram")
# tolerances of the reference's own Kaldi tests (kaldi_compatibility_impl.py:29,39,48)
REF_TOL = {"fbank": dict(rtol=1e-4, atol=1e-8), "spectrogram": dict(rtol=1e-4, atol=1e-6), "mfcc": dict(rtol=1e-4, atol=1e-5)}


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def kaldi_goldens():
    return np.load(os.path.join(GOLDEN, "kaldi_goldens.npz"))


@pytest.fixture(scope="module")
def kaldi_ref():
    return np.load(os.path.join(GOLDEN, "kaldi_ref_cases.npz"))


def _cases(fixture, kind):
    return [(i, json.loads(str(a))) for i, a in enumerate(fixture[f"{kind}_args"])]


# ---- CPU: the oracle is pinned -----------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_oracle_matches_kaldi_binaries(kaldi_goldens, kind):
    wave = kaldi_goldens["wave"]
    assert wave.shape == (1, 20)
    for i, kw in _cases(kaldi_goldens, kind):
        exp = kaldi_goldens[f"{kind}_{i}"]
        got = getattr(KO, kind)(wave, **kw)
        assert got.shape == exp.shape, (kind, i, kw)
        np.testing.assert_allclose(got, exp, err_msg=f"{kind} case {i}: {kw}", **REF_TOL[kind])


@pytest.mark.parametrize("kind", KINDS)
def test_oracle_matches_reference_on_long_signals(kaldi_ref, kind):
    wave = kaldi_ref["wave"][:1]
    for i, kw in _cases(kaldi_ref, kind):
        exp = kaldi_ref[f"{kind}_{i}"].astype(np.float64)
        got = getattr(KO, kind)(wave, **kw)
        assert got.shape == exp.shape
        # the reference ran in float32: log-domain values agree to ~1e-5 of the column range
        assert np.abs(got - exp).max() <= 2e-5 * np.abs(exp).max() + 1e-4, (kind, i, np.abs(got - exp).max())
    got = KO.fbank(kaldi_ref["wave"], channel=1, num_mel_bins=23)
    assert np.abs(got - kaldi_ref["fbank_channel1"]).max() <= 1e-3


def test_oracle_frame_counts():
    for n, size, shift in ((20, 17, 11), (400, 400, 160), (16000, 400, 160), (19999, 320, 128), (33, 32, 1)):
        assert KO.num_frames(n, size, shift, True) == 1 + (n - size) // shift
        assert KO.num_frames(n, size, shift, False) == (n + shift // 2) // shift
        assert KO.get_strided(np.arange(n, dtype=float), size, shift, False).shape == (KO.num_frames(n, size, shift, False), size)
    x = np.arange(10.0)
    fr = KO.get_strided(x, 4, 2, False)  # pad = 2 - 1 = 1: one mirrored sample in front
    assert fr[0].tolist() == [0.0, 0.0, 1.0, 2.0] and fr[-1].tolist() == [7.0, 8.0, 9.0, 9.0]


# ---- CPU: host side of the product ---------------------------------------------------------------------------------
def test_tables_bit_identical_to_reference(kaldi_ref):
    import audio_b200.compliance.kaldi as K

    b, c = K.get_mel_banks(23, 512, 16000.0, 20.0, 0.0, 100.0, -500.0, 1.0)
    assert np.array_equal(b.numpy(), kaldi_ref["banks_23_512"]) and np.array_equal(c.numpy(), kaldi_ref["centers_23_512"])
    b, c = K.get_mel_banks(30, 256, 8000.0, 60.0, -200.0, 200.0, -600.0, 1.1)
    assert np.array_equal(b.numpy(), kaldi_ref["banks_vtln"]) and np.array_equal(c.numpy(), kaldi_ref["centers_vtln"])
    assert np.array_equal(K._get_dct_matrix(13, 23).numpy(), kaldi_ref["dct_13_23"])
    assert np.array_equal(K._get_lifter_coeffs(13, 22.0).numpy(), kaldi_ref["lifter_13"])
    for wt in K.WINDOWS:
        w = K._feature_window_function(wt, 400, 0.42, torch.device("cpu"), torch.float32)
        assert np.array_equal(w.numpy(), kaldi_ref[f"window_{wt}"]), wt
    assert K.mel_scale_scalar(1000.0) == pytest.approx(1127.0 * np.log(1.0 + 1000.0 / 700.0))
    assert K.inverse_mel_scale_scalar(K.mel_scale_scalar(440.0)) == pytest.approx(440.0)


def test_module_surface_and_errors_cpu():
    import inspect

    import audio_b200.compliance.kaldi as K

    assert list(inspect.signature(K.fbank).parameters)[:4] == ["waveform", "blackman_coeff", "channel", "dither"]
    assert inspect.signature(K.fbank).parameters["num_mel_bins"].default == 23
    assert inspect.signature(K.mfcc).parameters["num_ceps"].default == 13
    assert inspect.signature(K.spectrogram).parameters["window_type"].default == "povey"
    with pytest.raises(RuntimeError, match="no CPU or ATen fallback"):
        K.fbank(torch.zeros(1, 16000))
    with pytest.raises(AssertionError, match="Must have at least 3 mel bins"):
        K.get_mel_banks(3, 512, 16000.0, 20.0, 0.0, 100.0, -500.0, 1.0)
    with pytest.raises(AssertionError, match="Bad values in options"):
        K.get_mel_banks(23, 512, 16000.0, 9000.0, 0.0, 100.0, -500.0, 1.0)


def test_c_abi_bookkeeping_cpu():
    from audio_b200 import _lib

    lib = _lib.lib()
    for n, size, shift in ((20, 17, 11), (400, 400, 160), (16000, 400, 160), (19999, 320, 128), (399, 400, 160)):
        for snip in (0, 1):
            assert lib.b200a_kaldi_num_frames(n, size, shift, snip) == KO.num_frames(n, size, shift, bool(snip))
    assert lib.b200a_kaldi_num_frames(-1, 400, 160, 1) == -1


# ---- GPU -----------------------------------------------------------------------------------------------------------
def _close(got, exp, rtol, atol, what):
    err = np.abs(got - exp) - (atol + rtol * np.abs(exp))
    assert got.shape == exp.shape, what
    assert err.max() <= 0, f"{what}: max excess {err.max():.3e} at {np.unravel_index(err.argmax(), err.shape)}"


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_gpu_matches_kaldi_binaries(kaldi_goldens, kind):
    """The reference's own Kaldi cases: 20 int16 samples, 1 ms frames, every option.  float32 on the GPU is held to the
    reference's rtol with a log-domain atol of 2e-5 (values are logs of O(1e6) energies; the reference's float32 run
    has the same spread against the Kaldi binaries)."""
    import audio_b200.compliance.kaldi as K

    wave = torch.from_numpy(kaldi_goldens["wave"]).cuda()
    for i, kw in _cases(kaldi_goldens, kind):
        exp = kaldi_goldens[f"{kind}_{i}"]
        got = getattr(K, kind)(wave, **kw).cpu().numpy()
        _close(got, exp, 1e-4, 2e-5 if (kind != "fbank" or kw.get("use_log_fbank", True)) else 1e-8, f"{kind} case {i}: {kw}")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_gpu_matches_reference_on_long_signals(kaldi_ref, kind):
    import audio_b200.compliance.kaldi as K

    wave = torch.from_numpy(kaldi_ref["wave"]).cuda()
    for i, kw in _cases(kaldi_ref, kind):
        exp = kaldi_ref[f"{kind}_{i}"]
        got = getattr(K, kind)(wave[:1], **kw)
        assert tuple(got.shape) == exp.shape and got.is_contiguous()
        oracle = getattr(KO, kind)(kaldi_ref["wave"][:1], **kw)
        scale = np.abs(oracle).max()
        assert np.abs(got.cpu().numpy() - oracle).max() <= 2e-5 * scale + 1e-4, (kind, i)
        assert np.abs(got.cpu().numpy() - exp).max() <= 4e-5 * scale + 2e-4, (kind, i)
    got = K.fbank(wave, channel=1, num_mel_bins=23).cpu().numpy()
    assert np.abs(got - kaldi_ref["fbank_channel1"]).max() <= 1e-3


@pytest.mark.gpu
def test_gpu_batch_extension_and_edges(kaldi_ref):
    import audio_b200.compliance.kaldi as K

    x = torch.from_numpy(kaldi_ref["wave"]).cuda()
    batch = torch.stack([x[0], x[1], x[0].flip(0)])
    got = K.fbank_batch(batch, num_mel_bins=40, snip_edges=False, use_energy=True)
    assert tuple(got.shape) == (3, 125, 41)
    for r in range(3):
        one = K.fbank(batch[r:r + 1], num_mel_bins=40, snip_edges=False, use_energy=True)
        assert torch.equal(got[r], one)
    m = K.mfcc_batch(batch, num_ceps=13, subtract_mean=True)
    assert tuple(m.shape) == (3, 123, 13)
    assert m.mean(1).abs().max() < 1e-3
    assert K.fbank(x[:1], min_duration=10.0).numel() == 0
    with pytest.raises(RuntimeError, match="dither"):
        K.fbank(x[:1], dither=1.0)
    with pytest.raises(AssertionError, match="choose a window size"):
        K.fbank(x[:1, :300])
    with pytest.raises(AssertionError, match="Invalid channel"):
        K.fbank(x, channel=2)


@pytest.mark.gpu
@pytest.mark.parametrize("sr,pow2", [pytest.param(22050.0, True, id="22050.0"), pytest.param(44100.0, True, id="44100.0"),
                                     pytest.param(11025.0, True, id="11025.0"),
                                     pytest.param(44100.0, False, id="44100.0-unrounded"),
                                     pytest.param(16000.0, False, id="16000.0-unrounded")])
@pytest.mark.parametrize("snip", [True, False])
def test_gpu_other_sample_rates_against_oracle(kaldi_ref, sr, pow2, snip):
    """Frame sizes that are not multiples of 4 samples (551 / 1102 / 275 at 25 ms) and shifts such as 220: the
    register path stages every unit through the gather (no 16-byte aligned bulk copy), 2048-point frames take the
    generic kernel.  round_to_power_of_two=False: the frame length itself is the FFT size (1102 = 2 * 19 * 29, 400),
    on the generic kernel."""
    import audio_b200.compliance.kaldi as K

    x = kaldi_ref["wave"][:1, :15000]
    kw = dict(sample_frequency=sr, num_mel_bins=40, snip_edges=snip, use_energy=True, low_freq=40.0,
              round_to_power_of_two=pow2)
    got = K.fbank(torch.from_numpy(x).cuda(), **kw).cpu().numpy()
    exp = KO.fbank(x, **kw)
    assert got.shape == exp.shape
    assert np.abs(got - exp).max() <= 2e-5 * np.abs(exp).max() + 1e-4
    kw = dict(sample_frequency=sr, snip_edges=snip, num_mel_bins=30, num_ceps=12, round_to_power_of_two=pow2)
    got = K.mfcc(torch.from_numpy(x).cuda(), **kw).cpu().numpy()
    exp = KO.mfcc(x, **kw)
    assert got.shape == exp.shape and np.abs(got - exp).max() <= 2e-5 * np.abs(exp).max() + 2e-4
