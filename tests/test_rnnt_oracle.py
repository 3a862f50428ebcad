"""The RNN-T feature chain without a GPU: the float64 oracle against the reference's float32 fixture, the fixture's
coverage of the three pieces and of silence, the chain's VJP against float64 torch.autograd through the reference's
own ``_piecewise_linear_log`` / ``_GlobalStatsNormalization`` (or, where torchaudio does not import, a torch
restatement of them), the extractor's state_dict against a reference extractor built locally, and the ABI validation of
the two new entry points."""
import ctypes
import json
import math
import os
import types

import numpy as np
import pytest
import torch

from oracle import frontend_oracle as O

import rnnt_grad_oracle as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LENGTHS = (201, 3200, 16000, 37920)

try:
    import torchaudio
    import torchaudio.pipelines.rnnt_pipeline as RP
except Exception:  # noqa: BLE001 -- any import failure means "use the restatement"
    torchaudio = RP = None


@pytest.fixture(scope="module")
def fx():
    with np.load(os.path.join(GOLDEN, "rnnt_ref_cases.npz")) as z:
        return {k: z[k] for k in z.files}


def _stats(fx, name="librispeech"):
    return fx[f"stats_{name}_mean"], fx[f"stats_{name}_invstddev"]


def _input(fx, n, i):
    return fx[f"base_{n}"] * fx["levels"][i]  # float32 product, as the fixture's inputs


def _mel64(x):
    return np.swapaxes(O.mel_spectrogram(np.asarray(x, np.float64), **R.MEL_ARGS), -1, -2)


def _piecewise_linear_log(x):
    """rnnt_pipeline.py:20-23 (used where torchaudio does not import)."""
    x[x > math.e] = torch.log(x[x > math.e])
    x[x <= math.e] = x[x <= math.e] / math.e
    return x


def _ref_chain(m, mean, invstd):
    """The reference's ``x * _gain`` -> ``_piecewise_linear_log`` -> ``(x - mean) * invstddev`` as torch ops."""
    if RP is not None:
        return (RP._piecewise_linear_log(m * RP._gain) - mean) * invstd
    return (_piecewise_linear_log(m * R.GAIN) - mean) * invstd


# ---- the oracle against the reference's float32 run -------------------------------------------------------------------
def _check_features(got, exp, mel):
    """The forward bar 1e-4 |e| + 1e-4 rms(e), on the elements whose float32 and float64 decisions agree; the others
    are counted and must be under 0.1 %."""
    flip = np.zeros(exp.shape, bool)
    flip[: mel.shape[0]] = R.pieces32(mel) != R.pieces64(mel)
    assert flip.mean() < 1e-3, f"{flip.sum()} of {flip.size} elements lie on a breakpoint"
    rms = float(np.sqrt(np.mean(exp.astype(np.float64) ** 2)))
    err = np.abs(got - exp)
    bad = (err > 1e-4 * np.abs(exp) + 1e-4 * rms) & ~flip
    assert not bad.any(), f"{bad.sum()} elements out of tolerance, worst {err[bad].max():.3e}"


@pytest.mark.parametrize("n", LENGTHS)
@pytest.mark.parametrize("i", range(3))
def test_oracle_matches_reference_extractors(fx, n, i):
    mean, invstd = _stats(fx)
    x = _input(fx, n, i)
    mel = _mel64(x)
    full = R.features(x, mean, invstd, None, right_padding=4)
    _check_features(full, fx[f"full_{n}_{i}"], mel)
    assert (fx[f"full_{n}_{i}"][-4:] == 0).all()  # literal zero rows after the normalisation
    _check_features(full[:-4], fx[f"stream_{n}_{i}"], mel)
    assert fx[f"full_{n}_{i}"].shape == (1 + n // 160 + 4, 80)


def test_oracle_matches_recipe_batch(fx):
    mean, invstd = _stats(fx, "tedlium3")
    base = fx["base_37920"]
    exp = fx["batch_feats"]
    t_max = exp.shape[1]
    for r, (n, lv) in enumerate(zip(fx["batch_lengths"], fx["batch_levels"])):
        mel = np.zeros((t_max, 80))
        m = _mel64(base[:n] * lv)
        assert m.shape[0] == fx["batch_frames"][r] == 1 + n // 160
        mel[: m.shape[0]] = m  # pad_sequence pads the mel values with zeros; they go through the chain
        _check_features(R.chain(mel, mean, invstd), exp[r], mel)


def test_fixture_hits_every_piece_and_silence(fx):
    mean, invstd = _stats(fx)
    counts = np.zeros(4, int)
    silent = 0
    for n in LENGTHS:
        for i in range(3):
            mel = _mel64(_input(fx, n, i))
            p = R.pieces64(mel)
            counts += np.bincount(p.ravel(), minlength=4)
            zero = (mel == 0).all(axis=1)
            silent += int(zero.sum())
            out = fx[f"stream_{n}_{i}"]
            # silence: y = 0, so the features are float32 (0 - mean) * invstddev exactly
            assert (out[zero] == (np.float32(0) - mean) * invstd).all()
    assert counts[0] == 0 and (counts[1:] > 100).all(), counts
    assert silent >= 10
    # the breakpoints in mel terms
    assert math.isclose(math.e / R.GAIN, 2.53e-9, rel_tol=1e-2) and math.isclose(math.e ** math.e / R.GAIN, 1.41e-8,
                                                                                  rel_tol=1e-2)


def test_three_pieces_of_the_reference():
    """The semantics the oracle keeps: 15 -> log(15)/e, 15.2 -> log(15.2), slope 1/(3e) at 3, jumps at e and e^e."""
    x = torch.tensor([0.5, 3.0, 15.0, 15.2], dtype=torch.float64, requires_grad=True)
    y = (RP._piecewise_linear_log if RP is not None else _piecewise_linear_log)(x * 1.0)
    assert torch.allclose(y.detach(), torch.tensor([0.5 / math.e, math.log(3) / math.e, math.log(15) / math.e,
                                                    math.log(15.2)], dtype=torch.float64))
    y[1].backward()
    assert math.isclose(float(x.grad[1]), 1 / (3 * math.e), rel_tol=1e-12)
    m = np.array([15.0, 15.2, 0.5]) / R.GAIN
    np.testing.assert_allclose(R.chain(m, 0.0, 1.0), [math.log(15) / math.e, math.log(15.2), 0.5 / math.e], rtol=1e-12)
    assert list(R.pieces32(np.array([0.0, 2.0e-9, 3.0e-9, 2.0e-8, np.nan], np.float32))) == [1, 1, 2, 3, 0]


# ---- the VJP against float64 autograd -------------------------------------------------------------------------------
def _away_from_breakpoints(m):
    x = m * R.GAIN
    return (np.abs(x / math.e - 1) > 1e-6) & (np.abs(x / math.e ** math.e - 1) > 1e-6)


def test_chain_vjp_matches_autograd(fx):
    mean, invstd = _stats(fx)
    rng = np.random.default_rng(11)
    m = 10.0 ** rng.uniform(-12, -2, size=(300, 80))
    m[:20] = 0.0  # silence
    m[m.shape[0] // 2, :] = math.e / R.GAIN * (1 + 1e-3)  # just past the first jump
    keep = _away_from_breakpoints(m)
    g = rng.standard_normal(m.shape)
    mt = torch.tensor(m, requires_grad=True)
    y = _ref_chain(mt, torch.tensor(mean, dtype=torch.float64), torch.tensor(invstd, dtype=torch.float64))
    (y * torch.tensor(g)).sum().backward()
    p = R.pieces64(m)
    assert set(np.unique(p[keep]).tolist()) == {1, 2, 3}
    np.testing.assert_allclose(R.chain(m, mean, invstd)[keep], y.detach().numpy()[keep], rtol=1e-10, atol=1e-10)
    got, exp = R.chain_vjp(m, g, invstd)[keep], mt.grad.numpy()[keep]
    assert np.abs(got - exp).max() <= 1e-10 * np.abs(exp).max()


def test_features_vjp_matches_autograd_through_the_mel_spectrogram(fx):
    """The whole extractor: float64 autograd through torch.stft + the mel matrix + the chain."""
    mean, invstd = _stats(fx)
    x = _input(fx, 3200, 1).astype(np.float64)
    fb = O.melscale_fbanks(201, 0.0, 8000.0, 80, 16000)
    xt = torch.tensor(x, requires_grad=True)
    spec = torch.stft(xt, 400, 160, window=torch.hann_window(400, dtype=torch.float64), center=True,
                      pad_mode="reflect", return_complex=True).abs().pow(2.0)
    mel = (spec.transpose(0, 1) @ torch.tensor(fb))  # (T, n_mels)
    y = _ref_chain(mel, torch.tensor(mean, dtype=torch.float64), torch.tensor(invstd, dtype=torch.float64))
    y = torch.nn.functional.pad(y, (0, 0, 0, 4))
    rng = np.random.default_rng(5)
    g = rng.standard_normal(tuple(y.shape))
    (y * torch.tensor(g)).sum().backward()
    m = mel.detach().numpy()
    assert _away_from_breakpoints(m).all()
    got = R.features_vjp(x, g, mean, invstd, fb, pieces=R.pieces64(m))
    exp = xt.grad.numpy()
    assert np.abs(got - exp).max() <= 1e-9 * np.abs(exp).max()


# ---- the module against a reference extractor built locally -----------------------------------------------------------
def _stats_file(tmp_path, fx):
    mean, invstd = _stats(fx)
    path = tmp_path / "global_stats.json"
    path.write_text(json.dumps({"mean": mean.tolist(), "invstddev": invstd.tolist()}))
    return str(path)


def test_state_dict_keys_and_load_from_reference(tmp_path, fx):
    if RP is None:
        pytest.skip("torchaudio does not import")
    from audio_b200.pipelines import RNNTFeatureExtractor

    path = _stats_file(tmp_path, fx)
    ref = RP._ModuleFeatureExtractor(torch.nn.Sequential(
        torchaudio.transforms.MelSpectrogram(sample_rate=16000, n_fft=400, n_mels=80, hop_length=160),
        RP._FunctionalModule(lambda x: x.transpose(1, 0)),
        RP._FunctionalModule(lambda x: RP._piecewise_linear_log(x * RP._gain)),
        RP._GlobalStatsNormalization(path),
        RP._FunctionalModule(lambda x: torch.nn.functional.pad(x, (0, 0, 0, 4))),
    ))
    ours = RNNTFeatureExtractor(path)
    assert list(ours.state_dict()) == list(ref.state_dict()) == [
        "pipeline.0.spectrogram.window", "pipeline.0.mel_scale.fb", "pipeline.3.mean", "pipeline.3.invstddev"]
    for k, v in ref.state_dict().items():
        assert torch.equal(ours.state_dict()[k], v), k
    sd = {k: v + 1.0 if k.endswith("mean") else v for k, v in ref.state_dict().items()}
    ours.load_state_dict(sd)
    assert torch.equal(ours.pipeline["3"].mean, sd["pipeline.3.mean"])


def test_from_bundle_reads_the_bundle_by_duck_typing(tmp_path, fx):
    from audio_b200.pipelines import RNNTFeatureExtractor

    path = _stats_file(tmp_path, fx)
    b = types.SimpleNamespace(sample_rate=8000, n_fft=256, n_mels=40, hop_length=80, _right_padding=3)
    e = RNNTFeatureExtractor.from_bundle(b, path)
    mel = e.pipeline["0"]
    assert (mel.sample_rate, mel.n_fft, mel.n_mels, mel.hop_length, e.right_padding) == (8000, 256, 40, 80, 3)
    assert RNNTFeatureExtractor.from_bundle(b, path, streaming=True).right_padding == 0
    if RP is not None:
        bundle = torchaudio.pipelines.EMFORMER_RNNT_BASE_LIBRISPEECH
        e = RNNTFeatureExtractor.from_bundle(bundle, path)
        mel = e.pipeline["0"]
        assert (mel.sample_rate, mel.n_fft, mel.n_mels, mel.hop_length, e.right_padding) == (16000, 400, 80, 160, 4)


def test_extractor_rejects_bad_arguments(tmp_path, fx):
    from audio_b200.pipelines import RNNTFeatureExtractor

    path = _stats_file(tmp_path, fx)
    with pytest.raises(ValueError):
        RNNTFeatureExtractor(path, right_padding=-1)
    e = RNNTFeatureExtractor(path)
    with pytest.raises(ValueError, match="1-D"):
        e(torch.zeros(2, 4000))
    with pytest.raises(ValueError, match="batch, time"):
        e.forward_batch(torch.zeros(4000))
    with pytest.raises(RuntimeError, match="CUDA device"):  # no CPU fallback
        e(torch.zeros(4000))


# ---- ABI validation ---------------------------------------------------------------------------------------------------
def _lib_or_skip():
    from audio_b200 import _lib

    try:
        return _lib, _lib.lib()
    except ImportError:
        pytest.skip("libb200audio.so is not built")


def test_rnnt_features_run_validation():
    L, lib = _lib_or_skip()
    from audio_b200._plans import FrontendPlan

    fake = ctypes.c_void_p(0x1000)

    def call(d=None, rows=2, length=16000, row_stride=16000, lengths=None, gain=1073676288.0, out_frames=101,
             ptrs=(True,) * 4, mel=None):
        if d is None:
            d = FrontendPlan.make_desc(400, 400, 160, 0, True, "reflect", True, False, False, 2.0, 80)
        p = [fake if ok else None for ok in ptrs]
        return lib.b200a_rnnt_features_run(d, p[0], p[1], rows, length, row_stride, lengths, p[2], gain, out_frames,
                                           p[3], mel, None)

    assert call(d=FrontendPlan.make_desc(400, 400, 160, 0, True, "reflect", True, False, False, 2.0, 0)) == L.EINVAL
    assert call(d=FrontendPlan.make_desc(400, 400, 160, 0, True, "reflect", True, False, False, -1.0, 80)) == L.EINVAL
    assert call(d=FrontendPlan.make_desc(400, 500, 160, 0, True, "reflect", True, False, False, 2.0, 80)) == L.EINVAL
    assert call(rows=-1) == L.EINVAL
    assert call(length=-1) == L.EINVAL
    assert call(out_frames=-1) == L.EINVAL
    assert call(row_stride=15999) == L.EINVAL
    assert call(gain=float("nan")) == L.EINVAL
    assert call(gain=float("inf")) == L.EINVAL
    for i in range(4):
        assert call(ptrs=tuple(j != i for j in range(4))) == L.EINVAL
    assert call(rows=0, ptrs=(False,) * 4) == L.OK  # nothing to enqueue: no pointer is read
    assert call(out_frames=0, ptrs=(False,) * 4) == L.OK
    assert call(length=200, row_stride=200) == L.ESHORT  # reflect needs n_fft/2 < length (one length for all rows)


def test_rnnt_features_backward_validation():
    L, lib = _lib_or_skip()
    fake = ctypes.c_void_p(0x1000)

    def call(rows=2, frames=101, n_mels=80, gain=1073676288.0, gs=(8080, 80, 1), ptrs=(True,) * 4):
        p = [fake if ok else None for ok in ptrs]
        return lib.b200a_rnnt_features_backward(p[0], gain, p[1], p[2], gs[0], gs[1], gs[2], rows, frames, n_mels, p[3],
                                                None)

    assert call(rows=-1) == L.EINVAL
    assert call(frames=-1) == L.EINVAL
    assert call(n_mels=0) == L.EINVAL
    assert call(gain=float("nan")) == L.EINVAL
    for i in range(3):
        assert call(gs=tuple(-1 if j == i else s for j, s in enumerate((8080, 80, 1)))) == L.EINVAL
    for i in range(4):
        assert call(ptrs=tuple(j != i for j in range(4))) == L.EINVAL
    assert call(rows=0, ptrs=(False,) * 4) == L.OK
    assert call(frames=0, ptrs=(False,) * 4) == L.OK


def test_forward_only_message_names_the_extractor():
    from audio_b200._plans import _no_autograd

    with pytest.raises(RuntimeError, match=r"RNNTFeatureExtractor.*differentiable\(features=True\)"):
        _no_autograd(torch.zeros(2, requires_grad=True))
