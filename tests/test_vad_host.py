"""vad without a GPU: the numpy oracle (tests/vad_oracle.py) against the reference fixture
(tests/golden/make_vad_golden.py), the host plan's constants against the reference's arithmetic, the errors and the
warning the Python surface raises before any launch, and the ABI statuses of b200a_vad_walk / b200a_vad_trigger."""
import ast
import ctypes
import os
import warnings

import numpy as np
import pytest
import torch

import vad_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vad_ref_cases.npz")


@pytest.fixture(scope="module")
def ref():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def cases(ref):
    return [k[4:] for k in ref if k.startswith("len_")]


def test_fixture_lengths_follow_from_its_measures(ref):
    """The oracle's trigger and flush rules on the recorded measures give the reference's output length, and every
    triggered case is at least 1e-3 from flipping a decision."""
    assert len(cases(ref)) == 22
    for c in cases(ref):
        x, sr, kw = O.case_input(ref, c), int(ref[f"sr_{c}"]), ast.literal_eval(str(ref[f"kw_{c}"]))
        (start, stop), hit, margins = O.trim(ref[f"meas_{c}"], x.shape[-1], sr, **kw)
        assert stop - start == int(ref[f"len_{c}"]), c
        assert hit < 0 or min(margins) >= 1e-3, c


def test_oracle_measures_match_fixture(ref):
    for c in ("mono_all", "stereo_all", "sr8000", "sr48000", "duration", "no_reduction", "burst_before"):
        x, sr, kw = O.case_input(ref, c), int(ref[f"sr_{c}"]), ast.literal_eval(str(ref[f"kw_{c}"]))
        exp = ref[f"meas_{c}"]
        got = O.measures(x, sr, **kw)[:exp.shape[0]]
        assert got.shape == exp.shape, c
        spread = np.abs(O.measures(x, sr, dtype=np.float64, **kw)[:exp.shape[0]] - exp).max()
        assert np.abs(got - exp).max() <= 2 * spread + 1e-5, (c, np.abs(got - exp).max(), spread)


@pytest.mark.parametrize("sr", [8000, 11025, 16000, 22050, 32000, 44100, 48000, 96000])
@pytest.mark.parametrize("kw", [{}, dict(measure_freq=25.0, search_time=0.7, allowed_gap=0.13, pre_trigger_time=0.03),
                                dict(measure_duration=0.07, boot_time=0.0, hp_filter_freq=120.0, lp_filter_freq=3000.0),
                                dict(hp_lifter_freq=300.0, lp_lifter_freq=1000.0, trigger_time=0.5)])
def test_plan_constants_match_reference_arithmetic(sr, kw):
    from audio_b200 import _filtering

    p = _filtering.VadPlan(sr, **kw)
    c = O.constants(sr, **kw)
    for name in ("measure_len_ws", "dft_len_ws", "measure_period_ns", "measures_len", "gap_len",
                 "fixed_pre_trigger_len_ns", "samples_len_ns", "spectrum_start", "spectrum_end", "cepstrum_start",
                 "cepstrum_end", "noise_up_time_mult", "noise_down_time_mult", "measure_smooth_time_mult",
                 "trigger_meas_time_mult", "boot_count_max"):
        assert getattr(p, name) == c[name], name
    assert np.array_equal(p.spectrum_window.numpy(), c["spectrum_window"])
    assert np.array_equal(p.cepstrum_window.numpy(), c["cepstrum_window"])
    d = p.desc(3)
    assert (d.channels, d.dft_len, d.period, d.fixed_pre_trigger) == (3, c["dft_len_ws"], c["measure_period_ns"],
                                                                       c["fixed_pre_trigger_len_ns"])


def test_reference_error_and_warning(ref):
    import audio_b200.functional as F
    import audio_b200.transforms as T

    x = torch.zeros(1, 16000)
    with pytest.raises(ValueError) as info:
        F.vad(x, 16000, lp_lifter_freq=100.0)
    assert f"ValueError: {info.value}" == str(ref["err_lifter"])
    with pytest.raises(ValueError):
        T.Vad(16000, lp_lifter_freq=100.0)(x)
    with pytest.warns(UserWarning) as rec, pytest.raises(RuntimeError, match="no CPU or ATen fallback"):
        F.vad(torch.zeros(1, 2, 16000), 16000)
    assert str(rec[0].message) == str(ref["warn_3d"])


def test_surface_rejects_cpu_and_other_dtypes():
    import audio_b200.functional as F
    import audio_b200.transforms as T

    with pytest.raises(RuntimeError, match="no CPU or ATen fallback"):
        F.vad(torch.zeros(2, 16000), 16000)
    with pytest.raises(RuntimeError, match="no CPU or ATen fallback"):
        T.Vad(16000)(torch.zeros(2, 16000, dtype=torch.float64))
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        with pytest.raises(RuntimeError, match="no CPU or ATen fallback"):
            F.vad(torch.zeros(16000), 16000)


def test_surface():
    import audio_b200.functional as F
    import audio_b200.transforms as T

    assert "vad" in F.__all__ and "Vad" in T.__all__
    m = T.Vad(16000, trigger_level=6.0, measure_duration=0.2)
    assert (m.sample_rate, m.trigger_level, m.measure_duration, m.lp_lifter_freq) == (16000, 6.0, 0.2, 2000.0)
    assert m.state_dict() == {}


# ---- the C ABI ---------------------------------------------------------------------------------------------------
def _desc(**kw):
    from audio_b200 import _filtering

    d = _filtering.VadPlan(16000).desc(2)
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def test_abi_statuses():
    from audio_b200 import _lib

    lib = _lib.lib()
    fake = 0x1000  # never dereferenced: every call below returns before a launch
    nbytes, walk, trigger = lib.b200a_vad_workspace_bytes, lib.b200a_vad_walk, lib.b200a_vad_trigger
    d = _desc()
    nb = nbytes(ctypes.byref(d), 1024)
    # status | S, N: 2 x 762 bins | mean: 2 | ring: 2 x 20 | addend: 2 x 1024 | first: 2 -- each rounded up to 256 bytes
    assert nb == 256 + 2 * 6144 + 256 + 256 + 8192 + 256
    assert nbytes(ctypes.byref(d), 7) < nb
    assert nbytes(ctypes.byref(_desc(dft_len=16384, spectrum_end=4000)), 1024) == 0
    assert walk(ctypes.byref(_desc(dft_len=16384, spectrum_end=4000)), 1024, 0, 1, fake, fake, fake, fake, 1 << 40,
                None) == _lib.EUNSUPPORTED
    assert trigger(ctypes.byref(d), 1 << 21, 0, 1, fake, fake, fake, 1 << 40, None) == _lib.EUNSUPPORTED
    assert walk(ctypes.byref(_desc(channels=65536)), 1, 0, 1, fake, fake, fake, fake, 1 << 40, None) == _lib.EUNSUPPORTED
    for bad in (dict(channels=0), dict(dft_len=1000), dict(dft_len=8), dict(spectrum_start=0),
                dict(spectrum_end=1025), dict(spectrum_start=800), dict(cepstrum_start=-1), dict(cepstrum_end=4),
                dict(cepstrum_end=513), dict(measures_len=0), dict(period=0)):
        assert nbytes(ctypes.byref(_desc(**bad)), 1024) == 0, bad
        assert walk(ctypes.byref(_desc(**bad)), 1024, 0, 1, fake, fake, fake, fake, 1 << 40, None) == _lib.EINVAL, bad
        assert trigger(ctypes.byref(_desc(**bad)), 1024, 0, 1, fake, fake, fake, 1 << 40, None) == _lib.EINVAL, bad
    assert nbytes(None, 1024) == 0 and nbytes(ctypes.byref(d), 0) == 0
    assert walk(None, 1024, 0, 1, fake, fake, fake, fake, nb, None) == _lib.EINVAL
    assert trigger(None, 1024, 0, 1, fake, fake, fake, nb, None) == _lib.EINVAL
    for frame0, frames in ((-1, 1), (0, -1), (0, 1025)):
        assert walk(ctypes.byref(d), 1024, frame0, frames, fake, fake, fake, fake, nb, None) == _lib.EINVAL
        assert trigger(ctypes.byref(d), 1024, frame0, frames, fake, fake, fake, nb, None) == _lib.EINVAL
    for i in range(4):  # spectrum, cepstrum_window, rows, workspace
        args = [fake] * 4
        args[i] = None
        assert walk(ctypes.byref(d), 1024, 0, 1, *args, nb, None) == _lib.EINVAL, i
    for i in range(3):  # power, measures, workspace
        args = [fake] * 3
        args[i] = None
        assert trigger(ctypes.byref(d), 1024, 0, 1, *args, nb, None) == _lib.EINVAL, i
    assert walk(ctypes.byref(d), 1024, 0, 1, fake, fake, fake, fake, nb - 1, None) == _lib.EWORKSPACE
    assert trigger(ctypes.byref(d), 1024, 0, 1, fake, fake, fake, nb - 1, None) == _lib.EWORKSPACE
    assert walk(ctypes.byref(d), 1024, 0, 0, fake, fake, fake, fake, nb, None) == _lib.OK  # nothing to enqueue
    assert trigger(ctypes.byref(d), 1024, 0, 0, fake, fake, fake, nb, None) == _lib.OK
