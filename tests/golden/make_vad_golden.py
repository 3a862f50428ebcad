#!/usr/bin/env python
"""Generate tests/golden/vad_ref_cases.npz, the vad fixture (needs a pytorch/audio checkout named by AUDIO_REFERENCE;
run once):

    AUDIO_REFERENCE=/path/to/audio python tests/golden/make_vad_golden.py

Per case ``c``, from the reference's CPU vad (tests/vad_oracle.py:case_input rebuilds the inputs):
- ``x_c``: the input, stored once: the two assets as their int16 samples (the reference reads them as samples / 32768),
  the resampled ones as float32; or the key of another case's input, with ``shape_c`` when it is reshaped;
- or, for the synthetic cases, ``noise_c`` = (seed, channels, samples, level) for seeded low-level noise and ``mix_c``
  rows (channel, offset, start, stop, scale) adding ``source_c[start:stop] * scale`` at ``offset``;
- ``sr_c``: the sample rate; ``kw_c``: the keyword arguments (a repr of a dict);
- ``len_c``: the output length; ``meas_c``: the (frames, channels) float64 measures the reference computed, recorded by
  wrapping ``filtering._measure``;
- ``margin_c``: the decision margins of tests/vad_oracle.py:trim.  Every triggered case clears 1e-3 on each.
Also ``err_*``: the reference's error strings ("<exception type>: <message>"), and ``warn_3d``: its warning.
"""
import os
import sys
import warnings

import numpy as np
import scipy.io.wavfile as wavfile
import torch

REF = os.environ["AUDIO_REFERENCE"]  # a pytorch/audio checkout at the pinned version
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(REF, "src"))
sys.path.insert(0, os.path.dirname(HERE))
import torchaudio  # noqa: E402
import torchaudio.functional as RF  # noqa: E402
from torchaudio.functional import filtering  # noqa: E402

import vad_oracle as O  # noqa: E402

assert torchaudio.__file__.startswith(REF), torchaudio.__file__

ASSETS = os.path.join(REF, "test", "torchaudio_unittest", "assets")
MARGIN = 1e-3


def load(name):
    sr, d = wavfile.read(os.path.join(ASSETS, name))
    return sr, np.ascontiguousarray(d.T if d.ndim == 2 else d[None])  # int16 (channels, time)


def err(fn):
    try:
        fn()
    except Exception as e:  # noqa: BLE001
        return f"{type(e).__name__}: {e}"
    raise AssertionError("expected an error")


def main():
    sr_m, mono = load("vad-go-mono-32000.wav")
    sr_s, stereo = load("vad-go-stereo-44100.wav")
    out = {"x_mono": mono, "x_stereo": stereo}
    speech = RF.resample(torch.from_numpy(O.case_input(out, "mono")), sr_m, 16000)[0].numpy()
    for sr in (8000, 16000, 22050, 48000):
        out[f"x_sr{sr}"] = speech[None] if sr == 16000 else \
            RF.resample(torch.from_numpy(O.case_input(out, "mono")), sr_m, sr).numpy()
    cases = {  # name -> (sample rate, kwargs); the inputs are in `out`
        "mono": (sr_m, {}),
        "stereo": (sr_s, {}),
        "mono_all": (sr_m, dict(trigger_level=1e9)),
        "stereo_all": (sr_s, dict(trigger_level=1e9)),
        "d1": (sr_m, {}),
        "d3": (sr_s, {}),
        "pre_trigger": (sr_m, dict(pre_trigger_time=0.1)),
        "gap": (sr_s, dict(allowed_gap=0.1)),
        "search": (sr_m, dict(search_time=0.5)),
        "no_boot": (sr_m, dict(boot_time=0.0)),
        "no_reduction": (sr_s, dict(noise_reduction_amount=0.0)),
        "duration": (sr_m, dict(measure_duration=0.15)),
        "sr8000": (8000, {}),
        "sr16000": (16000, {}),
        "sr22050": (22050, {}),
        "sr48000": (48000, {}),
        "never": (16000, {}),
        "short_below": (16000, dict(pre_trigger_time=0.01)),
        "short_above": (16000, dict(pre_trigger_time=0.5)),
        "burst_after": (16000, {}),
        "burst_before": (16000, {}),
        "long": (16000, {}),
    }
    for name, (sr, _) in cases.items():
        if name.startswith("mono") or name in ("pre_trigger", "search", "no_boot", "duration"):
            out[f"x_{name}"] = np.array("x_mono") if name != "mono" else mono
        elif name.startswith("stereo") or name in ("gap", "no_reduction"):
            out[f"x_{name}"] = np.array("x_stereo") if name != "stereo" else stereo
    out["x_d1"], out["shape_d1"] = np.array("x_mono"), np.array(mono.shape[1:])
    out["x_d3"], out["shape_d3"] = np.array("x_stereo"), np.array((1,) + stereo.shape)
    out["noise_never"] = np.array([1, 1, 32000, 1e-3])
    out["noise_short_below"] = out["noise_short_above"] = np.array([2, 1, 1000, 1e-3])
    # two channels of low noise; one has the word at 1.5 s, the other a 60 ms burst of its loudest part at 1.0 s: the
    # burst counts in the flush scan only when its channel comes after the triggering one
    loud = int(np.argmax(np.abs(speech)))
    word, burst = (24000, 0, speech.shape[0], 1.0), (16000, loud - 480, loud + 480, 0.5)
    for name, rows in (("burst_after", [(0,) + word, (1,) + burst]), ("burst_before", [(1,) + word, (0,) + burst])):
        out[f"noise_{name}"], out[f"mix_{name}"] = np.array([3, 2, 48000, 1e-3]), np.array(rows, dtype=np.float64)
        out[f"source_{name}"] = np.array("x_sr16000")
    # 64 s of seeded noise before the word at 16 kHz: 1300 frames, more than one 1024-frame chunk
    n_noise = 64 * 16000
    out["noise_long"] = np.array([7, 1, n_noise + speech.shape[0], 1e-3])
    out["mix_long"] = np.array([(0, n_noise, 0, speech.shape[0], 1.0)], dtype=np.float64)
    out["source_long"] = np.array("x_sr16000")

    record = []
    orig = filtering._measure

    def measure(*args, **kwargs):
        r = orig(*args, **kwargs)
        record.append(r)
        return r

    filtering._measure = measure
    for name, (sr, kw) in cases.items():
        x = torch.from_numpy(O.case_input(out, name))
        record.clear()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            y = RF.vad(x, sr, **kw)
        ch = int(np.prod(x.shape[:-1]))
        meas = np.array(record, dtype=np.float64).reshape(-1, ch)
        (start, stop), hit, margins = O.trim(meas, x.shape[-1], sr, **kw)
        assert stop - start == y.shape[-1], (name, start, stop, y.shape)
        if hit >= 0:
            assert min(margins) >= MARGIN, (name, margins)
        assert name != "long" or hit > 1024, hit
        out[f"sr_{name}"], out[f"kw_{name}"] = np.array(sr), np.array(repr(kw))
        out[f"len_{name}"], out[f"meas_{name}"], out[f"margin_{name}"] = np.array(y.shape[-1]), meas, np.array(margins)
        print(f"{name}: {tuple(x.shape)} @ {sr} -> {y.shape[-1]} (trigger frame {hit}, margins {margins})")
    filtering._measure = orig

    x_mono, x_stereo = torch.from_numpy(O.case_input(out, "mono")), torch.from_numpy(O.case_input(out, "stereo"))
    out["err_lifter"] = np.array(err(lambda: RF.vad(x_mono, 16000, lp_lifter_freq=100.0)))
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        RF.vad(x_stereo.reshape(1, 2, -1), sr_s)
    out["warn_3d"] = np.array(str(w[0].message))
    np.savez_compressed(os.path.join(HERE, "vad_ref_cases.npz"), **out)


if __name__ == "__main__":
    main()
