"""A numpy restatement of the reference's vad (pytorch/audio/src/torchaudio/functional/filtering.py:1414-1702), for the
fixture and the GPU tests.

``measures`` runs the measurement of every frame: the windowed rFFT, the smoothing and noise tracker, the cepstrum rFFT
and its band power.  With ``dtype=np.float32`` it keeps the reference's float32 / float64 mix (FFTs in float64, rounded
to float32); with ``np.float64`` everything is double, which gives the reference's own float32 error.  ``trim`` runs the
reference's trigger, flush and slicing rules on given measures, and reports how far every decision was from flipping.
The windows are the reference's torch expressions, evaluated on the CPU.
"""
import math

import numpy as np
import torch


def constants(sample_rate, trigger_level=7.0, trigger_time=0.25, search_time=1.0, allowed_gap=0.25,
              pre_trigger_time=0.0, boot_time=0.35, noise_up_time=0.1, noise_down_time=0.01,
              noise_reduction_amount=1.35, measure_freq=20.0, measure_duration=None, measure_smooth_time=0.4,
              hp_filter_freq=50.0, lp_filter_freq=6000.0, hp_lifter_freq=150.0, lp_lifter_freq=2000.0):
    """The host constants of filtering.py:1579-1629, by the same Python-float arithmetic."""
    md = 2.0 / measure_freq if measure_duration is None else measure_duration
    ws = int(sample_rate * md + 0.5)
    dft = 16
    while dft < ws:
        dft *= 2
    period = int(sample_rate / measure_freq + 0.5)
    n = math.ceil(search_time * measure_freq)
    fixed_pre = int(pre_trigger_time * sample_rate + 0.5)
    s0 = max(int(hp_filter_freq / sample_rate * dft + 0.5), 1)
    s1 = min(int(lp_filter_freq / sample_rate * dft + 0.5), dft // 2)
    c0 = math.ceil(sample_rate * 0.5 / lp_lifter_freq)
    c1 = min(math.floor(sample_rate * 0.5 / hp_lifter_freq), dft // 4)
    sw = torch.full((ws,), 2.0 / math.sqrt(float(ws))) * torch.hann_window(ws, dtype=torch.float)
    cw = torch.full((s1 - s0,), 2.0 / math.sqrt(float(s1) - s0)) * torch.hann_window(s1 - s0, dtype=torch.float)
    return dict(
        measure_len_ws=ws, dft_len_ws=dft, measure_period_ns=period, measures_len=n,
        gap_len=int(allowed_gap * measure_freq + 0.5), fixed_pre_trigger_len_ns=fixed_pre,
        samples_len_ns=fixed_pre + n * period + ws, spectrum_start=s0, spectrum_end=s1, cepstrum_start=c0,
        cepstrum_end=c1, spectrum_window=sw.numpy(), cepstrum_window=cw.numpy(),
        noise_up_time_mult=math.exp(-1.0 / (noise_up_time * measure_freq)),
        noise_down_time_mult=math.exp(-1.0 / (noise_down_time * measure_freq)),
        measure_smooth_time_mult=math.exp(-1.0 / (measure_smooth_time * measure_freq)),
        trigger_meas_time_mult=math.exp(-1.0 / (trigger_time * measure_freq)),
        boot_count_max=int(boot_time * measure_freq - 0.5), noise_reduction_amount=noise_reduction_amount,
        trigger_level=trigger_level)


def num_frames(c, length):
    return len(range(c["measure_len_ws"], length, c["measure_period_ns"]))


def measures(x, sample_rate, dtype=np.float32, **kw):
    """(frames, channels) float64 measures of every frame of the (..., time) input."""
    c = constants(sample_rate, **kw)
    x = np.asarray(x, dtype=np.float32)
    x = x.reshape(-1, x.shape[-1])
    ch, length = x.shape
    ws, dft, period = c["measure_len_ws"], c["dft_len_ws"], c["measure_period_ns"]
    s0, s1, c0, c1 = c["spectrum_start"], c["spectrum_end"], c["cepstrum_start"], c["cepstrum_end"]
    f = dtype
    sw, cw = c["spectrum_window"].astype(f), c["cepstrum_window"].astype(f)
    up, down = f(np.float32(c["noise_up_time_mult"])), f(np.float32(c["noise_down_time_mult"]))
    nra, msm = f(c["noise_reduction_amount"]), c["measure_smooth_time_mult"]
    spec = np.zeros((ch, s1 - s0), f)
    noise = np.zeros((ch, s1 - s0), f)
    out = []
    for g in range(num_frames(c, length)):
        pos = ws + g * period
        buf = np.zeros((ch, dft), np.float64)
        buf[:, :ws] = (x[:, pos - ws:pos].astype(f) * sw).astype(np.float64)
        mag = np.abs(np.fft.rfft(buf, axis=1))[:, s0:s1].astype(f)
        boot = c["boot_count_max"] < 0 or g <= c["boot_count_max"]
        mult = g / (1.0 + g) if boot else msm
        spec = spec * f(mult) + mag * f(1 - mult)
        d = spec * spec
        nm = np.zeros_like(d) if boot else np.where(d > noise, up, down)
        noise = noise * nm + d * (f(1) - nm)
        r = np.sqrt(np.maximum(f(0), d - nra * noise))
        cep = np.zeros((ch, dft // 2), np.float64)
        cep[:, s0:s1] = (r * cw).astype(np.float64)
        p = (np.abs(np.fft.rfft(cep, axis=1)) ** 2)[:, c0:c1].astype(f).sum(axis=1, dtype=f).astype(np.float64)
        out.append([max(0.0, 21 + math.log(v / (c1 - c0))) if v > 0 else 0.0 for v in p])
    return np.array(out, dtype=np.float64).reshape(-1, ch)


def trim(meas, length, sample_rate, **kw):
    """The reference's trigger and flush rules (filtering.py:1643-1702) on (frames, channels) measures, which must
    cover every frame the reference runs up to its trigger.  Returns (start, stop) of the kept samples, the trigger
    frame (-1 for none) and the decision margins: the least |mean - trigger_level| of every mean tested, the least
    |meas - trigger_level| and the least nonzero meas of every measure a flush scan read (inf when none was read)."""
    c = constants(sample_rate, **kw)
    meas = np.asarray(meas, dtype=np.float64)
    ch = meas.shape[1] if meas.ndim == 2 else 0
    n, gap, level = c["measures_len"], c["gap_len"], np.float32(c["trigger_level"])
    tm = c["trigger_meas_time_mult"]
    ring = np.zeros((ch, n), np.float32)
    mean = np.zeros(ch, np.float32)
    m_mean = m_meas = m_zero = math.inf
    frames = num_frames(c, length)
    pos, idx, flush, hit = 0, 0, 0, -1
    for g in range(frames):
        pos = c["measure_len_ws"] + g * c["measure_period_ns"]
        triggered = False
        for i in range(ch):
            v = meas[g, i]
            ring[i, idx] = np.float32(v)
            mean[i] = np.float32(mean[i] * np.float32(tm)) + np.float32(v * (1.0 - tm))
            m_mean = min(m_mean, abs(float(mean[i]) - float(level)))
            triggered = triggered or bool(mean[i] >= level)
            if triggered:
                k, j_trig, j_zero = idx, n, n
                for j in range(n):
                    m = ring[i, k]
                    m_meas = min(m_meas, abs(float(m) - float(level)))
                    if m != 0:
                        m_zero = min(m_zero, float(m))
                    if m >= level and j <= j_trig + gap:
                        j_zero = j_trig = j
                    elif m == 0 and j_trig >= j_zero:
                        j_zero = j
                    k = (k + n - 1) % n
                flush = min(max(flush, min(j, j_zero)), n)
        idx = (idx + 1) % n
        if triggered:
            hit = g
            break
    margins = (m_mean, m_meas, m_zero)
    fixed_pre = c["fixed_pre_trigger_len_ns"]
    if hit < 0 and length >= fixed_pre:
        return (0, fixed_pre), hit, margins
    flushed = (n - flush) * c["measure_period_ns"] if hit >= 0 else 0
    return (max(pos - c["samples_len_ns"] + flushed, 0), length), hit, margins


def _stored(x):
    """A stored input as float32: int16 samples become samples / 32768, as the reference loads the assets."""
    return x.astype(np.float32) / np.float32(32768) if x.dtype == np.int16 else x


def case_input(ref, name):
    """The float32 input of fixture case ``name``: stored, the input of another case (reshaped by ``shape_name``), or
    seeded low-level noise with parts of a stored input added (``noise_name``, ``mix_name``, ``source_name``)."""
    if f"x_{name}" in ref:
        x = ref[f"x_{name}"]
        if x.dtype.kind != "U":
            return _stored(x)
        x = _stored(ref[str(x)])
        return x.reshape(tuple(int(v) for v in ref[f"shape_{name}"])) if f"shape_{name}" in ref else x
    seed, channels, samples, level = ref[f"noise_{name}"]
    rng = np.random.default_rng(int(seed))
    x = (rng.standard_normal((int(channels), int(samples))) * level).astype(np.float32)
    if f"mix_{name}" in ref:
        src = _stored(ref[str(ref[f"source_{name}"])]).reshape(-1)
        for ch, offset, start, stop, scale in ref[f"mix_{name}"]:
            part = src[int(start):int(stop)] * np.float32(scale)
            x[int(ch), int(offset):int(offset) + part.shape[0]] += part
    return x
