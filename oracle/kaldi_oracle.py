"""CPU restatement (numpy, float64) of the reference's Kaldi-compatible features.

TEST INFRASTRUCTURE ONLY: imported by tests/, never by the product (audio_b200/ has no CPU path).

Follows pytorch/audio/src/torchaudio/compliance/kaldi.py; every function cites the lines it restates.
Parity PINNED: tests/test_kaldi.py checks this file against the 311 Kaldi-binary outputs the reference's own
tests hold (test/torchaudio_unittest/assets/kaldi_expected_results, consumed by
compliance/kaldi/kaldi_compatibility_impl.py:20-48 with rtol 1e-4) and against outputs of the reference
itself on longer signals (tests/golden/make_kaldi_golden.py -> kaldi_ref_cases.npz).
"""
import math

import numpy as np

EPS = float(np.finfo(np.float32).eps)  # kaldi.py:21-22


def next_power_of_2(x):
    """kaldi.py:39-41."""
    return 1 if x == 0 else 2 ** (x - 1).bit_length()


def num_frames(num_samples, window_size, window_shift, snip_edges):
    """m of _get_strided, kaldi.py:62-68."""
    if snip_edges:
        return 0 if num_samples < window_size else 1 + (num_samples - window_size) // window_shift
    return (num_samples + window_shift // 2) // window_shift


def get_strided(wave, window_size, window_shift, snip_edges):
    """kaldi.py:44-83: (m, window_size) frames; without snip_edges the signal is mirrored at both ends."""
    wave = np.asarray(wave, dtype=np.float64)
    n = wave.shape[0]
    m = num_frames(n, window_size, window_shift, snip_edges)
    if snip_edges:
        if m == 0:
            return np.zeros((0, 0))
        start = 0
        ext = wave
    else:
        pad = window_size // 2 - window_shift // 2
        rev = wave[::-1]
        if pad > 0:
            ext = np.concatenate([rev[n - pad:], wave, rev])
        else:
            ext = np.concatenate([wave[-pad:], rev])
        start = 0
    idx = start + window_shift * np.arange(m)[:, None] + np.arange(window_size)[None, :]
    return ext[idx]


def feature_window(window_type, window_size, blackman_coeff):
    """kaldi.py:86-113 (symmetric windows: the denominator is window_size - 1)."""
    i = np.arange(window_size, dtype=np.float64)
    a = 2.0 * math.pi / (window_size - 1)
    if window_type == "hanning":
        return 0.5 - 0.5 * np.cos(a * i)
    if window_type == "hamming":
        return 0.54 - 0.46 * np.cos(a * i)
    if window_type == "povey":
        return (0.5 - 0.5 * np.cos(a * i)) ** 0.85
    if window_type == "rectangular":
        return np.ones(window_size)
    if window_type == "blackman":
        return blackman_coeff - 0.5 * np.cos(a * i) + (0.5 - blackman_coeff) * np.cos(2 * a * i)
    raise Exception("Invalid window type " + window_type)


def log_energy(frames, energy_floor):
    """kaldi.py:116-123."""
    le = np.log(np.maximum((frames ** 2).sum(1), EPS))
    if energy_floor == 0.0:
        return le
    return np.maximum(le, math.log(energy_floor))


def window_properties(num_samples, sample_frequency, frame_shift, frame_length, round_to_power_of_two,
                      preemphasis_coefficient):
    """kaldi.py:126-151 (the assertions become the same AssertionErrors)."""
    window_shift = int(sample_frequency * frame_shift * 0.001)
    window_size = int(sample_frequency * frame_length * 0.001)
    padded = next_power_of_2(window_size) if round_to_power_of_two else window_size
    assert 2 <= window_size <= num_samples
    assert 0 < window_shift
    assert padded % 2 == 0
    assert 0.0 <= preemphasis_coefficient <= 1.0
    assert sample_frequency > 0
    return window_shift, window_size, padded


def get_window(wave, padded, window_size, window_shift, window_type, blackman_coeff, snip_edges, raw_energy,
               energy_floor, remove_dc_offset, preemphasis_coefficient):
    """kaldi.py:153-216 with dither = 0: conditioned, windowed, zero-padded frames and their log energy."""
    fr = get_strided(wave, window_size, window_shift, snip_edges)
    if fr.size == 0:
        return np.zeros((0, padded)), np.zeros(0)
    if remove_dc_offset:
        fr = fr - fr.mean(1, keepdims=True)
    if raw_energy:
        le = log_energy(fr, energy_floor)
    if preemphasis_coefficient != 0.0:
        prev = np.concatenate([fr[:, :1], fr[:, :-1]], axis=1)  # replicate padding on the left
        fr = fr - preemphasis_coefficient * prev
    fr = fr * feature_window(window_type, window_size, blackman_coeff)[None, :]
    if padded != window_size:
        fr = np.concatenate([fr, np.zeros((fr.shape[0], padded - window_size))], axis=1)
    if not raw_energy:
        le = log_energy(fr, energy_floor)
    return fr, le


def subtract_column_mean(x, subtract_mean):
    """kaldi.py:219-226."""
    return x - x.mean(0, keepdims=True) if subtract_mean else x


def spectrogram(wave, blackman_coeff=0.42, energy_floor=1.0, frame_length=25.0, frame_shift=10.0, min_duration=0.0,
                preemphasis_coefficient=0.97, raw_energy=True, remove_dc_offset=True, round_to_power_of_two=True,
                sample_frequency=16000.0, snip_edges=True, subtract_mean=False, window_type="povey", dither=0.0,
                channel=-1):
    """kaldi.py:229-316: log power spectrum, bin 0 replaced by the frame's log energy."""
    wave = np.asarray(wave, dtype=np.float64)
    if wave.ndim == 2:
        wave = wave[max(channel, 0)]
    shift, size, padded = window_properties(len(wave), sample_frequency, frame_shift, frame_length,
                                            round_to_power_of_two, preemphasis_coefficient)
    if len(wave) < min_duration * sample_frequency:
        return np.zeros(0)
    fr, le = get_window(wave, padded, size, shift, window_type, blackman_coeff, snip_edges, raw_energy, energy_floor,
                        remove_dc_offset, preemphasis_coefficient)
    spec = np.log(np.maximum(np.abs(np.fft.rfft(fr, axis=1)) ** 2, EPS))
    spec[:, 0] = le
    return subtract_column_mean(spec, subtract_mean)


def mel_scale(freq):
    """kaldi.py:326-331 (in the dtype of `freq`)."""
    freq = np.asarray(freq)
    return 1127.0 * np.log(1.0 + freq / 700.0)


def inverse_mel_scale(mel):
    """kaldi.py:318-323 (in the dtype of `mel`)."""
    mel = np.asarray(mel)
    return 700.0 * (np.exp(mel / 1127.0) - 1.0)


def vtln_warp_freq(vtln_low_cutoff, vtln_high_cutoff, low_freq, high_freq, vtln_warp_factor, freq):
    """kaldi.py:334-405: piecewise-linear warp with inflection points l and h; identity outside [low, high]."""
    assert vtln_low_cutoff > low_freq
    assert vtln_high_cutoff < high_freq
    lo = vtln_low_cutoff * max(1.0, vtln_warp_factor)
    hi = vtln_high_cutoff * min(1.0, vtln_warp_factor)
    scale = 1.0 / vtln_warp_factor
    f_lo, f_hi = scale * lo, scale * hi
    assert lo > low_freq and hi < high_freq
    scale_left = (f_lo - low_freq) / (lo - low_freq)
    scale_right = (high_freq - f_hi) / (high_freq - hi)
    freq = np.asarray(freq)
    res = np.where(freq >= hi, high_freq + scale_right * (freq - high_freq), scale * freq)
    res = np.where(freq < lo, low_freq + scale_left * (freq - low_freq), res)
    return np.where((freq < low_freq) | (freq > high_freq), freq, res).astype(freq.dtype)


def vtln_warp_mel_freq(vtln_low, vtln_high, low_freq, high_freq, warp, mel):
    """kaldi.py:408-433."""
    return mel_scale(vtln_warp_freq(vtln_low, vtln_high, low_freq, high_freq, warp, inverse_mel_scale(mel)))


def get_mel_banks(num_bins, window_length_padded, sample_freq, low_freq, high_freq, vtln_low, vtln_high, vtln_warp,
                  dtype=np.float32):
    """kaldi.py:436-511: (num_bins, padded/2) triangular filters in the mel domain, and their centre frequencies.

    The reference builds this table in float32 whatever the waveform's dtype (`torch.arange` / default dtype,
    :484-496) and the narrow high filters lose ~1e-5 relative to the cancellation in `mel - left_mel`; the Kaldi
    goldens are matched at rtol 1e-4 only with the same rounding, hence dtype=float32 arithmetic here as well."""
    assert num_bins > 3
    assert window_length_padded % 2 == 0
    num_fft_bins = window_length_padded // 2
    nyquist = 0.5 * sample_freq
    if high_freq <= 0.0:
        high_freq += nyquist
    assert (0.0 <= low_freq < nyquist) and (0.0 < high_freq <= nyquist) and (low_freq < high_freq)
    fft_bin_width = sample_freq / window_length_padded
    mel_low = 1127.0 * math.log(1.0 + low_freq / 700.0)  # mel_scale_scalar, python floats (:326-327)
    mel_high = 1127.0 * math.log(1.0 + high_freq / 700.0)
    delta = (mel_high - mel_low) / (num_bins + 1)
    if vtln_high < 0.0:
        vtln_high += nyquist
    assert vtln_warp == 1.0 or ((low_freq < vtln_low < high_freq) and (0.0 < vtln_high < high_freq)
                                and (vtln_low < vtln_high))
    b = np.arange(num_bins).astype(dtype)[:, None]
    left = (mel_low + b * dtype(delta)).astype(dtype)
    center = (mel_low + (b + dtype(1.0)) * dtype(delta)).astype(dtype)
    right = (mel_low + (b + dtype(2.0)) * dtype(delta)).astype(dtype)
    if vtln_warp != 1.0:
        left = vtln_warp_mel_freq(vtln_low, vtln_high, low_freq, high_freq, vtln_warp, left).astype(dtype)
        center = vtln_warp_mel_freq(vtln_low, vtln_high, low_freq, high_freq, vtln_warp, center).astype(dtype)
        right = vtln_warp_mel_freq(vtln_low, vtln_high, low_freq, high_freq, vtln_warp, right).astype(dtype)
    mel = mel_scale((fft_bin_width * np.arange(num_fft_bins).astype(dtype)).astype(dtype)).astype(dtype)[None, :]
    up = (mel - left) / (center - left)
    down = (right - mel) / (right - center)
    if vtln_warp == 1.0:
        bins = np.maximum(dtype(0.0), np.minimum(up, down))
    else:
        bins = np.zeros_like(up)
        up_idx = (mel > left) & (mel <= center)
        down_idx = (mel > center) & (mel < right)
        bins[up_idx] = up[up_idx]
        bins[down_idx] = down[down_idx]
    return bins.astype(np.float64), inverse_mel_scale(center)[:, 0].astype(np.float64)


def fbank(wave, blackman_coeff=0.42, energy_floor=1.0, frame_length=25.0, frame_shift=10.0, high_freq=0.0,
          htk_compat=False, low_freq=20.0, min_duration=0.0, num_mel_bins=23, preemphasis_coefficient=0.97,
          raw_energy=True, remove_dc_offset=True, round_to_power_of_two=True, sample_frequency=16000.0,
          snip_edges=True, subtract_mean=False, use_energy=False, use_log_fbank=True, use_power=True,
          vtln_high=-500.0, vtln_low=100.0, vtln_warp=1.0, window_type="povey", dither=0.0, channel=-1):
    """kaldi.py:514-645."""
    wave = np.asarray(wave, dtype=np.float64)
    if wave.ndim == 2:
        wave = wave[max(channel, 0)]
    shift, size, padded = window_properties(len(wave), sample_frequency, frame_shift, frame_length,
                                            round_to_power_of_two, preemphasis_coefficient)
    if len(wave) < min_duration * sample_frequency:
        return np.zeros(0)
    fr, le = get_window(wave, padded, size, shift, window_type, blackman_coeff, snip_edges, raw_energy, energy_floor,
                        remove_dc_offset, preemphasis_coefficient)
    spec = np.abs(np.fft.rfft(fr, axis=1))
    if use_power:
        spec = spec ** 2
    banks, _ = get_mel_banks(num_mel_bins, padded, sample_frequency, low_freq, high_freq, vtln_low, vtln_high, vtln_warp)
    banks = np.concatenate([banks, np.zeros((num_mel_bins, 1))], axis=1)  # the Nyquist bin gets no weight
    mel = spec @ banks.T
    if use_log_fbank:
        mel = np.log(np.maximum(mel, EPS))
    if use_energy:
        mel = np.concatenate([mel, le[:, None]], axis=1) if htk_compat else np.concatenate([le[:, None], mel], axis=1)
    return subtract_column_mean(mel, subtract_mean)


def dct_matrix(num_ceps, num_mel_bins):
    """kaldi.py:648-658: orthonormal DCT-II (functional.create_dct) with the first column set to sqrt(1/n)."""
    n = np.arange(num_mel_bins, dtype=np.float64)
    k = np.arange(num_mel_bins, dtype=np.float64)[:, None]
    dct = np.cos(math.pi / num_mel_bins * (n + 0.5) * k)
    dct[0] *= 1.0 / math.sqrt(2.0)
    dct *= math.sqrt(2.0 / num_mel_bins)
    dct = dct.T.copy()  # (num_mel_bins, num_mel_bins), right-multiplied
    dct[:, 0] = math.sqrt(1.0 / num_mel_bins)
    return dct[:, :num_ceps]


def lifter_coeffs(num_ceps, cepstral_lifter):
    """kaldi.py:661-666."""
    i = np.arange(num_ceps, dtype=np.float64)
    return 1.0 + 0.5 * cepstral_lifter * np.sin(math.pi * i / cepstral_lifter)


def mfcc(wave, blackman_coeff=0.42, cepstral_lifter=22.0, energy_floor=1.0, frame_length=25.0, frame_shift=10.0,
         high_freq=0.0, htk_compat=False, low_freq=20.0, num_ceps=13, min_duration=0.0, num_mel_bins=23,
         preemphasis_coefficient=0.97, raw_energy=True, remove_dc_offset=True, round_to_power_of_two=True,
         sample_frequency=16000.0, snip_edges=True, subtract_mean=False, use_energy=False, vtln_high=-500.0,
         vtln_low=100.0, vtln_warp=1.0, window_type="povey", dither=0.0, channel=-1):
    """kaldi.py:669-813."""
    assert num_ceps <= num_mel_bins
    feat = fbank(wave, blackman_coeff=blackman_coeff, energy_floor=energy_floor, frame_length=frame_length,
                 frame_shift=frame_shift, high_freq=high_freq, htk_compat=htk_compat, low_freq=low_freq,
                 min_duration=min_duration, num_mel_bins=num_mel_bins, preemphasis_coefficient=preemphasis_coefficient,
                 raw_energy=raw_energy, remove_dc_offset=remove_dc_offset, round_to_power_of_two=round_to_power_of_two,
                 sample_frequency=sample_frequency, snip_edges=snip_edges, subtract_mean=False, use_energy=use_energy,
                 use_log_fbank=True, use_power=True, vtln_high=vtln_high, vtln_low=vtln_low, vtln_warp=vtln_warp,
                 window_type=window_type, channel=channel)
    if feat.size == 0:
        return feat
    if use_energy:
        le = feat[:, num_mel_bins if htk_compat else 0]
        off = int(not htk_compat)
        feat = feat[:, off:num_mel_bins + off]
    feat = feat @ dct_matrix(num_ceps, num_mel_bins)
    if cepstral_lifter != 0.0:
        feat = feat * lifter_coeffs(num_ceps, cepstral_lifter)[None, :]
    if use_energy:
        feat[:, 0] = le
    if htk_compat:
        energy = feat[:, :1].copy()
        if not use_energy:
            energy *= math.sqrt(2)
        feat = np.concatenate([feat[:, 1:], energy], axis=1)
    return subtract_column_mean(feat, subtract_mean)
