"""Drop-in ``torchaudio.compliance.kaldi`` (spectrogram / fbank / mfcc), backed by libb200audio.so.

Same names, argument order, defaults, assertions and output shapes as the reference
(pytorch/audio/src/torchaudio/compliance/kaldi.py: ``spectrogram`` 229-316, ``fbank`` 514-645, ``mfcc`` 669-813,
``get_mel_banks`` 436-511 and the mel / VTLN helpers 318-433).  The constant tables (window, mel banks, DCT, lifter)
are built on the host with the reference's own op sequence in float32, so they are the reference's tables; the
per-frame work -- framing (snip_edges or mirrored edges), DC removal, log energy, pre-emphasis, window, zero padding,
FFT, power, mel projection, log -- is ONE fused kernel launch (``b200a_kaldi_run``), followed where asked for by the
DCT (``b200a_mfcc_finish``) and the column-mean subtraction (``b200a_subtract_column_mean``).

Waveform gradients are opt-in: inside ``audio_b200.differentiable(kaldi=True)`` a waveform that requires grad gets
torch's autograd of the reference op sequence, ties of the log floor and the energy floor included, from
``b200a_kaldi_backward`` (the same launches run forward, so the features are bit-identical to the no-grad call).
Outside it, or with only the other switches on, a waveform that requires grad raises "forward-only": Kaldi features
are usually data-pipeline preprocessing.  Gradients with respect to the window, mel banks, DCT or lifter, and
second-order gradients, are not offered.

Differences, all explicit: CUDA float32 waveforms only, and ``dither`` must be 0 (the reference draws it with
``torch.randn`` per frame element, which no other generator reproduces).  ``fbank_batch`` / ``mfcc_batch`` /
``spectrogram_batch`` are extensions that take ``(batch, time)`` and return ``(batch, frames, features)``.
"""
from __future__ import annotations

import math
from typing import Dict, Tuple

import torch
from torch import Tensor

from torch.autograd.function import once_differentiable

from .. import _lib, _ops
from .._constants import create_dct
from .._plans import (FrontendPlan, _no_autograd, _require_cuda_f32, _stream_ptr, _wants_grad, is_kaldi_differentiable,
                      pack_rows)

__all__ = [
    "get_mel_banks",
    "inverse_mel_scale",
    "inverse_mel_scale_scalar",
    "mel_scale",
    "mel_scale_scalar",
    "spectrogram",
    "fbank",
    "mfcc",
    "vtln_warp_freq",
    "vtln_warp_mel_freq",
    "spectrogram_batch",
    "fbank_batch",
    "mfcc_batch",
]

EPSILON = torch.tensor(torch.finfo(torch.float).eps)
MILLISECONDS_TO_SECONDS = 0.001

HAMMING = "hamming"
HANNING = "hanning"
POVEY = "povey"
RECTANGULAR = "rectangular"
BLACKMAN = "blackman"
WINDOWS = [HAMMING, HANNING, POVEY, RECTANGULAR, BLACKMAN]


# ---- scalar / tensor helpers of the mel axis (host math, reference kaldi.py:318-433) ---------------------------
def inverse_mel_scale_scalar(mel_freq: float) -> float:
    return 700.0 * (math.exp(mel_freq / 1127.0) - 1.0)


def inverse_mel_scale(mel_freq: Tensor) -> Tensor:
    return 700.0 * ((mel_freq / 1127.0).exp() - 1.0)


def mel_scale_scalar(freq: float) -> float:
    return 1127.0 * math.log(1.0 + freq / 700.0)


def mel_scale(freq: Tensor) -> Tensor:
    return 1127.0 * (1.0 + freq / 700.0).log()


def vtln_warp_freq(
    vtln_low_cutoff: float,
    vtln_high_cutoff: float,
    low_freq: float,
    high_freq: float,
    vtln_warp_factor: float,
    freq: Tensor,
) -> Tensor:
    """Three-piece linear warp F with F(low_freq) = low_freq, F(high_freq) = high_freq and slope 1/warp between the
    inflection points l = vtln_low * max(1, warp) and h = vtln_high * min(1, warp) (reference kaldi.py:334-405)."""
    assert vtln_low_cutoff > low_freq, "be sure to set the vtln_low option higher than low_freq"
    assert vtln_high_cutoff < high_freq, "be sure to set the vtln_high option lower than high_freq [or negative]"
    lower = vtln_low_cutoff * max(1.0, vtln_warp_factor)
    upper = vtln_high_cutoff * min(1.0, vtln_warp_factor)
    slope = 1.0 / vtln_warp_factor
    f_lower, f_upper = slope * lower, slope * upper
    assert lower > low_freq and upper < high_freq
    slope_left = (f_lower - low_freq) / (lower - low_freq)
    slope_right = (high_freq - f_upper) / (high_freq - upper)
    out = torch.empty_like(freq)
    # the assignment order resolves the overlaps exactly as the reference's masks do
    top = torch.ge(freq, upper)
    out[top] = high_freq + slope_right * (freq[top] - high_freq)
    mid = torch.lt(freq, upper)
    out[mid] = slope * freq[mid]
    bottom = torch.lt(freq, lower)
    out[bottom] = low_freq + slope_left * (freq[bottom] - low_freq)
    outside = torch.lt(freq, low_freq) | torch.gt(freq, high_freq)
    out[outside] = freq[outside]
    return out


def vtln_warp_mel_freq(
    vtln_low_cutoff: float,
    vtln_high_cutoff: float,
    low_freq,
    high_freq: float,
    vtln_warp_factor: float,
    mel_freq: Tensor,
) -> Tensor:
    return mel_scale(
        vtln_warp_freq(vtln_low_cutoff, vtln_high_cutoff, low_freq, high_freq, vtln_warp_factor, inverse_mel_scale(mel_freq))
    )


def get_mel_banks(
    num_bins: int,
    window_length_padded: int,
    sample_freq: float,
    low_freq: float,
    high_freq: float,
    vtln_low: float,
    vtln_high: float,
    vtln_warp_factor: float,
) -> Tuple[Tensor, Tensor]:
    """``(bins (num_bins, padded/2), center_freqs)`` -- triangles in the mel domain (reference kaldi.py:436-511).
    Float32 on the CPU whatever the caller's device, like the reference."""
    assert num_bins > 3, "Must have at least 3 mel bins"
    assert window_length_padded % 2 == 0
    num_fft_bins = window_length_padded / 2
    nyquist = 0.5 * sample_freq
    if high_freq <= 0.0:
        high_freq += nyquist
    assert (
        (0.0 <= low_freq < nyquist) and (0.0 < high_freq <= nyquist) and (low_freq < high_freq)
    ), "Bad values in options: low-freq {} and high-freq {} vs. nyquist {}".format(low_freq, high_freq, nyquist)
    fft_bin_width = sample_freq / window_length_padded
    mel_lo, mel_hi = mel_scale_scalar(low_freq), mel_scale_scalar(high_freq)
    step = (mel_hi - mel_lo) / (num_bins + 1)  # num_bins + 1: the triangles overlap by half
    if vtln_high < 0.0:
        vtln_high += nyquist
    assert vtln_warp_factor == 1.0 or (
        (low_freq < vtln_low < high_freq) and (0.0 < vtln_high < high_freq) and (vtln_low < vtln_high)
    ), "Bad values in options: vtln-low {} and vtln-high {}, versus " "low-freq {} and high-freq {}".format(
        vtln_low, vtln_high, low_freq, high_freq
    )
    index = torch.arange(num_bins).unsqueeze(1)
    edges = [mel_lo + index * step, mel_lo + (index + 1.0) * step, mel_lo + (index + 2.0) * step]
    if vtln_warp_factor != 1.0:
        edges = [vtln_warp_mel_freq(vtln_low, vtln_high, low_freq, high_freq, vtln_warp_factor, e) for e in edges]
    left, center, right = edges
    center_freqs = inverse_mel_scale(center)
    mel = mel_scale(fft_bin_width * torch.arange(num_fft_bins)).unsqueeze(0)
    rising = (mel - left) / (center - left)
    falling = (right - mel) / (right - center)
    if vtln_warp_factor == 1.0:
        bins = torch.max(torch.zeros(1), torch.min(rising, falling))
    else:  # warping may reorder the edges: take each slope only on its own side
        bins = torch.zeros_like(rising)
        on_rise = torch.gt(mel, left) & torch.le(mel, center)
        on_fall = torch.gt(mel, center) & torch.lt(mel, right)
        bins[on_rise] = rising[on_rise]
        bins[on_fall] = falling[on_fall]
    return bins, center_freqs


# ---- constant tables ---------------------------------------------------------------------------------------------
def _next_power_of_2(x: int) -> int:
    return 1 if x == 0 else 2 ** (x - 1).bit_length()


def _feature_window_function(window_type: str, window_size: int, blackman_coeff: float, device, dtype) -> Tensor:
    """Symmetric (non-periodic) windows, reference kaldi.py:86-113."""
    if window_type == HANNING:
        return torch.hann_window(window_size, periodic=False, device=device, dtype=dtype)
    if window_type == HAMMING:
        return torch.hamming_window(window_size, periodic=False, alpha=0.54, beta=0.46, device=device, dtype=dtype)
    if window_type == POVEY:
        return torch.hann_window(window_size, periodic=False, device=device, dtype=dtype).pow(0.85)
    if window_type == RECTANGULAR:
        return torch.ones(window_size, device=device, dtype=dtype)
    if window_type == BLACKMAN:
        a = 2 * math.pi / (window_size - 1)
        n = torch.arange(window_size, device=device, dtype=dtype)
        return (blackman_coeff - 0.5 * torch.cos(a * n) + (0.5 - blackman_coeff) * torch.cos(2 * a * n)).to(
            device=device, dtype=dtype
        )
    raise Exception("Invalid window type " + window_type)


def _get_dct_matrix(num_ceps: int, num_mel_bins: int) -> Tensor:
    """(num_mel_bins, num_ceps): orthonormal DCT-II whose C0 column is the plain sqrt(1/n) sum (kaldi.py:648-658)."""
    dct = create_dct(num_mel_bins, num_mel_bins, "ortho")
    dct[:, 0] = math.sqrt(1 / float(num_mel_bins))
    return dct[:, :num_ceps]


def _get_lifter_coeffs(num_ceps: int, cepstral_lifter: float) -> Tensor:
    """1 + Q/2 sin(pi i / Q), i = 0 .. num_ceps-1 (kaldi.py:661-666)."""
    i = torch.arange(num_ceps)
    return 1.0 + 0.5 * cepstral_lifter * torch.sin(math.pi * i / cepstral_lifter)


def _window_properties(num_samples, sample_frequency, frame_shift, frame_length, round_to_power_of_two,
                       preemphasis_coefficient) -> Tuple[int, int, int]:
    """(window_shift, window_size, padded_window_size) with the reference's assertions (kaldi.py:126-151)."""
    window_shift = int(sample_frequency * frame_shift * MILLISECONDS_TO_SECONDS)
    window_size = int(sample_frequency * frame_length * MILLISECONDS_TO_SECONDS)
    padded_window_size = _next_power_of_2(window_size) if round_to_power_of_two else window_size
    assert 2 <= window_size <= num_samples, "choose a window size {} that is [2, {}]".format(window_size, num_samples)
    assert 0 < window_shift, "`window_shift` must be greater than 0"
    assert padded_window_size % 2 == 0, (
        "the padded `window_size` must be divisible by two." " use `round_to_power_of_two` or change `frame_length`"
    )
    assert 0.0 <= preemphasis_coefficient <= 1.0, "`preemphasis_coefficient` must be between [0,1]"
    assert sample_frequency > 0, "`sample_frequency` must be greater than zero"
    return window_shift, window_size, padded_window_size


# ---- device plans ------------------------------------------------------------------------------------------------
class _KaldiPlan:
    """Descriptor pair + prepared workspace(s) for one option set on one device."""

    def __init__(self, device, window: Tensor, padded: int, shift: int, use_power: bool, banks, finish):
        self.window = window.to(device)
        self.fb = None if banks is None else banks.to(device)
        n_mels = 0 if banks is None else banks.shape[1]
        desc = FrontendPlan.make_desc(padded, padded, shift, 0, False, "reflect", True, False, False,
                                      2.0 if use_power else 1.0, n_mels=n_mels)
        self.front = FrontendPlan(desc)
        self.ws = self.front.workspace(self.window, self.fb, None)
        self.finish = None
        if finish is not None:  # MFCC: (inputs, num_ceps) matrix applied by b200a_mfcc_finish
            self.matrix = finish.to(device)
            fdesc = FrontendPlan.make_desc(padded, padded, shift, 0, False, "reflect", True, False, False, 2.0,
                                           n_mels=finish.shape[0], n_mfcc=finish.shape[1])
            self.finish = FrontendPlan(fdesc)
            # this workspace only serves b200a_mfcc_finish; its filterbank slot is never read
            self.no_fb = torch.zeros(padded // 2 + 1, finish.shape[0], dtype=torch.float32, device=device)
            self.finish_ws = self.finish.workspace(self.window, self.no_fb, self.matrix)


_PLANS: Dict[tuple, _KaldiPlan] = {}


def _launch(flat: Tensor, plan: _KaldiPlan, kd_lists, stage: int, frames: int, width: int, stride: int,
            subtract_mean: bool) -> Tensor:
    """The forward launches: b200a_kaldi_run [+ b200a_mfcc_finish] [+ b200a_subtract_column_mean]."""
    out = _ops.kaldi_run(flat, plan.ws, *plan.front._packed_desc(), *kd_lists, stage, frames, width, stride)
    if plan.finish is not None:
        out = plan.finish.mfcc_finish(plan.finish_ws, out, None, 1, None)
    if subtract_mean:
        dev = out.device
        with torch.cuda.device(dev):
            rc = _lib.lib().b200a_subtract_column_mean(out.data_ptr(), out.shape[0], out.shape[1], out.shape[2],
                                                       _stream_ptr(dev))
        _lib.check(rc, "subtract_column_mean")
    return out


class _KaldiFunction(torch.autograd.Function):
    """The Kaldi features of the packed (rows, L) waveform with exactly the no-grad launches (so the output is
    bit-identical to the no-grad call), and their waveform gradient: the column-mean subtraction (symmetric, its own
    adjoint), the MFCC finishing matrix transposed (b200audio::apply_fbank_backward), then b200audio::kaldi_backward.
    The waveform goes through save_for_backward, so in-place edits of it are detected; the plan (workspace, finishing
    matrix) is held, so its eviction from the cache cannot free what backward reads."""

    @staticmethod
    def forward(ctx, flat, plan, kd_lists, stage, frames, width, stride, subtract_mean):
        out = _launch(flat, plan, kd_lists, stage, frames, width, stride, subtract_mean)
        ctx.save_for_backward(flat)
        ctx.plan, ctx.args = plan, (kd_lists, stage, frames, width, stride, subtract_mean)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        (flat,) = ctx.saved_tensors
        plan = ctx.plan
        kd_lists, stage, frames, width, stride, subtract_mean = ctx.args
        g = grad_out
        if subtract_mean:
            g = g.contiguous().clone()
            dev = g.device
            with torch.cuda.device(dev):
                rc = _lib.lib().b200a_subtract_column_mean(g.data_ptr(), g.shape[0], g.shape[1], g.shape[2],
                                                           _stream_ptr(dev))
            _lib.check(rc, "subtract_column_mean")
        if plan.finish is not None:  # one row of rows * T frames: the op's row limit never applies
            rows = g.shape[0]
            g = _ops.apply_fbank_backward(g.contiguous().reshape(1, rows * frames, g.shape[2]), plan.matrix)
            g = g.reshape(rows, frames, width)
        grad = _ops.kaldi_backward(flat, plan.ws, *plan.front._packed_desc(), *kd_lists, stage, stride, g)
        return grad, None, None, None, None, None, None, None


def _select_channel(waveform: Tensor, channel: int) -> Tensor:
    channel = max(channel, 0)
    assert channel < waveform.size(0), "Invalid channel {} for size {}".format(channel, waveform.size(0))
    return waveform[channel : channel + 1, :]


def _features(kind: str, rows: Tensor, o: dict) -> Tensor:
    """rows (B, n) -> (B, m, width) Kaldi features of `kind` for the option dict `o` (all keys of the public API)."""
    _require_cuda_f32(rows, "waveform")
    grad = _wants_grad(rows, (), is_kaldi_differentiable)
    if not grad:
        _no_autograd(rows)
    if o["dither"] != 0.0:
        raise RuntimeError(
            "audio_b200.compliance.kaldi: dither != 0 is not implemented (the reference draws the noise with "
            "torch.randn per frame element, which cannot be reproduced); pass dither=0.0"
        )
    assert o["window_type"] in WINDOWS, "Invalid window type " + str(o["window_type"])
    num_samples = rows.shape[-1]
    shift, size, padded = _window_properties(num_samples, o["sample_frequency"], o["frame_shift"], o["frame_length"],
                                             o["round_to_power_of_two"], o["preemphasis_coefficient"])
    dev = rows.device
    if num_samples < o["min_duration"] * o["sample_frequency"]:
        return torch.empty(0, device=dev, dtype=rows.dtype)
    lib = _lib.lib()
    frames = lib.b200a_kaldi_num_frames(num_samples, size, shift, int(bool(o["snip_edges"])))
    mel = kind != "spectrogram"
    use_energy = True if kind == "spectrogram" else bool(o["use_energy"])
    n_mels = int(o["num_mel_bins"]) if mel else 0
    num_ceps = int(o["num_ceps"]) if kind == "mfcc" else 0
    if kind == "mfcc":
        assert num_ceps <= n_mels, "num_ceps cannot be larger than num_mel_bins: %d vs %d" % (num_ceps, n_mels)
    htk = bool(o.get("htk_compat", False))

    key = (kind, str(dev), size, shift, padded, o["window_type"], float(o["blackman_coeff"]), n_mels,
           float(o["sample_frequency"]), float(o.get("low_freq", 0.0)), float(o.get("high_freq", 0.0)),
           float(o.get("vtln_low", 0.0)), float(o.get("vtln_high", 0.0)), float(o.get("vtln_warp", 1.0)),
           bool(o.get("use_power", True)), num_ceps, float(o.get("cepstral_lifter", 0.0)), htk, use_energy)
    plan = _PLANS.get(key)
    if plan is None:
        window = torch.zeros(padded, dtype=torch.float32)
        window[:size] = _feature_window_function(o["window_type"], size, o["blackman_coeff"], torch.device("cpu"),
                                                 torch.float32)
        banks = finish = None
        if mel:
            bins, _ = get_mel_banks(n_mels, padded, o["sample_frequency"], o["low_freq"], o["high_freq"], o["vtln_low"],
                                    o["vtln_high"], o["vtln_warp"])
            # (padded/2 + 1, n_mels): transposed for the frame-major contraction; the Nyquist bin gets no weight
            banks = torch.nn.functional.pad(bins.to(torch.float32), (0, 1), mode="constant", value=0).T.contiguous()
        if kind == "mfcc":
            mat = _get_dct_matrix(num_ceps, n_mels).clone()
            if o["cepstral_lifter"] != 0.0:
                mat = mat * _get_lifter_coeffs(num_ceps, o["cepstral_lifter"]).unsqueeze(0)
            if use_energy:  # C0 is replaced by the log energy, which rides along as one more input column
                mat[:, 0] = 0.0
                route = torch.zeros(1, num_ceps)
                route[0, 0] = 1.0
                mat = torch.cat((mat, route), dim=0)
            if htk:  # HTK order: C1 .. C(n-1), then C0 (x sqrt 2 when it is a cepstrum, kaldi.py:800-808)
                first = mat[:, :1] if use_energy else mat[:, :1] * math.sqrt(2)
                mat = torch.cat((mat[:, 1:], first), dim=1)
            finish = mat.to(torch.float32).contiguous()
        plan = _KaldiPlan(dev, window, padded, shift, bool(o.get("use_power", True)) if mel else True, banks, finish)
        _PLANS[key] = plan
        if len(_PLANS) > 32:  # bounded: drop the oldest plan (dict preserves insertion order)
            _PLANS.pop(next(iter(_PLANS)))

    # where the kernel puts things: [energy |] values, or values [| energy]
    if kind == "spectrogram":
        values, width, col0, energy_col, use_log = padded // 2 + 1, padded // 2 + 1, 0, 0, True
    elif kind == "fbank":
        values = n_mels
        width = n_mels + int(use_energy)
        col0 = 1 if (use_energy and not htk) else 0
        energy_col = -1 if not use_energy else (n_mels if htk else 0)
        use_log = bool(o["use_log_fbank"])
    else:  # mfcc: log-mel energies (+ the energy column the finishing matrix routes to C0)
        values = n_mels
        width = n_mels + int(use_energy)
        col0 = 0
        energy_col = n_mels if use_energy else -1
        use_log = True
    kd = _lib.KaldiDesc()
    kd.window_size, kd.window_shift, kd.padded_size = size, shift, padded
    kd.snip_edges, kd.remove_dc_offset = int(bool(o["snip_edges"])), int(bool(o["remove_dc_offset"]))
    kd.preemphasis = float(o["preemphasis_coefficient"])
    kd.energy_mode = 0 if energy_col < 0 else (1 if o["raw_energy"] else 2)
    kd.energy_floor = float(o["energy_floor"])
    kd.energy_col, kd.out_width, kd.out_col0, kd.use_log = energy_col, width, col0, int(use_log)

    flat, stride = pack_rows(rows)
    batch = flat.shape[0]
    stage = _lib.STAGE_MEL if mel else _lib.STAGE_POWER
    if frames > 0 and batch > 0:
        args = (flat, plan, _ops.pack(kd), stage, frames, width, stride, bool(o["subtract_mean"]))
        return _KaldiFunction.apply(*args) if grad else _launch(*args)
    with torch.cuda.device(dev):
        out = torch.empty((batch, frames, width), dtype=torch.float32, device=dev)
    if kind == "mfcc" and frames > 0:
        out = plan.finish.mfcc_finish(plan.finish_ws, out, None, 1, None)
    return out


def _single(kind: str, waveform: Tensor, o: dict) -> Tensor:
    out = _features(kind, _select_channel(waveform, o.pop("channel")), o)
    return out[0] if out.dim() == 3 else out


# ---- public API (reference signatures) ---------------------------------------------------------------------------
def spectrogram(
    waveform: Tensor,
    blackman_coeff: float = 0.42,
    channel: int = -1,
    dither: float = 0.0,
    energy_floor: float = 1.0,
    frame_length: float = 25.0,
    frame_shift: float = 10.0,
    min_duration: float = 0.0,
    preemphasis_coefficient: float = 0.97,
    raw_energy: bool = True,
    remove_dc_offset: bool = True,
    round_to_power_of_two: bool = True,
    sample_frequency: float = 16000.0,
    snip_edges: bool = True,
    subtract_mean: bool = False,
    window_type: str = POVEY,
) -> Tensor:
    """``(c, n) -> (m, padded_window_size // 2 + 1)`` log power spectrum with the log energy in column 0
    (Kaldi ``compute-spectrogram-feats``; reference kaldi.py:229-316)."""
    return _single("spectrogram", waveform, dict(locals(), waveform=None))


def fbank(
    waveform: Tensor,
    blackman_coeff: float = 0.42,
    channel: int = -1,
    dither: float = 0.0,
    energy_floor: float = 1.0,
    frame_length: float = 25.0,
    frame_shift: float = 10.0,
    high_freq: float = 0.0,
    htk_compat: bool = False,
    low_freq: float = 20.0,
    min_duration: float = 0.0,
    num_mel_bins: int = 23,
    preemphasis_coefficient: float = 0.97,
    raw_energy: bool = True,
    remove_dc_offset: bool = True,
    round_to_power_of_two: bool = True,
    sample_frequency: float = 16000.0,
    snip_edges: bool = True,
    subtract_mean: bool = False,
    use_energy: bool = False,
    use_log_fbank: bool = True,
    use_power: bool = True,
    vtln_high: float = -500.0,
    vtln_low: float = 100.0,
    vtln_warp: float = 1.0,
    window_type: str = POVEY,
) -> Tensor:
    """``(c, n) -> (m, num_mel_bins + use_energy)`` (Kaldi ``compute-fbank-feats``; reference kaldi.py:514-645)."""
    return _single("fbank", waveform, dict(locals(), waveform=None))


def mfcc(
    waveform: Tensor,
    blackman_coeff: float = 0.42,
    cepstral_lifter: float = 22.0,
    channel: int = -1,
    dither: float = 0.0,
    energy_floor: float = 1.0,
    frame_length: float = 25.0,
    frame_shift: float = 10.0,
    high_freq: float = 0.0,
    htk_compat: bool = False,
    low_freq: float = 20.0,
    num_ceps: int = 13,
    min_duration: float = 0.0,
    num_mel_bins: int = 23,
    preemphasis_coefficient: float = 0.97,
    raw_energy: bool = True,
    remove_dc_offset: bool = True,
    round_to_power_of_two: bool = True,
    sample_frequency: float = 16000.0,
    snip_edges: bool = True,
    subtract_mean: bool = False,
    use_energy: bool = False,
    vtln_high: float = -500.0,
    vtln_low: float = 100.0,
    vtln_warp: float = 1.0,
    window_type: str = POVEY,
) -> Tensor:
    """``(c, n) -> (m, num_ceps)`` (Kaldi ``compute-mfcc-feats``; reference kaldi.py:669-813)."""
    return _single("mfcc", waveform, dict(locals(), waveform=None, use_power=True, use_log_fbank=True))


# ---- batched extensions: (batch, time) -> (batch, frames, features), same keyword arguments --------------------
def _batched(kind: str, fn, waveforms: Tensor, kwargs: dict) -> Tensor:
    import inspect

    o = {k: v.default for k, v in inspect.signature(fn).parameters.items() if v.default is not inspect.Parameter.empty}
    unknown = set(kwargs) - set(o)
    if unknown:
        raise TypeError(f"{fn.__name__}_batch() got unexpected keyword arguments {sorted(unknown)}")
    o.update(kwargs)
    o.pop("channel")
    if kind == "mfcc":
        o.update(use_power=True, use_log_fbank=True)
    if waveforms.dim() != 2:
        raise ValueError(f"expected (batch, time), got a tensor of shape {tuple(waveforms.shape)}")
    return _features(kind, waveforms, o)


def spectrogram_batch(waveforms: Tensor, **kwargs) -> Tensor:
    return _batched("spectrogram", spectrogram, waveforms, kwargs)


def fbank_batch(waveforms: Tensor, **kwargs) -> Tensor:
    return _batched("fbank", fbank, waveforms, kwargs)


def mfcc_batch(waveforms: Tensor, **kwargs) -> Tensor:
    return _batched("mfcc", mfcc, waveforms, kwargs)
