"""The shared-memory Stockham kernels of csrc/frontend_generic.cu at their plan limits, against the float64 oracle.

These kernels run every n_fft outside {256, 512, 1024, 2048}, two-sided output, complex output at 2048 and above,
more than 512 mel filters, and every inverse STFT at n_fft >= 2048 or not a power of two (so Griffin-Lim at 2048).
Covered here: which kernel a call launches, n_fft by factorisation class (radix 2/4, 3, 5 towers, mixed sizes, primes
on the direct-sum stage, repeated direct stages, 4096 / 8192), frame counts around the CTA tile of 2 * pairs frames,
the framing options, layouts and batches, the inverse STFT and Griffin-Lim.

The bar is scaled_tol_close (rel 1e-4) applied to each row of the batch.  The two frames of a pair share one complex
FFT, so a frame's float32 error grows with its partner's magnitude; pairs never cross rows, and no test here puts a
per-frame bar on a frame next to a much louder partner."""
import time
import warnings

import numpy as np
import pytest
import torch
from conftest import scaled_tol_close
from test_inverse import _stable

import audio_b200.functional as F
import audio_b200.transforms as T
from oracle import frontend_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def randn(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed))


def rows_close(got, exp, what="", rel=1e-4):
    """scaled_tol_close on each row (leading index) by itself: a quiet row is held to its own scale, an all-zero row
    to exactly 0."""
    got = got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got)
    exp = np.asarray(exp)
    assert got.shape == exp.shape, f"{what}: shape {got.shape} vs {exp.shape}"
    assert np.isfinite(got).all(), f"{what}: non-finite output"  # a NaN would pass the |err| <= tol test
    got, exp = got.reshape(exp.shape[0], -1), exp.reshape(exp.shape[0], -1)
    for r in range(exp.shape[0]):
        scaled_tol_close(got[r], exp[r], rel, what=f"{what} row {r}")


def stockham_pairs(n_fft, frames):
    """Frame pairs per CTA as launch_stockham (csrc/frontend_generic.cu) chooses them: the 2 * pairs frames' ping-pong
    buffers within 48 KB, 1 to 8 pairs, and no pair wholly past the last frame."""
    pairs = min(max(49152 // (16 * n_fft), 1), 8)
    while pairs > 1 and 2 * (pairs - 1) >= frames:
        pairs -= 1
    return pairs


def length_for(frames, n_fft, hop, center):
    """A signal length that torch.stft frames into exactly `frames` frames, with hop // 2 samples after the last."""
    lead = 2 * (n_fft // 2) if center else 0
    length = n_fft - lead + (frames - 1) * hop + hop // 2
    assert O.num_frames(length, n_fft, hop, center) == frames
    return length


def tile_frame_counts(n_fft):
    """1, 2, one below / at / one above the full tile of 2 * pairs frames, and a long odd count with a ragged tile."""
    p = stockham_pairs(n_fft, 1 << 30)
    return sorted({1, 2, 2 * p - 1, 2 * p, 2 * p + 1, 14 * p + 3})


# ---- a. which kernels a call launches -------------------------------------------------------------------------------
PROFILER_PAD = 0.02
def launched_kernels(fn, expected):
    """Names of the CUDA kernels `fn` launches, from torch.profiler.  A profiler session now and then comes back
    without some or all of its kernel records, more often for short sessions late in a long test run: each session
    is padded with PROFILER_PAD seconds of idle time at both ends, the deterministic call runs three times per
    session, and in up to ten sessions, until every name in `expected` was recorded."""
    fn()  # workspace and plan set-up stay outside the recorded call
    for attempt in range(10):
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            time.sleep(PROFILER_PAD)
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            time.sleep(PROFILER_PAD)
        names = {ev.name for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA}
        names = {n for n in names if "Memcpy" not in n and "Memset" not in n}
        if all(any(e in n for n in names) for e in expected):
            break
    print(f"profiler sessions: {attempt + 1}")
    return names


FORWARD_PINS = {
    "400": lambda: T.Spectrogram(n_fft=400),
    "97": lambda: T.Spectrogram(n_fft=97, hop_length=24),
    "4096": lambda: T.Spectrogram(n_fft=4096),
    "8192": lambda: T.Spectrogram(n_fft=8192),
    "2048-complex": lambda: T.Spectrogram(n_fft=2048, power=None),
    "512-twosided": lambda: T.Spectrogram(n_fft=512, onesided=False),
    "1024-520mels": lambda: T.MelSpectrogram(16000, n_fft=1024, hop_length=256, n_mels=520),
}


@pytest.mark.parametrize("case", list(FORWARD_PINS))
def test_forward_runs_the_generic_kernel(case):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")  # empty mel filters at 520 mels
        mod = FORWARD_PINS[case]().to(DEV)
    x = randn((2, 20000), 1).to(DEV)
    names = launched_kernels(lambda: mod(x), ["stft_generic_kernel"])
    assert any("stft_generic_kernel" in n for n in names), names
    assert not any("stft_pow2" in n or "stft2048" in n for n in names), names


@pytest.mark.parametrize("n_fft", [2048, 600, 77])
def test_inverse_runs_the_stockham_frame_stage(n_fft):
    spec = torch.complex(randn((2, n_fft // 2 + 1, 9), 2), randn((2, n_fft // 2 + 1, 9), 3)).to(DEV)
    inv = T.InverseSpectrogram(n_fft=n_fft, hop_length=n_fft // 4).to(DEV)
    names = launched_kernels(lambda: inv(spec), ["istft_frames_kernel", "istft_ola_kernel"])
    assert any("istft_frames_kernel" in n for n in names) and any("istft_ola_kernel" in n for n in names), names
    assert not any("pow2" in n for n in names), names


# ---- b. sizes by factorisation class --------------------------------------------------------------------------------
SIZES = {
    "small": [2, 3, 4, 5, 8, 16, 32, 64, 128],
    "radix3-5": [243, 729, 2187, 125, 625, 3125],
    "mixed": [210, 882, 960, 1200, 2310],
    "prime": [13, 97, 251, 1021, 4093, 8191],
    "direct-repeat": [1331, 2401],
    "pow2-large": [4096, 8192],
}
TWO_SIDED = {2, 3, 5, 16, 125, 243, 13, 97, 210, 1331, 4096}


@pytest.mark.parametrize("n_fft", [pytest.param(n, id=f"{cls}-{n}") for cls, ns in SIZES.items() for n in ns])
def test_sizes_by_factorisation(n_fft):
    hop = max(1, n_fft // 4)
    # the direct-sum stage costs n_fft * R per frame pair: few frames at the large primes
    frames = 5 if n_fft > 4000 else 6 * stockham_pairs(n_fft, 1 << 30) + 1
    length = length_for(frames, n_fft, hop, True)
    x = randn((2, length), n_fft)
    xd = x.to(DEV)
    w = torch.hann_window(n_fft).double().numpy()
    for power, onesided in [(None, True), (2.0, True)] + ([(None, False)] if n_fft in TWO_SIDED else []):
        got = T.Spectrogram(n_fft=n_fft, hop_length=hop, power=power, onesided=onesided).to(DEV)(xd)
        exp = O.spectrogram(x.numpy(), 0, w, n_fft, hop, n_fft, power, onesided=onesided)
        assert exp.shape[-1] == frames
        rows_close(got, exp, f"n_fft={n_fft} power={power} onesided={onesided}")


def test_largest_size_plus_one_is_refused():
    x = randn((1, 20000), 0).to(DEV)
    with pytest.raises(RuntimeError, match="not supported"):
        T.Spectrogram(n_fft=8193).to(DEV)(x)
    with pytest.raises(RuntimeError, match="not supported"):
        F.spectrogram(x, 0, torch.hann_window(8193, device=DEV), 8193, 2048, 8193, None, False)
    spec = torch.zeros(1, 4097, 4, dtype=torch.complex64, device=DEV)
    with pytest.raises(RuntimeError, match="not supported"):
        T.InverseSpectrogram(n_fft=8193, hop_length=2048).to(DEV)(spec)


# ---- c. tile tails --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_fft", [13, 97, 400, 600, 1021, 1200, 2310])
@pytest.mark.parametrize("hop_kind", ["quarter", "odd", "beyond"])
def test_tile_tails(n_fft, hop_kind):
    """Frame counts around the CTA tile, three rows, complex output (both frames of a pair un-packed).  A hop larger
    than n_fft leaves samples between frames unread.  Reflect padding needs more than n_fft // 2 samples, so the
    centred calls pad with zeros."""
    hop = {"quarter": max(1, n_fft // 4), "odd": (n_fft // 3) | 1, "beyond": n_fft + n_fft // 3 + 1}[hop_kind]
    w = torch.hann_window(n_fft).double().numpy()
    for frames in tile_frame_counts(n_fft):
        for center in (False, True):
            length = length_for(frames, n_fft, hop, center)
            x = randn((3, length), n_fft + frames + hop)
            mod = T.Spectrogram(n_fft=n_fft, hop_length=hop, power=None, center=center, pad_mode="constant").to(DEV)
            exp = O.spectrogram(x.numpy(), 0, w, n_fft, hop, n_fft, None, center=center, pad_mode="constant")
            rows_close(mod(x.to(DEV)), exp, f"n_fft={n_fft} hop={hop} T={frames} center={center}")


# ---- d. framing options and features at generic sizes --------------------------------------------------------------
def _option_cases(n_fft):
    win = 301 if n_fft == 400 else 80  # n_fft - win odd: the window sits one sample left of centre
    cases = [dict(pad_mode=m, center=c, power=None) for m in ("reflect", "constant", "replicate", "circular")
             for c in (True, False)]
    return cases + [
        dict(pad=13, power=None), dict(pad=7, pad_mode="replicate"),
        dict(win_length=win, hop_length=n_fft // 4, power=None), dict(win_length=win, hop_length=n_fft // 4 + 1),
        dict(normalized=True), dict(normalized="frame_length", power=None), dict(normalized="window", power=1.0),
        dict(power=1.0), dict(power=3.0),
    ]


@pytest.mark.parametrize("n_fft", [400, 97])
def test_framing_options(n_fft):
    x = randn((2, 9 * n_fft + 17), n_fft)
    xd = x.to(DEV)
    for kw in _option_cases(n_fft):
        win = kw.get("win_length", n_fft)
        hop = kw.get("hop_length", win // 2)
        got = T.Spectrogram(n_fft=n_fft, **kw).to(DEV)(xd)
        exp = O.spectrogram(x.numpy(), kw.get("pad", 0), torch.hann_window(win).double().numpy(), n_fft, hop, win,
                            kw.get("power", 2.0), kw.get("normalized", False), kw.get("center", True),
                            kw.get("pad_mode", "reflect"))
        rows_close(got, exp, f"n_fft={n_fft} {kw}")


@pytest.mark.parametrize("n_fft,n_mels", [(97, 16), (401, 40)])
def test_features_at_odd_sizes(n_fft, n_mels):
    """MelSpectrogram, MFCC on the dB and the log-mel paths, and LFCC, with the modules' own filterbank and DCT."""
    x = randn((3, 12 * n_fft + 5), n_fft + n_mels)
    xd = x.to(DEV)
    melkw = dict(n_fft=n_fft, hop_length=n_fft // 4, n_mels=n_mels)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")  # the narrowest mel filters may hold no bin
        mel = T.MelSpectrogram(16000, **melkw).to(DEV)
        mfccs = [T.MFCC(16000, n_mfcc=13, log_mels=lm, melkwargs=melkw).to(DEV) for lm in (False, True)]
    fb = mel.mel_scale.fb.double().cpu().numpy()
    rows_close(mel(xd), O.mel_spectrogram(x.numpy(), 16000, fb=fb, **melkw), f"mel n_fft={n_fft}")
    for mf in mfccs:
        exp = O.mfcc(x.numpy(), 16000, 13, "ortho", mf.log_mels, melkw,
                     fb=mf.MelSpectrogram.mel_scale.fb.double().cpu().numpy(), dct=mf.dct_mat.double().cpu().numpy())
        rows_close(mf(xd), exp, f"mfcc n_fft={n_fft} log_mels={mf.log_mels}")
    speckw = dict(n_fft=n_fft, hop_length=n_fft // 4)
    lf = T.LFCC(16000, n_filter=2 * n_mels, n_lfcc=12, speckwargs=speckw).to(DEV)
    exp = O.lfcc(x.numpy(), 16000, 2 * n_mels, n_lfcc=12, speckwargs=speckw,
                 filter_mat=lf.filter_mat.double().cpu().numpy(), dct=lf.dct_mat.double().cpu().numpy())
    rows_close(lf(xd), exp, f"lfcc n_fft={n_fft}")


# ---- e. layouts and batches -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_fft", [97, 400, 1021])
def test_layouts_and_batches(n_fft):
    hop = n_fft // 4
    w = torch.hann_window(n_fft).double().numpy()
    mod = T.Spectrogram(n_fft=n_fft, hop_length=hop, power=None).to(DEV)
    length = length_for(2 * stockham_pairs(n_fft, 1 << 30) + 3, n_fft, hop, True)

    def oracle(x):
        return O.spectrogram(np.asarray(x, dtype=np.float64), 0, w, n_fft, hop, n_fft, None)

    x1 = randn((length,), 1)
    got = mod(x1.to(DEV))
    rows_close(got[None], oracle(x1.numpy())[None], "1-D")
    x3 = randn((2, 3, length), 2)
    got = mod(x3.to(DEV))
    assert tuple(got.shape[:2]) == (2, 3)
    rows_close(got.reshape(6, *got.shape[2:]), oracle(x3.numpy()).reshape(6, *got.shape[2:]), "3-D")
    big = randn((8, length + 64), 3).to(DEV)
    for view in (big[:, 3:3 + length], big[::2, 1:1 + length]):  # offset base, row pitch > length, every other row
        got = mod(view)
        rows_close(got, oracle(view.cpu().numpy()), "view")
        assert torch.equal(got, mod(view.contiguous()))
    # frames pair only within a row: each row is held to its own scale, the silent row is exactly 0
    x = randn((4, length), 4)
    x[0] *= 1e3
    x[2] *= 1e-3
    x[3] = 0
    got = mod(x.to(DEV))
    rows_close(got, oracle(x.numpy()), "scaled rows")
    assert torch.count_nonzero(got[3]).item() == 0
    for r in range(4):
        assert torch.equal(mod(x[r:r + 1].to(DEV)), got[r:r + 1]), r


# ---- f. inverse STFT ------------------------------------------------------------------------------------------------
INVERSE_SIZES = [2048, 4096, 8192, 600, 882, 1200, 2310, 77, 401, 2187]


def _inverse_cases(n_fft):
    """(frames, center, win_length, normalized, length - default length or None, zero tail) at the pair boundaries.

    A centred call returns n_fft // 2 samples less at each end than the frames cover.  A zero tail (a `length` past the
    last frame) needs a window whose overlap-added square stays above 1e-11 up to that frame's last sample: the
    Hamming window of the uncentred calls, not a zero-padded short window or a Hann window at n_fft >= 2048."""
    p = stockham_pairs(n_fft, 1 << 30)
    hop = n_fft // 4
    win = n_fft * 3 // 4
    win -= (n_fft - win) % 2 == 0  # odd difference: the window sits one sample left of centre
    return [
        (2 * p + 1, True, n_fft, False, None, False),
        (max(2, 2 * p - 1), True, n_fft, "frame_length", -(hop // 2 + 1), False),  # shorter than the default
        (2 * p, True, win, True, hop + 3, False),  # longer than the default, inside what the frames cover
        (2 * p + 1, False, n_fft, "window", None, False),
        (2 * p, False, n_fft, True, hop + 3, True),  # past the last frame: a zero tail of hop + 3 samples
    ]


@pytest.mark.parametrize("n_fft", INVERSE_SIZES)
def test_inverse_against_oracle(n_fft):
    """Inconsistent spectrograms (a forward STFT of noise times 1 + 0.1 noise), on output positions whose window
    envelope does not vanish."""
    hop = n_fft // 4
    rng = np.random.default_rng(n_fft)
    for frames, center, win, normalized, delta, tail in _inverse_cases(n_fft):
        # centred calls use the Hann window; uncentred ones a Hamming window, whose envelope stays positive at the ends
        window = (torch.hann_window if center else torch.hamming_window)(win)
        w = window.double().numpy()
        x = rng.standard_normal((2, length_for(frames, n_fft, hop, center)))
        spec = O.spectrogram(x, 0, w, n_fft, hop, win, None, normalized, center, "constant")
        spec = (spec * (1 + 0.1 * rng.standard_normal(spec.shape))).astype(np.complex64)
        expected = n_fft + hop * (frames - 1)
        start = n_fft // 2 if center else 0
        default = expected - 2 * start if center else expected
        length = None if delta is None else default + delta
        out_len = default if length is None else length
        inv = T.InverseSpectrogram(n_fft=n_fft, win_length=win, hop_length=hop, normalized=normalized, center=center,
                                   window_fn=torch.hann_window if center else torch.hamming_window).to(DEV)
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            got = inv(torch.from_numpy(spec).to(DEV), length).cpu().numpy()
        what = f"n_fft={n_fft} T={frames} center={center} win={win} normalized={normalized} length={length}"
        assert (start + out_len > expected) == tail, what
        assert any("padded with zeros" in str(c.message) for c in caught) == tail, what
        exp = O.inverse_spectrogram(spec, length, 0, w, n_fft, hop, win, normalized, center)
        assert got.shape == exp.shape == (2, out_len)
        ok = _stable(dict(n_fft=n_fft, win=win, center=center, hop=hop, pad=0), frames, out_len)
        rows_close(got[:, ok], exp[:, ok], what)
        if tail:
            assert got.shape[1] - (expected - start) == hop + 3 and not got[:, expected - start:].any(), what


@pytest.mark.parametrize("n_fft", INVERSE_SIZES)
def test_inverse_round_trip(n_fft):
    hop = n_fft // 4
    frames = 2 * stockham_pairs(n_fft, 1 << 30) + 1
    length = length_for(frames, n_fft, hop, True)
    x = randn((2, length), n_fft)
    fwd = T.Spectrogram(n_fft=n_fft, hop_length=hop, power=None).to(DEV)
    inv = T.InverseSpectrogram(n_fft=n_fft, hop_length=hop).to(DEV)
    spec = fwd(x.to(DEV))
    assert spec.shape[-1] == frames
    rows_close(inv(spec, length), x.numpy(), f"n_fft={n_fft}")


# ---- g. Griffin-Lim -------------------------------------------------------------------------------------------------
# max |GPU - float64| / max |float64| after n_iter float32 iterations.  Measured on an H100 80GB HBM3 (700 W): at most
# 1.0e-4 (n_fft 1200, 6 iterations, momentum 0.99), 1.1e-5 at 2048 and 3.0e-5 at 401; the bar is 5x the largest.
# Momentum amplifies the round-off of bins whose rebuilt magnitude is near 0, where the phase is ill-conditioned.
GL_BAR = 5e-4


@pytest.mark.parametrize("n_fft,n_iter,momentum", [(2048, 8, 0.99), (2048, 4, 0.0), (1200, 6, 0.99), (1200, 8, 0.0),
                                                   (401, 8, 0.99), (401, 5, 0.0)])
def test_griffinlim_against_oracle(n_fft, n_iter, momentum):
    hop = n_fft // 4
    length = 12 * hop + 7
    x = randn((2, length), n_fft + n_iter)
    w = torch.hann_window(n_fft).double().numpy()
    spec = O.spectrogram(x.numpy(), 0, w, n_fft, hop, n_fft, 2.0).astype(np.float32)
    gl = T.GriffinLim(n_fft=n_fft, n_iter=n_iter, hop_length=hop, power=2.0, momentum=momentum, length=length,
                      rand_init=False).to(DEV)
    got = gl(torch.from_numpy(spec).to(DEV)).cpu().numpy()
    exp = O.griffinlim(spec, w, n_fft, hop, n_fft, 2.0, n_iter, momentum, length)
    assert got.shape == exp.shape == (2, length)
    ratio = np.abs(got - exp).max() / np.abs(exp).max()
    print(f"griffinlim n_fft={n_fft} n_iter={n_iter} momentum={momentum}: {ratio:.3e}")
    assert ratio < GL_BAR
