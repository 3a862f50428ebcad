"""The banded TF32x3 mel contraction and the cepstral finish at the limits of their plans, against the float64 oracle.

The mel plan (prepare_mma_kernel) cuts the filterbank into groups of 8 filters and hands them to contraction warps; past
64 groups (512 filters) the generic kernel runs, past the shared-memory fragment reserve (100 / 112 / 112 / 136 k-steps
at n_fft 1024 / 512 / 256 / 2048) the fragments are read from global memory, and the n_fft 2048 kernel lists at most 32
groups per contraction warp.  Custom banks (all zero, one live filter, interior zero runs, negative weights, a few
full-band groups among many empty or one-step ones) reach corners real banks rarely do.  The finish picks one of four
kernels from n_mfcc, n_mels and the clamp; the mel gradient runs fused while its upstream rows fit in shared memory.

Every case also checks, under torch.profiler, that the kernel it was written for ran, so that a change of a dispatch
threshold cannot quietly move a case off its path.  Outputs are allocated over a block filled with NaN first, so a
column the kernel never stores is caught even when the allocator would have handed out zeros."""
import os
import re
import warnings

import numpy as np
import pytest
import torch
from conftest import GOLDEN, assert_close, scaled_tol_close

import audio_b200
import audio_b200.compliance.kaldi as K
import audio_b200.transforms as T
from oracle import frontend_oracle as O
from oracle import kaldi_oracle as KO

import grad_oracle as V

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NFFTS = [256, 512, 1024, 2048]
MEL_KERNEL = {256: "stft_pow2_mel_kernel", 512: "stft_pow2_mel_kernel", 1024: "stft_pow2_mel_kernel",
              2048: "stft2048_mel_kernel"}
FRAG_RESERVE = {256: 112, 512: 112, 1024: 100, 2048: 136}  # k-steps of fragments the mel kernel keeps in shared memory


def randn(rows, length, seed):
    return torch.randn(rows, length, generator=torch.Generator().manual_seed(seed))


def launched(fn, before=lambda: None):
    """before(), then fn() under torch.profiler: its result and the names of the CUDA kernels it launched.  Now and then
    the profiler hands back a session without any kernel record; the pair is then run again (fn is deterministic)."""
    for _ in range(3):
        before()
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        if names:
            return out, names
    raise AssertionError("torch.profiler recorded no CUDA kernel in 3 sessions: the path assertions cannot be checked")


def ran(names, kernel):
    """Whether a kernel of this name (template arguments included, if given) is among the launched ones."""
    pat = re.compile(r"(?<![\w])" + re.escape(kernel) + r"(?![\w])")
    return any(pat.search(n) for n in names)


def assert_ran(names, kernel, absent=()):
    assert ran(names, kernel), f"{kernel} did not run; launched: {sorted(set(names))}"
    for k in absent:
        assert not ran(names, k), f"{k} ran; launched: {sorted(set(names))}"


def poisoned(fn, *numels):
    """fn() once to build its plan and workspace, then again with the caching allocator's free blocks of each output
    size (float32 elements) filled with NaN: returns the second result and the kernels it launched."""
    fn()

    def poison():
        blocks = [torch.full((n,), float("nan"), device=DEV) for n in numels]
        del blocks

    return launched(fn, poison)


def plan_steps(fb):
    """k-steps of the mel plan: per group of 8 filters, the 8-bin steps from its first to its last live bin."""
    total = 0
    for t in range((fb.shape[1] + 7) // 8):
        live = np.nonzero(np.any(fb[:, 8 * t : 8 * t + 8] != 0, axis=1))[0]
        if live.size:
            total += (live[-1] + 1 - (live[0] & ~7) + 7) // 8
    return total


def mel_module(n_fft, n_mels, fb=None, power=2.0):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")  # banks with all-zero filters warn
        m = T.MelSpectrogram(16000, n_fft=n_fft, hop_length=n_fft // 4, n_mels=n_mels, power=power).to(DEV)
    if fb is not None:
        m.mel_scale.fb.copy_(torch.as_tensor(fb, dtype=torch.float32).to(DEV))
    return m


def check_mel(n_fft, m, x, what):
    """m(x) on poisoned memory against the oracle with the module's own bank; all-zero filters come out exactly 0."""
    fb = m.mel_scale.fb.cpu().numpy()
    n_mels = fb.shape[1]
    xd = x.to(DEV)
    frames = 1 + x.shape[-1] // (n_fft // 4)
    got, names = poisoned(lambda: m(xd), x.shape[0] * frames * n_mels)
    got = got.cpu()
    bad = int((~torch.isfinite(got)).sum())
    assert bad == 0, f"{what}: {bad} non-finite outputs (columns never stored)"
    exp = O.mel_spectrogram(x.numpy(), sample_rate=16000, n_fft=n_fft, hop_length=n_fft // 4, n_mels=n_mels, fb=fb)
    scaled_tol_close(got.numpy(), exp, what=what)
    zero = np.all(fb == 0, axis=0)
    assert (got.numpy()[:, zero, :] == 0).all(), f"{what}: all-zero filters must give exact zeros"
    return got, names


# ---- 1. filter counts ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_fft", NFFTS)
@pytest.mark.parametrize("n_mels", [1, 3, 13, 129, 256, 384, 511, 512])
def test_filter_counts(n_fft, n_mels):
    """Up to 64 groups on the register-FFT mel kernel: partial last groups, 2--5 empty groups at n_fft 256 (384--512
    mels), fragments in global memory at n_fft 1024 (384--512 mels) and 2048 (every count past 13)."""
    x = randn(3, 7 * n_fft + 123, n_fft + n_mels)
    _, names = check_mel(n_fft, mel_module(n_fft, n_mels), x, f"n_fft={n_fft} n_mels={n_mels}")
    assert_ran(names, MEL_KERNEL[n_fft], absent=("stft_generic_kernel",))


@pytest.mark.parametrize("n_fft", NFFTS)
def test_513_filters_take_the_generic_kernel(n_fft):
    x = randn(3, 7 * n_fft + 123, n_fft + 513)
    _, names = check_mel(n_fft, mel_module(n_fft, 513), x, f"n_fft={n_fft} n_mels=513")
    assert_ran(names, "stft_generic_kernel", absent=(MEL_KERNEL[n_fft],))


# ---- 2. custom banks -----------------------------------------------------------------------------------------------
FULL_BAND_GROUPS = (5, 31, 60)


def custom_bank(kind, n_bins, seed):
    g = torch.Generator().manual_seed(seed)

    def rand(*shape):
        return torch.rand(*shape, generator=g).double().numpy() + 0.05

    if kind == "all_zero":
        return np.zeros((n_bins, 40))
    if kind == "one_live_filter_in_partial_group":  # filters 40..42 form the last group, only 42 is live
        fb = np.zeros((n_bins, 43))
        fb[n_bins // 3 : n_bins // 2, 42] = rand(n_bins // 2 - n_bins // 3)
        return fb
    if kind == "interior_zero_run":
        fb = O.melscale_fbanks(n_bins, 0.0, 8000.0, 16, 16000)
        a, b = n_bins // 8, n_bins // 2
        fb[:, 5] = 0.0
        fb[a:b, 5] = rand(b - a)
        fb[a + (b - a) // 3 : a + 2 * (b - a) // 3, 5] = 0.0
        return fb
    if kind == "negative_weights":
        fb = O.melscale_fbanks(n_bins, 0.0, 8000.0, 24, 16000)
        return fb * np.where(rand(*fb.shape) < 0.55, -1.0, 1.0)
    fb = np.zeros((n_bins, 512))
    for t in FULL_BAND_GROUPS:
        fb[:, 8 * t : 8 * t + 8] = rand(n_bins, 8)
    if kind == "skewed_full_band_and_empty":
        return fb
    assert kind == "skewed_full_band_and_one_step"
    for t in range(64):
        if t not in FULL_BAND_GROUPS:
            s = t % (n_bins // 8)
            fb[8 * s : 8 * s + 8, 8 * t : 8 * t + 8] = rand(8, 8)
    return fb


# (a dense bank at every n_fft: tests/test_gpu_fast_paths.py::test_dense_filterbank_matrix)
BANKS = ["all_zero", "one_live_filter_in_partial_group", "interior_zero_run", "negative_weights",
         "skewed_full_band_and_empty", "skewed_full_band_and_one_step"]


@pytest.mark.parametrize("n_fft", NFFTS)
@pytest.mark.parametrize("kind", BANKS)
def test_custom_banks(n_fft, kind):
    """Banks written into mel_scale.fb in place.  The two skewed banks (3 full-band groups among 61 empty or one-step
    ones, 512 filters) put more than 32 groups on one of the n_fft 2048 kernel's contraction warps unless the plan
    caps its lists."""
    fb = custom_bank(kind, n_fft // 2 + 1, n_fft + len(kind))
    x = randn(3, 7 * n_fft + 123, n_fft + 7)
    _, names = check_mel(n_fft, mel_module(n_fft, fb.shape[1], fb), x, f"n_fft={n_fft} {kind}")
    assert_ran(names, MEL_KERNEL[n_fft])


# ---- 3. a group's bits do not depend on its warp or on where its fragments live ----------------------------------
@pytest.mark.parametrize("n_fft", NFFTS)
@pytest.mark.parametrize("power", [2.0, 1.0])
def test_group_values_do_not_depend_on_schedule(n_fft, power):
    """64 filters whose fragments fit in shared memory, then the same 64 with dense groups appended until the plan
    passes the fragment reserve (another warp assignment, fragments from global memory): columns [0, 64) bit-equal."""
    n_bins = n_fft // 2 + 1
    base = O.melscale_fbanks(n_bins, 0.0, 4000.0, 64, 16000).astype(np.float32)
    dense_steps = (n_bins + 7) // 8
    extra = 8 * (FRAG_RESERVE[n_fft] // dense_steps + 1)
    g = torch.Generator().manual_seed(n_fft)
    wide = np.concatenate([base, torch.rand(n_bins, extra, generator=g).numpy()], axis=1)
    assert plan_steps(base) <= FRAG_RESERVE[n_fft] < plan_steps(wide) and wide.shape[1] <= 512
    x = randn(3, 7 * n_fft + 123, n_fft + 11).to(DEV)
    outs = []
    for fb in (base, wide):
        m = mel_module(n_fft, fb.shape[1], fb, power)
        out, names = launched(lambda: m(x))
        assert_ran(names, MEL_KERNEL[n_fft])
        outs.append(out)
    assert torch.equal(outs[1][:, :64], outs[0])


# ---- 4. feature stage and the four finish kernels ------------------------------------------------------------------
FEATURE_CASES = [
    # transform, n_fft, n_filters, n_coeffs, log, finish kernel
    ("mfcc", 1024, 256, 40, False, "mfcc_finish_tiled_kernel<5>"),  # mma tile 215 KB > 200 KB
    ("mfcc", 1024, 512, 40, False, "mfcc_finish_kernel"),  # tiled tile 337 KB > 200 KB
    ("mfcc", 1024, 128, 64, False, "mfcc_finish_mma_kernel"),
    ("mfcc", 1024, 128, 128, False, "mfcc_finish_kernel"),  # n_mfcc > 64
    ("mfcc", 1024, 128, 60, True, "mfcc_finish_tiled_kernel<8>"),  # log_mels: no clamp, n_mfcc 41..64
    ("lfcc", 512, 40, 80, False, "mfcc_finish_kernel"),  # n_lfcc 80 > n_filter 40
]


@pytest.mark.parametrize("case", FEATURE_CASES, ids=lambda c: "-".join(str(v) for v in c[:5]))
def test_feature_finish_kernels(case):
    kind, n_fft, n_filt, n_coef, log, finish = case
    x = randn(4, 12 * n_fft + 77, n_filt + n_coef)
    x[1] *= 1e-3  # a quiet row: the batch-global clamp bites there
    if kind == "mfcc":
        kw = dict(n_fft=n_fft, hop_length=n_fft // 4, n_mels=n_filt)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            mod = T.MFCC(16000, n_mfcc=n_coef, log_mels=log, melkwargs=kw).to(DEV)
        fb, dct = mod.MelSpectrogram.mel_scale.fb.cpu().numpy(), mod.dct_mat.cpu().numpy()
        oracle = lambda v: O.mfcc(v, 16000, n_coef, "ortho", log, kw, fb=fb, dct=dct)  # noqa: E731
    else:
        kw = dict(n_fft=n_fft, hop_length=n_fft // 4)
        mod = T.LFCC(16000, n_filter=n_filt, n_lfcc=n_coef, log_lf=log, speckwargs=kw).to(DEV)
        filt, dct = mod.filter_mat.cpu().numpy(), mod.dct_mat.cpu().numpy()
        oracle = lambda v: O.lfcc(v, 16000, n_filt, n_lfcc=n_coef, log_lf=log, speckwargs=kw, filter_mat=filt,  # noqa: E731
                                  dct=dct)
    for v, what in ((x, "2-D (batch-global clamp)"), (x[:, None], "3-D (per-item clamp)")):
        got, names = launched(lambda: mod(v.to(DEV)))
        assert_ran(names, MEL_KERNEL[n_fft])
        assert_ran(names, finish)
        assert_close(got.cpu().numpy(), oracle(v.numpy()), rtol=1e-4, atol=5e-3, what=f"{case} {what}")


def test_mfcc_on_skewed_bank_2048():
    """The MFCC feature stage shares the mel plan: the skewed bank at n_fft 2048 (unwritten feature columns would
    reach every coefficient through the DCT)."""
    kw = dict(n_fft=2048, hop_length=512, n_mels=512)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        mod = T.MFCC(16000, n_mfcc=40, melkwargs=kw).to(DEV)
    fb = custom_bank("skewed_full_band_and_one_step", 1025, 2048)
    mod.MelSpectrogram.mel_scale.fb.copy_(torch.as_tensor(fb, dtype=torch.float32).to(DEV))
    x = randn(3, 9 * 2048 + 123, 17)
    x[1] *= 1e-3
    xd = x.to(DEV)
    frames = 1 + x.shape[-1] // 512
    got, names = poisoned(lambda: mod(xd), 3 * frames * 512, 3 * frames * 40)
    assert_ran(names, "stft2048_mel_kernel")
    assert_ran(names, "mfcc_finish_kernel")
    got = got.cpu()
    assert bool(torch.isfinite(got).all()), "non-finite coefficients (feature columns never stored)"
    exp = O.mfcc(x.numpy(), 16000, 40, "ortho", False, kw, fb=mod.MelSpectrogram.mel_scale.fb.cpu().numpy(),
                 dct=mod.dct_mat.cpu().numpy())
    assert_close(got.numpy(), exp, rtol=1e-4, atol=5e-3, what="skewed bank MFCC")


# ---- 5. mel gradient on either side of the fused kernel's shared-memory limit -------------------------------------
FUSED, COMPOSED = "stft_pow2_backward_kernel", "spec_vjp_kernel"
GRAD_CASES = [
    # n_fft, n_mels, kernel: the fused kernel holds 16 warps x frames-per-unit x n_mels floats of the upstream gradient
    (256, 149, FUSED),
    (256, 150, COMPOSED),
    (512, 331, FUSED),
    (512, 332, COMPOSED),
    (1024, 512, FUSED),
    (256, 384, COMPOSED),  # with 2 empty filter groups
]


@pytest.mark.parametrize("n_fft,n_mels,kernel", GRAD_CASES)
def test_mel_grad_fused_limit(n_fft, n_mels, kernel):
    gen = torch.Generator().manual_seed(n_fft + n_mels)
    x = torch.randn(3, 9000, generator=gen)
    mod = mel_module(n_fft, n_mels)
    fb = mod.mel_scale.fb.double().cpu().numpy()
    hop = n_fft // 4
    g = torch.randn(3, n_mels, 1 + 9000 // hop, generator=gen)

    def grad():
        with audio_b200.differentiable():
            xt = x.to(DEV).requires_grad_()
            mod(xt).backward(g.to(DEV))
        return xt.grad

    got, names = launched(grad)
    assert_ran(names, kernel, absent=({FUSED, COMPOSED} - {kernel}))
    exp = V.mel_spectrogram_vjp(x.double().numpy(), g.numpy(), 16000, n_fft=n_fft, hop_length=hop, fb=fb)
    got = got.double().cpu().numpy()
    err = np.abs(got - exp)
    tol = 1e-4 * np.abs(exp) + 1e-4 * float(np.sqrt(np.mean(exp**2)))  # test_gpu_grad.py's bar for power 2
    assert (err <= tol).all(), f"max err {err.max():.3e}, worst ratio {(err / tol).max():.3f}"


# ---- 6. Kaldi features with many bins on the register path --------------------------------------------------------
@pytest.mark.parametrize("kind", ["fbank", "mfcc"])
def test_kaldi_many_bins(kind):
    """512-point frames at 16 kHz, 128 mel bins, the energy column in front of the mel columns."""
    with np.load(os.path.join(GOLDEN, "kaldi_ref_cases.npz")) as z:
        wave = z["wave"][:1, :16000].astype(np.float32)
    kw = dict(num_mel_bins=128, use_energy=True)
    got, names = launched(lambda: getattr(K, kind)(torch.from_numpy(wave).to(DEV), **kw))
    assert_ran(names, "stft_pow2_mel_kernel", absent=("stft_generic_kernel",))
    got = got.cpu().numpy()
    exp = getattr(KO, kind)(wave, **kw)
    assert got.shape == exp.shape == (exp.shape[0], 129 if kind == "fbank" else 13)
    # test_kaldi.py's bars against the oracle
    bar = 2e-5 * np.abs(exp).max() + (1e-4 if kind == "fbank" else 2e-4)
    assert np.abs(got - exp).max() <= bar, (kind, np.abs(got - exp).max(), bar)
