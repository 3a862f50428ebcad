"""GPU checks of the Kaldi feature gradients (compliance.kaldi spectrogram / fbank / mfcc inside
audio_b200.differentiable(kaldi=True)) against the float64 numpy VJPs of tests/kaldi_grad_oracle.py.

The bar follows DESIGN §4's precedent for the feature gradients: the GPU gradient's largest error is at most twice that
of the float32 CPU run of the same op sequence (tests/kaldi_grad_oracle.py:torch_kaldi), and it meets the forward bar
wherever that run does.  Where neither holds, the pinned bar of the STFT-amplified MFCC gradient applies (relative L2 at
most 5e-3, largest error at most 2e-2 of the largest magnitude): the 1/v of the log amplifies the GPU FFT's round-off on
quiet bins, which is larger than the CPU float32 FFT's, and a log(max(v, eps)) whose v sits within round-off of eps
decides the other side of the floor on one of the two runs.  Measured on an H100 (the module prints every case that
needs the pinned bar): the option sets on tones with a 60 dB quieter stretch, e.g. use_power=False fbank at relative L2
4.9e-4 / max 3.6e-4 of scale, most others at relative L2 1e-5 to 7e-5 / max 1e-5 to 6e-5, where the CPU float32 run is
at 2e-7 to 3e-6 of scale.  Those cases stay 10x inside the pinned bar, so a regression of 10x goes unnoticed only there."""
import json
import os

import numpy as np
import pytest
import torch

import audio_b200
import audio_b200.compliance.kaldi as K
import audio_b200.transforms as T
from oracle import kaldi_oracle as KO

import kaldi_grad_oracle as V
from resample_grad_oracle import resample_vjp

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
KINDS = ("spectrogram", "fbank", "mfcc")


def _np(t):
    return t.detach().double().cpu().numpy()


def check(got, exp, f32):
    assert np.isfinite(exp).all() and np.isfinite(got).all()
    scale = float(np.abs(exp).max())
    if scale == 0.0:
        assert np.abs(got).max() == 0.0
        return
    e_gpu, e_f32 = np.abs(got - exp), np.abs(f32 - exp)
    tol = 1e-4 * np.abs(exp) + 1e-4 * float(np.sqrt(np.mean(exp**2)))
    evidence = e_gpu.max() <= 2.0 * e_f32.max() + 1e-6 * scale and (not (e_f32 <= tol).all() or (e_gpu <= tol).all())
    if evidence:
        return
    rel = float(np.sqrt((e_gpu**2).sum() / (exp**2).sum()))
    FALLBACKS.append((os.environ.get("PYTEST_CURRENT_TEST", "").split(" ")[0], rel, e_gpu.max() / scale,
                      e_f32.max() / scale))
    assert rel <= 5e-3 and e_gpu.max() <= 2e-2 * scale, (
        f"relative L2 {rel:.3e}, max {e_gpu.max() / scale:.3e} of scale; float32 cpu max {e_f32.max() / scale:.3e}")


FALLBACKS = []  # (test, relative L2, max / scale, float32 cpu max / scale) of every case held to the pinned bar


@pytest.fixture(scope="module", autouse=True)
def _report_fallbacks():
    yield
    for case in FALLBACKS:
        print("pinned bar: %s rel L2 %.3e max %.3e (float32 cpu max %.3e)" % case)


def launched(fn, expect):
    """fn() under torch.profiler: its result and the CUDA kernel names it launched.  A session now and then comes back
    without some of its kernel records; fn (deterministic) then runs again, up to three sessions, until every name in
    `expect` was recorded."""
    names = []
    for _ in range(3):
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        if all(any(k in n for n in names) for k in expect):
            return out, names
    return out, names


def grad_of(fn, x, g=None):
    """(output, waveform gradient) of fn on a CUDA copy of x; g: the upstream gradient (None: sum)."""
    with audio_b200.differentiable(kaldi=True):
        xt = x.detach().to(DEV, copy=True).requires_grad_()
        y = fn(xt)
        y.backward(g.to(DEV) if g is not None else torch.ones_like(y))
    return y.detach(), xt.grad


def _against_oracle(kind, wave, kw, seed):
    """wave: (1, n) float32 numpy."""
    shape = tuple(V.torch_kaldi(kind, torch.from_numpy(wave[0]).double(), **kw).shape)
    g = np.random.default_rng(seed).standard_normal(shape)
    _, dx = grad_of(lambda t: getattr(K, kind)(t, **kw), torch.from_numpy(wave), torch.from_numpy(g).float())
    exp = V.kaldi_vjp(kind, wave[0], g, **kw)
    f32 = V.torch_vjp(kind, wave[0], g, dtype=torch.float32, **kw)
    check(_np(dx)[0], exp, f32)


def _cases(fixture, kind):
    return [json.loads(str(a)) for a in fixture[f"{kind}_args"]]


@pytest.mark.parametrize("kind", KINDS)
def test_kaldi_goldens_against_oracle(kind):
    fx = np.load(os.path.join(GOLDEN, "kaldi_goldens.npz"))
    wave = fx["wave"].astype(np.float32)
    for i, kw in enumerate(_cases(fx, kind)):
        kw = {k: v for k, v in kw.items() if k != "dither"}
        _against_oracle(kind, wave, kw, i)


@pytest.mark.parametrize("kind", KINDS)
def test_long_signals_against_oracle(kind):
    fx = np.load(os.path.join(GOLDEN, "kaldi_ref_cases.npz"))
    wave = fx["wave"][:1].astype(np.float32)
    for i, kw in enumerate(_cases(fx, kind)):
        _against_oracle(kind, wave, kw, 100 + i)


def _wave(n, seed, sr=16000.0):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / sr
    x = 0.3 * np.sin(2 * np.pi * 440.0 * t) + 0.05 * rng.standard_normal(n)
    x[n // 3: n // 3 + n // 10] *= 1e-3  # a quiet stretch
    return x[None].astype(np.float32)


OPTION_SETS = [
    dict(window_type="hamming"), dict(window_type="hanning"), dict(window_type="rectangular"),
    dict(window_type="blackman"), dict(window_type="povey", snip_edges=False),
    dict(use_power=False), dict(use_log_fbank=False), dict(htk_compat=True, use_energy=True),
    dict(use_energy=True, raw_energy=False), dict(use_energy=True, raw_energy=True, snip_edges=False),
    dict(vtln_warp=1.1), dict(subtract_mean=True, use_energy=True), dict(energy_floor=0.0, use_energy=True),
    dict(remove_dc_offset=False, preemphasis_coefficient=0.0, use_energy=True),
]


@pytest.mark.parametrize("kind", ("fbank", "mfcc", "spectrogram"))
@pytest.mark.parametrize("opt", range(len(OPTION_SETS)))
def test_options_against_oracle(kind, opt):
    kw = dict(OPTION_SETS[opt])
    if kind == "spectrogram":
        kw = {k: v for k, v in kw.items() if k not in ("use_power", "use_log_fbank", "htk_compat", "use_energy", "vtln_warp")}
    if kind == "mfcc":
        kw.pop("use_power", None)
        kw.pop("use_log_fbank", None)
    _against_oracle(kind, _wave(8000, opt), kw, opt)


# sample rate -> padded FFT size at 25 ms: 256 / 512 / 1024 (fused) / 2048; round_to_power_of_two=False -> 320 / 400
PATHS = [(8000.0, True), (16000.0, True), (32000.0, True), (48000.0, True), (12800.0, False), (16000.0, False)]
FUSED = ("stft_pow2_backward_kernel", "kaldi_log_vjp_kernel", "kaldi_cond_vjp_kernel", "frame_fold_kernel")
COMPOSED = ("kaldi_log_vjp_kernel", "stft_generic_kernel", "spec_vjp_kernel", "kaldi_cond_vjp_kernel", "frame_fold_kernel")


@pytest.mark.parametrize("kind", ["fbank", "spectrogram"])
@pytest.mark.parametrize("sr,pow2", PATHS)
@pytest.mark.parametrize("snip", [True, False])
def test_paths(kind, sr, pow2, snip):
    """Padded 256 / 512 / 1024 take the fused kernel (the Kaldi variant of stft_pow2_backward_kernel; no complex
    spectrum, no spec_vjp_kernel); every other size the composition.  Both against the oracle."""
    x = torch.from_numpy(_wave(int(sr), 3, sr)).to(DEV)
    kw = dict(sample_frequency=sr, round_to_power_of_two=pow2, snip_edges=snip)
    if kind == "fbank":
        kw.update(use_energy=True, num_mel_bins=40)
    fn = getattr(K, kind)

    def run():
        with audio_b200.differentiable(kaldi=True):
            xt = x.clone().requires_grad_()
            fn(xt, **kw).sum().backward()
        return xt.grad

    fused = pow2 and sr <= 32000.0
    expect = FUSED if fused else COMPOSED
    _, names = launched(run, expect)
    for kern in expect:
        assert any(kern in n for n in names), (kern, sorted(set(names)))
    if fused:
        assert not any("spec_vjp_kernel" in n for n in names), sorted(set(names))
    dx = run()
    w = x.cpu().numpy()[0]
    ones = np.ones_like(getattr(KO, kind)(w.astype(np.float64), **kw))
    check(_np(dx)[0], V.kaldi_vjp(kind, w, ones, **kw), V.torch_vjp(kind, w, ones, dtype=torch.float32, **kw))


def test_fused_path_declines_from_the_descriptors_alone():
    """The fused kernel stages the mel gradient rows of a unit in shared memory: past 331 filters at padded 512 they do
    not fit and the composition runs -- the same choice for one row and for a batch."""
    x = torch.from_numpy(_wave(16000, 8)).to(DEV)
    for rows in (1, 3):
        xb = x.repeat(rows, 1)

        def run():
            with audio_b200.differentiable(kaldi=True):
                xt = xb.clone().requires_grad_()
                K.fbank_batch(xt, num_mel_bins=340, low_freq=0.0).sum().backward()
            return xt.grad

        _, names = launched(run, COMPOSED)
        assert any("spec_vjp_kernel" in n for n in names) and not any("stft_pow2_backward_kernel" in n for n in names)


def test_golden_frame_sizes_run_the_composition():
    fx = np.load(os.path.join(GOLDEN, "kaldi_goldens.npz"))
    x = torch.from_numpy(fx["wave"].astype(np.float32)).to(DEV)

    def run():
        with audio_b200.differentiable(kaldi=True):
            xt = x.clone().requires_grad_()
            K.fbank(xt, frame_length=1.0, frame_shift=0.5, num_mel_bins=4, low_freq=0.0, sample_frequency=17000.0,
                    use_energy=True).sum().backward()  # 17-sample frames in a 32-point FFT
        return xt.grad

    _, names = launched(run, COMPOSED)
    for kern in COMPOSED:
        assert any(kern in n for n in names), (kern, sorted(set(names)))


@pytest.mark.parametrize("sr", [8000.0, 16000.0])
def test_energy_floor_tie_gets_half_on_the_device(sr):
    """Rectangular window, no DC removal, no pre-emphasis, frames of ones with E = win = energy_floor (exact in float32):
    the floor's maximum ties and the energy column's gradient is halved -- 1/win per sample.  8 kHz: 16-sample frames
    in 16-point FFTs; 16 kHz: 400-sample frames in 512-point FFTs."""
    win = 16 if sr == 8000.0 else 400
    kw = dict(window_type="rectangular", remove_dc_offset=False, preemphasis_coefficient=0.0, energy_floor=float(win),
              frame_length=1000.0 * win / sr, frame_shift=1000.0 * win / sr, sample_frequency=sr, use_energy=True,
              num_mel_bins=4, low_freq=0.0)
    x = torch.ones(1, 3 * win)
    y = K.fbank(x.to(DEV), **kw)
    g = torch.zeros(y.shape)
    g[:, 0] = 1.0  # the energy column only
    _, dx = grad_of(lambda t: K.fbank(t, **kw), x, g)
    exp = V.kaldi_vjp("fbank", x[0].numpy(), g.numpy(), **kw)
    assert np.allclose(exp, 1.0 / win)
    assert np.abs(_np(dx)[0] - exp).max() <= 1e-6 / win


def test_channel_selection_gives_zero_to_other_channel():
    x = torch.from_numpy(np.concatenate([_wave(6000, 1), _wave(6000, 2)]))
    _, dx = grad_of(lambda t: K.fbank(t, channel=1, use_energy=True), x)
    assert torch.count_nonzero(dx[0]) == 0 and torch.count_nonzero(dx[1]) > 0


def test_expanded_and_non_contiguous_grads():
    x = torch.from_numpy(_wave(8000, 4))
    _, d_sum = grad_of(lambda t: K.mfcc(t, use_energy=True).sum(), x)
    ones = torch.ones_like(K.mfcc(x.to(DEV), use_energy=True))
    _, d_ones = grad_of(lambda t: K.mfcc(t, use_energy=True), x, ones.cpu())
    assert torch.equal(d_sum, d_ones)
    for fn, kw in ((K.mfcc, dict(use_energy=True)), (K.fbank, dict(use_energy=True)), (K.spectrogram, {}),
                   (K.fbank, dict(round_to_power_of_two=False))):
        y = fn(x.to(DEV), **kw)
        gt = torch.randn(y.shape[1], y.shape[0]).t()  # non-contiguous: the log adjoint reads it at strides (1, T)
        assert gt.stride() == (1, y.shape[0])
        _, d_nc = grad_of(lambda t: fn(t, **kw), x, gt)
        _, d_c = grad_of(lambda t: fn(t, **kw), x, gt.contiguous())
        assert torch.equal(d_nc, d_c)


def _config_input(rows=256, length=160000, seed=21):
    g = torch.Generator().manual_seed(seed)
    return (0.1 * torch.randn(rows, length, generator=g)).to(DEV)


def test_large_batch_deterministic_row_independent_and_forward_unchanged():
    x = _config_input()
    kw = dict(num_mel_bins=80, use_energy=True)
    with torch.no_grad():
        ref = K.fbank_batch(x, **kw)
    with audio_b200.differentiable(kaldi=True):
        xt = x.clone().requires_grad_()
        y = K.fbank_batch(xt, **kw)
        g = torch.randn(y.shape, generator=torch.Generator().manual_seed(3)).to(DEV)
        (d1,) = torch.autograd.grad(y, xt, g)
        (d2,) = torch.autograd.grad(K.fbank_batch(xt, **kw), xt, g)
        x1 = x[17:18].clone().requires_grad_()
        (d_row,) = torch.autograd.grad(K.fbank_batch(x1, **kw), x1, g[17:18])
    assert torch.equal(y.detach(), ref)
    assert torch.equal(d1, d2)
    assert torch.equal(d_row[0], d1[17])
    for r in (0, 255):
        exp = V.kaldi_vjp("fbank", _np(x[r]), _np(g[r]), **kw)
        f32 = V.torch_vjp("fbank", _np(x[r]), _np(g[r]), dtype=torch.float32, **kw)
        check(_np(d1[r]), exp, f32)


def test_chain_resample_fbank_l1():
    rs = T.Resample(48000, 16000).to(DEV)
    x = torch.from_numpy(_wave(48000, 5, 48000.0).repeat(2, 0))
    x[1] *= 0.5
    kw = dict(num_mel_bins=40, use_energy=True)
    with audio_b200.differentiable(resample=True, kaldi=True):
        xt = x.to(DEV).requires_grad_()
        r = rs(xt)
        y = K.fbank_batch(r, **kw)
        y.abs().sum().backward()
    for b in range(2):
        rb = _np(r[b])
        g = np.sign(_np(y[b]))
        g_r = V.kaldi_vjp("fbank", rb, g, **kw)
        exp = resample_vjp(g_r[None], rs.orig_freq, rs.new_freq, rs.gcd, rs.kernel.double().cpu().numpy(), rs.width,
                           x.shape[1])[0]
        err = np.abs(_np(xt.grad[b]) - exp)
        rel = float(np.sqrt((err**2).sum() / (exp**2).sum()))
        assert rel <= 5e-3 and err.max() <= 2e-2 * np.abs(exp).max(), (rel, err.max() / np.abs(exp).max())


def test_error_cases():
    x = torch.from_numpy(_wave(8000, 6)).to(DEV)
    with audio_b200.differentiable(kaldi=True):
        xt = x.clone().requires_grad_()
        y = K.fbank(xt)
        (g,) = torch.autograd.grad(y.sum(), xt, create_graph=True)
        with pytest.raises(RuntimeError):
            g.sum().backward()
        xt2 = x.clone().requires_grad_()
        leaf = xt2 * 1.0
        y2 = K.fbank(leaf)
        with torch.no_grad():
            leaf.add_(1.0)
        with pytest.raises(RuntimeError, match="modified by an inplace operation"):
            y2.sum().backward()
        with pytest.raises(RuntimeError, match="dither"):
            K.fbank(x.clone().requires_grad_(), dither=1.0)
        assert K.fbank(x.clone().requires_grad_(), min_duration=10.0).numel() == 0
    for kwargs in (dict(), dict(inverse=True), dict(resample=True), dict(features=True),
                   dict(inverse=True, resample=True, features=True)):
        with audio_b200.differentiable(**kwargs):
            for fn in (K.fbank, K.mfcc, K.spectrogram):
                with pytest.raises(RuntimeError, match=r"kaldi=True"):
                    fn(x.clone().requires_grad_())
