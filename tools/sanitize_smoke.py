"""Small invocations of every kernel family for compute-sanitizer:
    compute-sanitizer --tool memcheck python tools/sanitize_smoke.py
(racecheck reports the mbarrier-synchronised hand-offs as hazards -- the bulk-copy staging of every register-FFT
kernel and the warp-specialised n_fft = 2048 mel kernel -- because it does not model mbarrier ordering; memcheck and
initcheck are the meaningful tools here)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import audio_b200  # noqa: E402
import audio_b200.compliance.kaldi as K  # noqa: E402
import audio_b200.transforms as T  # noqa: E402

x = torch.randn(3, 12000, device="cuda")
for n_fft in (256, 512, 1024, 2048, 400):
    T.MelSpectrogram(16000, n_fft=n_fft, hop_length=n_fft // 4, n_mels=40).cuda()(x)
    T.Spectrogram(n_fft=n_fft, hop_length=n_fft // 4).cuda()(x)
    spec = T.Spectrogram(n_fft=n_fft, hop_length=n_fft // 4, power=None).cuda()(x)
    T.InverseSpectrogram(n_fft=n_fft, hop_length=n_fft // 4).cuda()(spec, 12000)
# mel plans at their limits: 512 mels with empty filter groups at n_fft 256; at n_fft 2048 a skewed bank (3 full-band
# groups, 61 empty ones) that would put more than 32 groups on one contraction warp without the per-warp cap
T.MelSpectrogram(16000, n_fft=256, hop_length=64, n_mels=512).cuda()(x)
skewed = T.MelSpectrogram(16000, n_fft=2048, hop_length=512, n_mels=512).cuda()
skewed.mel_scale.fb.zero_()
for t in (5, 31, 60):
    skewed.mel_scale.fb[:, 8 * t : 8 * t + 8] = torch.rand(1025, 8, device="cuda")
skewed(x)
with audio_b200.differentiable():  # waveform gradients: the fused path (512 / 1024), the composition path (400 / 2048)
    for mod in (T.MelSpectrogram(16000, n_fft=1024, hop_length=256, n_mels=40), T.Spectrogram(n_fft=512, power=1.0),
                T.Spectrogram(n_fft=512, power=None), T.MelSpectrogram(16000, n_fft=2048, hop_length=512, n_mels=40),
                T.Spectrogram(n_fft=400, power=None, onesided=False)):
        xg = x.clone().requires_grad_()
        mod.cuda()(xg).abs().sum().backward()
with audio_b200.differentiable(inverse=True):  # spectrogram gradients: fused (256 / 1024), composition (400 / 2048)
    for n_fft, pad in ((256, 0), (1024, 5), (400, 3), (2048, 0)):
        spec = T.Spectrogram(n_fft=n_fft, hop_length=n_fft // 4, power=None).cuda()(x).requires_grad_()
        T.InverseSpectrogram(n_fft=n_fft, hop_length=n_fft // 4, pad=pad).cuda()(spec, 11000).sum().backward()
with audio_b200.differentiable(features=True):  # feature gradients: MFCC clamp + ties, log path, LFCC, the stand-alones
    for mod, xin in ((T.MFCC(16000, n_mfcc=13, melkwargs=dict(n_fft=512, hop_length=160, n_mels=40)), x),
                     (T.MFCC(16000, n_mfcc=20, log_mels=True), x.reshape(1, 3, -1)),
                     (T.LFCC(16000, n_lfcc=13, speckwargs=dict(n_fft=400)), x),
                     (T.SpectralCentroid(16000, n_fft=512), x)):
        mod.cuda()(xin.clone().requires_grad_()).sum().backward()
    spec = T.Spectrogram(n_fft=400).cuda()(x).requires_grad_()
    T.AmplitudeToDB(top_db=0.0)(T.MelScale(40, 16000, n_stft=201).cuda()(spec)).sum().backward()
    # InverseMelScale forward + backward: a frame-major input with a partial last tile, a contiguous 2-D one
    mel = T.MelSpectrogram(16000, n_fft=512, hop_length=128, n_mels=40, power=1.0).cuda()(x).requires_grad_()
    T.InverseMelScale(257, 40, 16000).cuda()(mel).sum().backward()
    T.InverseMelScale(257, 40, 16000).cuda()(mel.detach()[0].contiguous().requires_grad_()).sum().backward()
T.MFCC(16000, n_mfcc=13, melkwargs=dict(n_fft=512, hop_length=160, n_mels=40)).cuda()(x)
T.MFCC(16000, n_mfcc=40, melkwargs=dict(n_fft=1024, hop_length=256, n_mels=80)).cuda()(x.reshape(1, 3, -1))
for kw in (dict(num_mel_bins=40, snip_edges=False, use_energy=True), dict(num_mel_bins=23), dict(frame_length=20.0, round_to_power_of_two=False)):
    K.fbank_batch(x * 1000, **kw)
K.mfcc_batch(x * 1000, subtract_mean=True)
K.spectrogram_batch(x * 1000)
with audio_b200.differentiable(kaldi=True):  # Kaldi waveform gradients: 512-point frames with mirrored edges, 400-point
    for fn, kw in ((K.fbank_batch, dict(num_mel_bins=40, snip_edges=False, use_energy=True)),
                   (K.mfcc_batch, dict(round_to_power_of_two=False, use_energy=True, subtract_mean=True))):
        fn((x * 1000).requires_grad_(), **kw).sum().backward()
T.Resample(44100, 16000).cuda()(x)
T.Resample(16000, 22050, resampling_method="sinc_interp_kaiser").cuda()(x)
with audio_b200.differentiable(resample=True):  # resampler waveform gradients: the mma kernel, the direct kernel
    for o, n in ((44100, 16000), (2003, 1999)):
        T.Resample(o, n).cuda()(x.clone().requires_grad_()).sum().backward()
T.GriffinLim(n_fft=512, hop_length=128, n_iter=3, length=12000, rand_init=False).cuda()(
    T.Spectrogram(n_fft=512, hop_length=128).cuda()(x))
T.PitchShift(16000, 12).cuda()(x)
T.TimeStretch(hop_length=128, n_freq=257, fixed_rate=1.3).cuda()(T.Spectrogram(n_fft=512, hop_length=128, power=None).cuda()(x))
with audio_b200.differentiable(vocoder=True):  # phase-vocoder adjoint: TimeStretch alone, then the whole PitchShift chain
    spec = T.Spectrogram(n_fft=512, hop_length=128, power=None).cuda()(x).requires_grad_()
    T.TimeStretch(hop_length=128, n_freq=257, fixed_rate=0.8).cuda()(spec).abs().sum().backward()
    T.PitchShift(16000, -3).cuda()(x.clone().requires_grad_()).sum().backward()
import audio_b200.functional as F  # noqa: E402

# IIR filtering: lfilter forward + backward over several tiles, filtfilt, a pure gain (n_order = 1), a signal shorter
# than one chunk, the order cap and batching=False (stride-0 rows)
with audio_b200.differentiable(filtering=True):
    xg = x.clone().requires_grad_()
    a = torch.tensor([1.0, -1.8, 0.81], device="cuda", requires_grad=True)
    b = torch.tensor([0.01, 0.02, 0.01], device="cuda", requires_grad=True)
    F.lfilter(xg, a, b).sum().backward()
    F.filtfilt(xg, a, b).sum().backward()
    F.lfilter(xg, a[:1], b[:1]).sum().backward()
    F.lfilter(xg[:, :20], a, b).sum().backward()
a16 = 0.01 * torch.rand(3, 17, device="cuda")
a16[:, 0] = 1.0
F.lfilter(x, a16, torch.rand(3, 17, device="cuda"), batching=False)
F.deemphasis(x)
# FFT convolution: a broadcast two-partition filter forward + backward (swapped operands), and "same" with P = 1
with audio_b200.differentiable(filtering=True):
    xg = x.clone().requires_grad_()
    F.fftconvolve(torch.randn(1, 1, 2500, device="cuda", requires_grad=True), xg[:, None, :3000]).sum().backward()
F.fftconvolve(x, torch.randn(3, 255, device="cuda"), "same")
# direct convolution: a broadcast filter forward + backward (swapped operands), and "same" with fragments streamed
with audio_b200.differentiable(filtering=True):
    xg = x.clone().requires_grad_()
    F.convolve(torch.randn(1, 1, 200, device="cuda", requires_grad=True), xg[:, None, :3000]).sum().backward()
F.convolve(x, torch.randn(3, 1025, device="cuda"), "same")
# vad: a trim over several chunks with carried state, and an input shorter than one measurement frame
from audio_b200 import _filtering  # noqa: E402
_filtering.VadPlan(16000, trigger_level=1e9).run(x, chunk=7)
F.vad(x[:1, :1000], 16000)
# rnnt_loss: forward + backward in float32 and float16 with ragged lengths and a V with a vector tail, U + 1 > 1024
# (more cells per diagonal than threads), the non-fused path, and a forward without a gradient
for dt, (B_, T_, U_, V_) in ((torch.float32, (3, 9, 6, 29)), (torch.float16, (2, 5, 4, 4097)),
                             (torch.float16, (2, 3, 1030, 3))):
    lg = torch.randn(B_, T_, U_, V_, device="cuda", dtype=dt, requires_grad=True)
    tl = torch.tensor([T_] + [max(1, T_ - 2)] * (B_ - 1), dtype=torch.int32, device="cuda")
    ul = torch.tensor([max(0, U_ - 3)] * (B_ - 1) + [U_ - 1], dtype=torch.int32, device="cuda")
    tg = torch.randint(0, V_ - 1, (B_, U_ - 1), dtype=torch.int32, device="cuda")
    F.rnnt_loss(lg, tg, tl, ul).backward()
    F.rnnt_loss(lg, tg, tl, ul, clamp=0.1, fused_log_softmax=False, reduction="none").sum().backward()
    with torch.no_grad():
        F.rnnt_loss(lg, tg, tl, ul, blank=0)
# forced_align: a ragged float16 batch with int64 targets, a row without targets and padding frames
lp_ = torch.log_softmax(torch.randn(3, 40, 7, device="cuda"), -1).half()
tg_ = torch.randint(1, 7, (3, 12), device="cuda")
F.forced_align(lp_, tg_, torch.tensor([40, 31, 9], device="cuda"), torch.tensor([12, 0, 4], device="cuda"))
# cuda_ctc_decoder: a ragged batch with an empty row, a row that stops early and merges from a small vocabulary
from audio_b200.models.decoder import cuda_ctc_decoder  # noqa: E402
lp_ = torch.log_softmax(torch.randn(4, 50, 6, device="cuda") * 3, -1)
cuda_ctc_decoder(list("abcdef"), nbest=5, beam_size=5)(lp_, torch.tensor([50, 0, 17, 1], dtype=torch.int32,
                                                                          device="cuda"))
torch.cuda.synchronize()
print("done")
