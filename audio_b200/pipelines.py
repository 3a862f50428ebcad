"""The RNN-T feature extractors of ``torchaudio.pipelines`` (``RNNTBundle.get_feature_extractor()`` /
``get_streaming_feature_extractor()``, pipelines/rnnt_pipeline.py:20-47, :80-105, :310-343) and the batched form of the
same chain in the Emformer / Conformer RNN-T training recipes (examples/asr/librispeech_conformer_rnnt/transforms.py:
13-78, examples/asr/emformer_rnnt/common.py:24-28, :81-92):

    MelSpectrogram -> transpose -> piecewise log of (x * 32767^2) -> (x - mean) * invstddev [-> right padding]

as one launch of the fused front end (``b200audio::rnnt_features``), with no host round trip.  This module is
unrelated to :mod:`audio_b200.pipeline`, the host-side loader pipeline.  Nothing here downloads: the global statistics
are read from a local JSON file with ``mean`` and ``invstddev`` lists.
"""
from __future__ import annotations

import json
import math
from typing import Optional, Sequence, Tuple, Union

import torch
from torch import Tensor

from . import _lib, _ops
from ._plans import (_no_autograd, _require_cuda_f32, _RNNTFunction, _wants_grad, StampCache, is_feature_differentiable,
                     pack_rows)
from .transforms import MelSpectrogram

__all__ = ["RNNTFeatureExtractor"]

# rnnt_pipeline.py:16-17: 32767^2 as the reference computes it; the kernels multiply by its float32 value, 1073676288
_decibel = 2 * 20 * math.log10(torch.iinfo(torch.int16).max)
_gain = pow(10, 0.05 * _decibel)


class _GlobalStatsNormalization(torch.nn.Module):
    """Holds the ``mean`` / ``invstddev`` buffers of rnnt_pipeline.py:35-47 (the normalisation itself runs in the
    fused kernel)."""

    def __init__(self, global_stats_path: str) -> None:
        super().__init__()
        with open(global_stats_path) as f:
            blob = json.loads(f.read())
        self.register_buffer("mean", torch.tensor(blob["mean"]))
        self.register_buffer("invstddev", torch.tensor(blob["invstddev"]))


class RNNTFeatureExtractor(torch.nn.Module):
    r"""RNN-T features of a 16 kHz waveform in one launch: ``(time,) -> ((frames + right_padding, n_mels), length)``.

    The reference's non-streaming extractor is ``right_padding=4`` (its bundles' ``_right_padding``), the streaming one
    ``right_padding=0``.  The ``state_dict`` keys are the reference extractor's (``pipeline.0.spectrogram.window``,
    ``pipeline.0.mel_scale.fb``, ``pipeline.3.mean``, ``pipeline.3.invstddev``), so its state loads as is.

    The piecewise log is the reference's two in-place statements, which make three pieces: ``x / e`` for
    ``x <= e``, ``log(x) / e`` for ``e < x <= e^e`` and ``log(x)`` above; silence gives ``(0 - mean) * invstddev``.

    Inside ``audio_b200.differentiable(features=True)`` a 1-D waveform (and ``forward_batch`` without ``lengths``)
    that requires grad gets its gradient.
    """

    def __init__(self, global_stats_path: str, sample_rate: int = 16000, n_fft: int = 400, n_mels: int = 80,
                 hop_length: int = 160, right_padding: int = 4) -> None:
        super().__init__()
        if right_padding < 0:
            raise ValueError(f"right_padding must be non-negative, got {right_padding}")
        mel = MelSpectrogram(sample_rate=sample_rate, n_fft=n_fft, n_mels=n_mels, hop_length=hop_length)
        # indices 1, 2 (and 4) of the reference's Sequential are the parameterless transpose, log and pad steps
        self.pipeline = torch.nn.ModuleDict({"0": mel, "3": _GlobalStatsNormalization(global_stats_path)})
        self.right_padding = int(right_padding)
        self._stats = StampCache()

    @classmethod
    def from_bundle(cls, bundle, global_stats_path: str, streaming: bool = False) -> "RNNTFeatureExtractor":
        """The extractor of an ``RNNTBundle``-like object, read by duck typing (``sample_rate``, ``n_fft``, ``n_mels``,
        ``hop_length``, ``_right_padding``); ``global_stats_path`` is a local copy of its statistics file."""
        return cls(global_stats_path, sample_rate=int(bundle.sample_rate), n_fft=int(bundle.n_fft),
                   n_mels=int(bundle.n_mels), hop_length=int(bundle.hop_length),
                   right_padding=0 if streaming else int(bundle._right_padding))

    def _constants(self):
        mel, norm = self.pipeline["0"], self.pipeline["3"]
        return (("window", mel.spectrogram.window), ("fb", mel.mel_scale.fb), ("mean", norm.mean),
                ("invstddev", norm.invstddev))

    def _packed_stats(self, device: torch.device) -> Tensor:
        """[2][n_mels] (mean, invstddev) on the workspace's device, rebuilt only when either buffer changes."""
        norm = self.pipeline["3"]
        return self._stats.get((norm.mean, norm.invstddev), lambda mean, invstd: self._pack_stats(mean, invstd, device))

    def _pack_stats(self, mean: Tensor, invstd: Tensor, device: torch.device) -> Tensor:
        n_mels = self.pipeline["0"].mel_scale.fb.shape[1]
        for name, t in (("mean", mean), ("invstddev", invstd)):
            _require_cuda_f32(t, name)
            if t.device != device:
                raise RuntimeError(f"audio_b200: {name} is on {t.device} but the window is on {device}")
            if t.numel() != n_mels:
                raise RuntimeError(f"audio_b200: {name} has {t.numel()} elements, expected n_mels={n_mels}")
        with torch.no_grad():
            return torch.stack([mean.reshape(-1), invstd.reshape(-1)]).contiguous()

    def _prepare(self, waveform: Tensor, lengths_given: bool = False):
        """The plan, workspace, packed statistics and whether the call carries a gradient."""
        mel = self.pipeline["0"]
        plan = mel._fused_plan()
        _require_cuda_f32(waveform, "waveform")
        grad = _wants_grad(waveform, self._constants(), is_feature_differentiable)
        if grad and lengths_given:
            raise RuntimeError(
                "audio_b200: RNNTFeatureExtractor.forward_batch computes no gradient for a ragged batch (lengths "
                "given); call it without lengths on equal-length rows, or detach() the waveforms")
        if not grad:
            _no_autograd(waveform)
        ws = plan.workspace(mel.spectrogram.window, mel.mel_scale.fb, None)
        return plan, ws, self._packed_stats(ws.device), grad

    def _run(self, waveform: Tensor, pad_frames: int) -> Tuple[Tensor, int]:
        """(rows, T + pad_frames, n_mels) features of equal-length rows, and T."""
        plan, ws, stats, grad = self._prepare(waveform)
        flat, stride, frames = plan._pack(ws, waveform)
        desc_i, desc_f = plan._packed_desc()
        if grad:
            norm = self.pipeline["3"]
            out = _RNNTFunction.apply(flat, ws, desc_i, desc_f, stats, norm.mean, norm.invstddev, _gain, frames,
                                      pad_frames, stride)
        else:
            out, _ = _ops.rnnt_features(flat, ws, desc_i, desc_f, None, stats, _gain, frames, pad_frames, stride, False)
        return out, frames

    def forward(self, input: Tensor) -> Tuple[Tensor, Tensor]:
        """``(time,)`` waveform -> ``(features, length)``: contiguous ``(T + right_padding, n_mels)`` float32 features
        (the padding rows are zeros) and ``torch.tensor([T + right_padding])`` (int64, on the CPU)."""
        if input.dim() != 1:
            raise ValueError(f"RNNTFeatureExtractor expects a 1-D waveform, got shape {tuple(input.shape)}; "
                             "use forward_batch for a batch")
        out, frames = self._run(input, self.right_padding)
        features = out[0]
        return features, torch.tensor([features.shape[0]])

    def forward_batch(self, waveforms: Tensor,
                      lengths: Optional[Union[Tensor, Sequence[int]]] = None) -> Tuple[Tensor, Tensor]:
        """The recipes' ``_extract_features`` followed by the piecewise log and the normalisation (no SpecAugment):
        ``(B, L)`` waveforms, row r using its first ``lengths[r]`` samples (all ``L`` when ``lengths`` is None) ->
        ``((B, T_max, n_mels) features, (B,) int32 CPU frame counts)``.  Frames past a row's count hold the features of
        zero mel values, ``(0 - mean) * invstddev``, as the recipes' zero-padded mel batch does.

        ``lengths`` is host-side (a CPU tensor or a sequence of ints); it reaches the device without a host sync.  No
        right padding is added (the recipes add none)."""
        if waveforms.dim() != 2:
            raise ValueError(f"forward_batch expects (batch, time) waveforms, got shape {tuple(waveforms.shape)}")
        if lengths is None:
            out, frames = self._run(waveforms, 0)
            return out, torch.full((waveforms.shape[0],), frames, dtype=torch.int32)
        if isinstance(lengths, Tensor):
            if lengths.device.type != "cpu":
                raise ValueError("audio_b200: lengths must be a CPU tensor or a sequence (reading a device tensor "
                                 "would synchronise the host)")
            if lengths.dim() != 1 or lengths.is_floating_point() or lengths.is_complex():
                raise ValueError(f"lengths must be a 1-D integer tensor, got {lengths.dtype} of shape "
                                 f"{tuple(lengths.shape)}")
            lens = [int(v) for v in lengths.tolist()]
        else:
            lens = [int(v) for v in lengths]
        rows, total = waveforms.shape
        if len(lens) != rows:
            raise ValueError(f"lengths has {len(lens)} entries for a batch of {rows} waveforms")
        plan, ws, stats, _ = self._prepare(waveforms, lengths_given=True)
        if waveforms.device != ws.device:
            raise RuntimeError(f"audio_b200: waveform is on {waveforms.device} but the module buffers are on {ws.device}")
        d = plan.desc
        frames = []
        for r, n in enumerate(lens):
            if n < 0 or n > total:
                raise ValueError(f"lengths[{r}] = {n} is outside [0, {total}]")
            ext = n + 2 * d.pad
            half = d.n_fft // 2
            if d.center and ((d.pad_mode == _lib.PAD_MODE["reflect"] and half >= ext) or
                             (d.pad_mode == _lib.PAD_MODE["circular"] and half > ext)):
                # what torch.stft raises for the utterance on its own
                raise RuntimeError(
                    f"audio_b200: padding size n_fft//2={half} should be less than the input length {ext} for "
                    f"pad_mode reflect/circular (torch.stft raises the same way) (lengths[{r}] = {n})")
            t = plan.frames(n)
            if t < 1:
                raise RuntimeError(f"audio_b200: lengths[{r}] = {n} samples is too short for n_fft={d.n_fft}")
            frames.append(t)
        t_max = max(frames) if frames else 0
        flat, stride = pack_rows(waveforms)
        dev_lengths = torch.tensor(lens, dtype=torch.int64)
        if rows > 0:
            dev_lengths = dev_lengths.pin_memory().to(ws.device, non_blocking=True)
        desc_i, desc_f = plan._packed_desc()
        out, _ = _ops.rnnt_features(flat, ws, desc_i, desc_f, dev_lengths, stats, _gain, t_max, 0, stride, False)
        return out, torch.tensor(frames, dtype=torch.int32)
