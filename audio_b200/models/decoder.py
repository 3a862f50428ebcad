"""GPU CTC prefix beam search with torchaudio's ``cuda_ctc_decoder`` interface, on ``csrc/ctc_decoder.cu``.

``cuda_ctc_decoder(tokens, nbest, beam_size, blank_skip_threshold)`` builds a :class:`CUCTCDecoder`; calling it on
float32 log-probabilities ``(B, T, V)`` and int32 lengths ``(B,)`` on one CUDA device returns, per sequence, the
``nbest`` best :class:`CUCTCHypothesis` (``tokens``: an int32 CPU tensor, ``words``: vocabulary entries, ``score``: a
0-d float32 tensor).  One kernel launch decodes the batch; its outputs come back in a single device-to-host copy.

Where the interfaces differ (INTEGRATION.md): a beam outside [1, 128] once clamped to the vocabulary, or above
``log_prob.shape[2]``, raises ``ValueError``, as does an ``encoder_out_lens`` entry outside [0, T]; a sequence with no
frame below the blank-skip threshold decodes to empty hypotheses scored 0.0; among bit-equal keys the lower
``beam * V + token`` is kept (a beam staying put counts as token 0); NaN keys rank below every number.
"""
from __future__ import annotations

import math
from typing import List, NamedTuple, Optional, Union

import torch

from .. import _lib

__all__ = ["CUCTCHypothesis", "CUCTCDecoder", "cuda_ctc_decoder"]

_DEFAULT_BLANK_SKIP_THRESHOLD = 0.95


def _get_vocab_list(path: str) -> List[str]:
    """The first whitespace-separated field of every line of a UTF-8 token file."""
    with open(path, encoding="utf-8") as fh:
        return [line.split()[0] for line in fh]


class CUCTCHypothesis(NamedTuple):
    """One decoded sequence."""

    tokens: List[int]
    """Token ids of the hypothesis, blanks and repeats removed: an int32 tensor of shape ``(L,)``."""

    words: List[str]
    """``vocab_list[i]`` for each token id ``i``."""

    score: float
    """The hypothesis's log-probability in the beam search (a 0-d float32 tensor)."""


class CUCTCDecoder:
    """Batched CTC prefix beam search on a CUDA device; build it with :func:`cuda_ctc_decoder`.

    Args:
        vocab_list: the token of each class id; class 0 is the blank.
        blank_id: must be 0.
        beam_size: prefixes kept per step, clamped to ``len(vocab_list)``; at most 128.
        nbest: hypotheses returned per sequence, best first.
        blank_skip_threshold: a frame whose blank probability is at least this is skipped (in [0, 1]).
        cuda_stream: the stream the decoder runs on; by default the current stream when the decoder is made.
    """

    def __init__(
        self,
        vocab_list: List[str],
        blank_id: int = 0,
        beam_size: int = 10,
        nbest: int = 1,
        blank_skip_threshold: float = _DEFAULT_BLANK_SKIP_THRESHOLD,
        cuda_stream: Optional[torch.cuda.Stream] = None,
    ):
        if cuda_stream and not isinstance(cuda_stream, torch.cuda.streams.Stream):
            raise AssertionError("cuda_stream must be torch.cuda.streams.Stream")
        # Without a CUDA device the stream is resolved at the first call, so that a decoder (and its argument errors)
        # can be made on a machine without a GPU.
        if cuda_stream:
            self._stream = cuda_stream
        else:
            self._stream = torch.cuda.current_stream() if torch.cuda.is_available() else None
        if blank_id != 0:
            raise AssertionError("blank_id must be 0")
        if not 0 <= blank_skip_threshold <= 1:
            raise AssertionError("blank_skip_threshold must be between 0 and 1")
        self.blank_id = blank_id
        self.space_id = 0
        self.vocab_list = vocab_list
        self.nbest = nbest
        self.blank_skip_threshold = math.log(blank_skip_threshold)  # math.log(0) raises ValueError, as torchaudio's
        self.beam_size = min(beam_size, len(vocab_list))
        if not 1 <= self.beam_size <= _lib.CTC_DECODER_MAX_BEAM:
            raise ValueError(f"beam_size must be in [1, {_lib.CTC_DECODER_MAX_BEAM}] after clamping to the vocabulary "
                             f"size (got {self.beam_size})")
        self._ws = None  # device workspace, reused by later calls that need no more

    def _check(self, log_prob: torch.Tensor, lengths: torch.Tensor) -> None:
        # torchaudio's messages and order
        for bad, msg in (
            (lengths.dtype != torch.int32, "encoder_out_lens must be torch.int32"),
            (log_prob.dtype != torch.float32, "log_prob must be torch.float32"),
            (not log_prob.is_cuda, "log_prob must be cuda tensor"),
            (not lengths.is_cuda, "encoder_out_lens must be cuda tensor"),
            (log_prob.device != lengths.device, "log_prob and encoder_out_lens must be on the same device"),
            (not log_prob.is_contiguous(), "log_prob must be contiguous"),
            (not lengths.is_contiguous(), "encoder_out_lens must be contiguous"),
        ):
            if bad:
                raise RuntimeError(msg)
        if log_prob.dim() != 3:
            raise ValueError(f"log_prob must be (batch, frame, num_tokens); got shape {tuple(log_prob.shape)}")
        batch, _, vocab = log_prob.shape
        if lengths.dim() != 1 or lengths.numel() != batch:
            raise ValueError(f"encoder_out_lens must have shape ({batch},); got {tuple(lengths.shape)}")
        if self.beam_size > vocab:
            raise ValueError(f"beam_size {self.beam_size} is above log_prob.shape[2] = {vocab}")
        if vocab > _lib.CTC_DECODER_MAX_VOCAB:
            raise ValueError(f"log_prob.shape[2] = {vocab} is above the supported {_lib.CTC_DECODER_MAX_VOCAB}")

    def __call__(self, log_prob: torch.Tensor, encoder_out_lens: torch.Tensor) -> List[List[CUCTCHypothesis]]:
        """Decode ``log_prob`` ``(B, T, V)`` (float32) over the first ``encoder_out_lens[b]`` (int32) frames of each
        sequence; returns ``B`` lists of ``nbest`` hypotheses, best first."""
        self._check(log_prob, encoder_out_lens)
        batch, max_t, vocab = log_prob.shape
        if batch == 0:
            return []
        dev = log_prob.device
        stream = self._stream if self._stream is not None else torch.cuda.current_stream(dev)
        beam = self.beam_size
        desc = _lib.CtcDecoderDesc(batch, max_t, vocab, beam, self.blank_skip_threshold)
        lib = _lib.lib()
        need = lib.b200a_ctc_decoder_workspace_bytes(desc)
        nb = batch * beam
        with torch.cuda.device(dev), torch.cuda.stream(stream):
            if self._ws is None or self._ws.device != dev or self._ws.numel() < need:
                self._ws = torch.empty(need, dtype=torch.uint8, device=dev)
            # one int32 block: status [B] | lengths [B][beam] | scores [B][beam] (float32 bits) | tokens [B][beam][T]
            out = torch.empty(batch + 2 * nb + nb * max_t, dtype=torch.int32, device=dev)
            status, lens, scores, tokens = out.split([batch, nb, nb, nb * max_t])
            rc = lib.b200a_ctc_decoder_run(desc, log_prob.data_ptr(), encoder_out_lens.data_ptr(), tokens.data_ptr(),
                                           lens.data_ptr(), scores.data_ptr(), status.data_ptr(), self._ws.data_ptr(),
                                           self._ws.numel(), stream.cuda_stream)
            _lib.check(rc, "ctc_decoder")
            host = out.cpu()
        status, lens, scores, tokens = host.split([batch, nb, nb, nb * max_t])
        if bool(status.any()):
            raise ValueError(f"encoder_out_lens[{int(status.nonzero()[0, 0])}] must be in [0, {max_t}]")
        lens = lens.view(batch, beam).tolist()
        scores = scores.view(torch.float32).view(batch, beam)
        tokens = tokens.view(batch, beam, max_t)
        vocab_list = self.vocab_list
        result = []
        for b in range(batch):
            row = []
            for r in range(self.nbest):
                ids = tokens[b, r, : lens[b][r]]  # an IndexError past the beam, as torchaudio's indexing gives
                row.append(CUCTCHypothesis(ids, [vocab_list[i] for i in ids.tolist()], scores[b, r]))
            result.append(row)
        return result


def cuda_ctc_decoder(
    tokens: Union[str, List[str]],
    nbest: int = 1,
    beam_size: int = 10,
    blank_skip_threshold: float = _DEFAULT_BLANK_SKIP_THRESHOLD,
) -> CUCTCDecoder:
    """Make a :class:`CUCTCDecoder` from a token list, or from the path of a file with one token per line (its first
    field); the other arguments are :class:`CUCTCDecoder`'s."""
    vocab = _get_vocab_list(tokens) if isinstance(tokens, str) else tokens
    return CUCTCDecoder(vocab_list=vocab, beam_size=beam_size, nbest=nbest, blank_skip_threshold=blank_skip_threshold)
