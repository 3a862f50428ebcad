"""Integer bookkeeping of the front-end path (pure Python, no torch).

Every function here has a C twin exported from ``libb200audio.so``
(``include/b200audio.h``: ``b200a_num_frames``, ``b200a_resample_len``,
``b200a_resample_width``, ``b200a_pad_index``); ``tests/test_bookkeeping.py``
checks both against the reference's shapes bit-exactly (tests/golden/ref_integers.npz).

Reference call sites (relative to pytorch/audio):
  * frame count      -- torch.stft as called at src/torchaudio/functional/functional.py:123-134
  * resample lengths -- src/torchaudio/functional/functional.py:1359, 1424-1428
"""
from __future__ import annotations

import math
import struct

PAD_MODES = ("reflect", "constant", "replicate", "circular")


def num_frames(length: int, n_fft: int, hop: int, center: bool, pad: int = 0) -> int:
    """Number of STFT frames, or -1 when the padded signal is shorter than n_fft."""
    span = length + 2 * pad + (2 * (n_fft // 2) if center else 0)
    if span < n_fft:
        return -1
    return 1 + (span - n_fft) // hop


def pad_index(i: int, n: int, mode: int) -> int:
    """Map an index of the centre-padded signal back into [0, n); -1 == zero."""
    if 0 <= i < n:
        return i
    if mode == 1:
        return -1
    if mode == 0:
        return -i if i < 0 else 2 * (n - 1) - i
    if mode == 2:
        return 0 if i < 0 else n - 1
    return i % n


def resample_ratio(orig_freq: int, new_freq: int):
    """(orig', new', gcd) with the common factor removed (transforms/_transforms.py:948)."""
    g = math.gcd(int(orig_freq), int(new_freq))
    return int(orig_freq) // g, int(new_freq) // g, g


def resample_width(orig_r: int, new_r: int, lowpass_filter_width: int, rolloff: float) -> int:
    """Half-width (in input samples) of the FIR, functional.py:1359."""
    return math.ceil(lowpass_filter_width * orig_r / (min(orig_r, new_r) * rolloff))


def resample_len(length: int, orig_r: int, new_r: int) -> int:
    """Output length, functional.py:1427: torch.ceil(torch.as_tensor(new*L/orig)) -- the python
    float quotient is rounded to float32 (default dtype) before the ceil."""
    q = struct.unpack("f", struct.pack("f", new_r * length / orig_r))[0]
    return int(math.ceil(q))


def shard_bounds(total: int, world: int, rank: int):
    """Contiguous, balanced [begin, end) slice of ``total`` utterances for ``rank``."""
    base, extra = divmod(total, world)
    begin = rank * base + min(rank, extra)
    return begin, begin + base + (1 if rank < extra else 0)
