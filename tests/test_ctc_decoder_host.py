"""cuda_ctc_decoder without a GPU: the vocabulary file, the constructor's errors and their order, the beam clamp, the
deviations that raise, CPU tensors, the C ABI's descriptor checks, and the pinned log-sum-exp in the kernel's SASS."""
import ctypes
import math
import os
import re
import shutil
import subprocess

import pytest
import torch

from audio_b200 import _lib
from audio_b200.models import decoder as D
from audio_b200.models.decoder import CUCTCDecoder, CUCTCHypothesis, cuda_ctc_decoder
from conftest import ROOT


def test_vocab_file_first_field(tmp_path):
    p = tmp_path / "tokens.txt"
    p.write_text("<blk> 0\n▁the 1\n  a\tb  \nz\n", encoding="utf-8")
    dec = cuda_ctc_decoder(str(p))
    assert dec.vocab_list == ["<blk>", "▁the", "a", "z"]
    assert D._get_vocab_list(str(p)) == dec.vocab_list


def test_defaults_and_attributes():
    dec = cuda_ctc_decoder(["-", "a", "b"] * 10)
    assert (dec.nbest, dec.beam_size, dec.blank_id, dec.space_id) == (1, 10, 0, 0)
    assert dec.blank_skip_threshold == math.log(0.95)
    assert cuda_ctc_decoder(["-", "a", "b"], beam_size=10).beam_size == 3  # clamped to the vocabulary
    dec = cuda_ctc_decoder(["-", "a"], nbest=2, beam_size=2, blank_skip_threshold=1.0)
    assert dec.blank_skip_threshold == 0.0 and dec.nbest == 2
    assert CUCTCHypothesis._fields == ("tokens", "words", "score")


def test_constructor_errors_in_order():
    with pytest.raises(AssertionError, match="cuda_stream must be torch.cuda.streams.Stream"):
        CUCTCDecoder(["-", "a"], blank_id=1, blank_skip_threshold=2.0, cuda_stream=object())
    with pytest.raises(AssertionError, match="blank_id must be 0"):
        CUCTCDecoder(["-", "a"], blank_id=1, blank_skip_threshold=2.0)
    with pytest.raises(AssertionError, match="blank_skip_threshold must be between 0 and 1"):
        CUCTCDecoder(["-", "a"], blank_skip_threshold=2.0)
    with pytest.raises(AssertionError, match="blank_skip_threshold must be between 0 and 1"):
        CUCTCDecoder(["-", "a"], blank_skip_threshold=-0.1)
    with pytest.raises(ValueError, match="math domain error"):  # the reference's math.log(0)
        CUCTCDecoder(["-", "a"], blank_skip_threshold=0.0)


@pytest.mark.parametrize("beam,vocab", [(0, 5), (-3, 5), (129, 200), (10, 0)])
def test_invalid_beam_raises_at_construction(beam, vocab):
    with pytest.raises(ValueError, match="beam_size"):
        cuda_ctc_decoder([str(i) for i in range(vocab)], beam_size=beam)


def test_beam_128_and_clamped_200_are_accepted():
    assert cuda_ctc_decoder([str(i) for i in range(200)], beam_size=128).beam_size == 128
    assert cuda_ctc_decoder([str(i) for i in range(100)], beam_size=200).beam_size == 100


def test_call_errors_before_any_device_work():
    dec = cuda_ctc_decoder([str(i) for i in range(8)], beam_size=4)
    lp = torch.zeros(2, 5, 8)
    n = torch.full((2,), 5, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="encoder_out_lens must be torch.int32"):
        dec(lp, n.long())
    with pytest.raises(RuntimeError, match="log_prob must be torch.float32"):
        dec(lp.double(), n)
    with pytest.raises(RuntimeError, match="log_prob must be cuda tensor"):
        dec(lp, n)


def _desc(**kw):
    f = dict(batch=2, max_t=10, vocab=50, beam=10, threshold=-0.05)
    f.update(kw)
    return _lib.CtcDecoderDesc(**f)


@pytest.mark.parametrize("bad", [dict(batch=0), dict(max_t=-1), dict(vocab=0), dict(vocab=(1 << 24) + 1),
                                 dict(beam=0), dict(beam=129), dict(beam=51), dict(threshold=float("nan"))])
def test_c_abi_rejects_bad_descriptors(bad):
    lib = _lib.lib()
    d = _desc(**bad)
    assert lib.b200a_ctc_decoder_workspace_bytes(ctypes.byref(d)) == 0
    p = ctypes.c_void_p(16)
    rc = lib.b200a_ctc_decoder_run(ctypes.byref(d), p, p, p, p, p, p, p, 1 << 30, None)
    assert rc == _lib.EINVAL


def test_c_abi_workspace_and_null_checks():
    lib = _lib.lib()
    d = _desc()
    need = lib.b200a_ctc_decoder_workspace_bytes(ctypes.byref(d))
    assert need >= 2 * 10 * 4 + 2 * 10 * 10 * 8
    p = ctypes.c_void_p(16)
    assert lib.b200a_ctc_decoder_run(ctypes.byref(d), p, None, p, p, p, p, p, need, None) == _lib.EINVAL
    assert lib.b200a_ctc_decoder_run(ctypes.byref(d), p, p, p, p, p, p, p, need - 1, None) == _lib.EWORKSPACE
    z = _desc(max_t=0)  # no frames: log_prob and tokens may be null
    assert lib.b200a_ctc_decoder_run(ctypes.byref(z), None, p, None, p, p, p, p, 0, None) == _lib.EWORKSPACE


def test_kernel_sass_has_the_pinned_lse():
    """The reference's lse compiles to FMUL by log2(e), non-ftz MUFU.EX2, FADD 1, MUFU.LG2 and one FFMA by ln 2 onto
    the max; the decode kernel must contain that sequence."""
    obj = os.path.join(ROOT, "audio_b200", "build", "ctc_decoder.o")
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(obj) or not os.path.exists(tool):
        pytest.skip("needs the built object and cuobjdump")
    sass = subprocess.run([tool, "-sass", obj], capture_output=True, text=True, check=True).stdout
    ops = [re.sub(r"^\s*/\*[0-9a-f]+\*/\s*", "", ln).split(";")[0].strip() for ln in sass.splitlines()
           if re.match(r"^\s*/\*[0-9a-f]+\*/", ln)]
    found = 0
    for i, op in enumerate(ops):
        if not re.search(r"\bFMUL R\d+, R\d+, 1\.4426950216293334961$", op):
            continue
        reg = op.split()[1].rstrip(",")
        window = ops[i: i + 12]
        ex2 = next((k for k, o in enumerate(window) if re.search(rf"MUFU\.EX2 R\d+, {reg}$", o)), None)
        if ex2 is None or any(".FTZ" in o for o in window[: ex2 + 1]):
            continue
        e = window[ex2].split()[1].rstrip(",")
        add = next((k for k, o in enumerate(window) if re.search(rf"FADD R\d+, {e}, 1$", o)), None)
        if add is None:
            continue
        s = window[add].split()[1].rstrip(",")
        lg = next((k for k, o in enumerate(window) if re.search(rf"MUFU\.LG2 R\d+, {s}$", o)), None)
        if lg is None:
            continue
        lreg = window[lg].split()[1].rstrip(",")
        if any(re.search(rf"FFMA R\d+, {lreg}, 0\.69314718246459960938, R\d+$", o) for o in window[lg:]):
            found += 1
    assert found >= 4, found
