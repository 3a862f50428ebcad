"""CPU tests of the torch binding layer: descriptor packing derived from the ctypes structures, the Meta
implementation of every ``b200audio`` op, and the rebuild rule of the workspace caches."""
import ctypes
import gc
import weakref

import pytest
import torch

from audio_b200 import _lib, _ops
from audio_b200._plans import StampCache

DESCRIPTORS = (_lib.FrontendDesc, _lib.KaldiDesc, _lib.VadDesc)


def _distinct(cls):
    """A ``cls`` with every field set to its own non-zero value (floats exact in float32)."""
    d = cls()
    for i, (name, ctype) in enumerate(cls._fields_, start=1):
        setattr(d, name, 0.25 + i if ctype in (ctypes.c_float, ctypes.c_double) else 100 + i)
    return d


@pytest.mark.parametrize("cls", DESCRIPTORS, ids=lambda c: c.__name__)
def test_pack_unpack_round_trip(cls):
    d = _distinct(cls)
    ints, floats = _ops.pack(d)
    back = _ops.unpack(cls, ints, floats)
    for name, _ in cls._fields_:
        assert getattr(back, name) == getattr(d, name), name
    assert bytes(back) == bytes(d)


@pytest.mark.parametrize("cls", DESCRIPTORS, ids=lambda c: c.__name__)
def test_packed_lists_cover_every_field(cls):
    d = _distinct(cls)
    ints, floats = _ops.pack(d)
    assert len(ints) + len(floats) == len(cls._fields_)
    assert all(type(v) is int for v in ints) and all(type(v) is float for v in floats)
    # every value is distinct, so this says each field is packed exactly once, in struct order within its list
    kinds = [(ctype in (ctypes.c_float, ctypes.c_double), getattr(d, name)) for name, ctype in cls._fields_]
    assert ints == [v for is_float, v in kinds if not is_float]
    assert floats == [v for is_float, v in kinds if is_float]
    for name, _ in cls._fields_:
        v = getattr(d, name)
        assert (ints if type(v) is int else floats)[_ops.field_index(cls, name)] == v


def test_unpack_refuses_lists_of_the_wrong_length():
    ints, floats = _ops.pack(_distinct(_lib.FrontendDesc))
    with pytest.raises(ValueError, match="FrontendDesc"):
        _ops.unpack(_lib.FrontendDesc, ints[:-1], floats)
    with pytest.raises(ValueError, match="FrontendDesc"):
        _ops.unpack(_lib.FrontendDesc, ints, floats + [1.0])


def test_pointer_descriptor_is_not_packable():
    with pytest.raises(TypeError, match="FftconvolveDesc"):
        _ops.pack(_lib.FftconvolveDesc())


# ---- Meta implementations ------------------------------------------------------------------------------------------
def _meta(*shape, dtype=torch.float32):
    return torch.empty(shape, dtype=dtype, device="meta")


def _frontend_lists():
    d = _lib.FrontendDesc(n_fft=400, win_length=400, hop=160, n_mels=80, n_mfcc=13, power=2.0)
    return _ops.pack(d)


def _meta_cases():
    """(op name, call on meta tensors, the (shape, dtype) of each output the CUDA implementation allocates)."""
    di, df = _frontend_lists()
    ki, kf = _ops.pack(_lib.KaldiDesc(window_size=400, window_shift=160, padded_size=512, out_width=23))
    vi, vf = _ops.pack(_lib.VadDesc(channels=2, dft_len=1024))
    ws = _meta(64, dtype=torch.uint8)
    rows, length, frames, f32 = 3, 16000, 98, torch.float32
    idx = _meta(rows, dtype=torch.int64)
    return [
        ("frontend_run", lambda: _ops.frontend_run(_meta(rows, length), ws, di, df, _lib.STAGE_COMPLEX, frames, 201, length,
                                                   None, 1), [((rows, frames, 201, 2), f32)]),
        ("frontend_backward", lambda: _ops.frontend_backward(_meta(rows, length), ws, di, df, _lib.STAGE_MEL, length,
                                                             _meta(rows, frames, 80)), [((rows, length), f32)]),
        ("istft_backward", lambda: _ops.istft_backward(_meta(rows, length), ws, di, df, 0, frames),
         [((rows, frames, 201, 2), f32)]),
        ("mfcc_finish", lambda: _ops.mfcc_finish(_meta(rows, frames, 80), ws, di, df, None, 1, 80.0),
         [((rows, frames, 13), f32)]),
        ("mfcc_backward", lambda: _ops.mfcc_backward(_meta(rows, frames, 13), _meta(rows, frames, 80),
                                                     _meta(rows, frames, 80), None, ws, di, df, 1, -1.0),
         [((rows, frames, 80), f32)]),
        ("amplitude_to_db_backward", lambda: _ops.amplitude_to_db_backward(_meta(rows, 80, frames), _meta(rows, 80, frames),
                                                                           None, 0, 10.0, 1e-10, 0.0, -1.0),
         [((rows, 80, frames), f32)]),
        ("apply_fbank_backward", lambda: _ops.apply_fbank_backward(_meta(rows, frames, 80), _meta(201, 80)),
         [((rows, frames, 201), f32)]),
        ("ratio_backward", lambda: _ops.ratio_backward(_meta(rows, frames), _meta(rows, frames, 2)),
         [((rows, frames, 2), f32)]),
        ("resample_run", lambda: _ops.resample_run(_meta(rows, 44100), ws, _meta(160, 475), 441, 160, 17, 44100, 16000,
                                                   16160), [((rows, 16160), f32)]),
        ("resample_backward", lambda: _ops.resample_backward(_meta(rows, 16000), ws, 441, 160, 17, 44100),
         [((rows, 44100), f32)]),
        ("kaldi_run", lambda: _ops.kaldi_run(_meta(rows, length), ws, di, df, ki, kf, _lib.STAGE_MEL, frames, 23, length),
         [((rows, frames, 23), f32)]),
        ("kaldi_backward", lambda: _ops.kaldi_backward(_meta(rows, length), ws, di, df, ki, kf, _lib.STAGE_MEL, length,
                                                       _meta(rows, frames, 23)), [((rows, length), f32)]),
        ("phase_vocoder_backward", lambda: _ops.phase_vocoder_backward(
            _meta(rows, 201, frames, dtype=torch.complex64), _meta(rows, 75, 201, 2),
            _meta(rows, 201, 75, dtype=torch.complex64), 1.3), [((rows, frames, 201, 2), f32)]),
        ("rnnt_features", lambda: _ops.rnnt_features(_meta(1, length), ws, di, df, None, _meta(2, 80), 1.0, frames, 4,
                                                     length, True), [((1, frames + 4, 80), f32), ((1, frames, 80), f32)]),
        ("rnnt_features_backward", lambda: _ops.rnnt_features_backward(_meta(2, 80), 1.0, _meta(rows, frames, 80),
                                                                       _meta(rows, frames, 80)),
         [((rows, frames, 80), f32)]),
        ("inverse_mel", lambda: _ops.inverse_mel(_meta(rows, 80, frames), ws, 201), [((rows, frames, 201), f32)]),
        ("inverse_mel_backward", lambda: _ops.inverse_mel_backward(_meta(rows, frames, 201), _meta(rows, 80, frames), ws,
                                                                   201), [((rows, frames, 80), f32)]),
        ("lfilter", lambda: _ops.lfilter(_meta(2, rows, length), _meta(rows, 3), _meta(rows, 3), True, False, True),
         [((2, rows, length), f32), ((2, rows, length), f32)]),
        ("lfilter_backward", lambda: _ops.lfilter_backward(_meta(2, rows, length), _meta(2, rows, length),
                                                           _meta(2, rows, length), _meta(rows, 3), _meta(rows, 3), True,
                                                           False),
         [((2, rows, length), f32), ((rows, 3), f32), ((rows, 3), f32)]),
        ("fftconvolve", lambda: _ops.fftconvolve(_meta(2, length), _meta(1, 255), idx, idx, 0, length + 254),
         [((rows, length + 254), f32)]),
        ("fftconvolve_backward", lambda: _ops.fftconvolve_backward(_meta(rows, length + 254), _meta(2, length),
                                                                   _meta(1, 255), idx, idx, 0),
         [((rows, length), f32), ((rows, 255), f32)]),
        ("convolve", lambda: _ops.convolve(_meta(2, length), _meta(1, 32), idx, idx, 31, length - 31),
         [((rows, length - 31), f32)]),
        ("convolve_backward", lambda: _ops.convolve_backward(_meta(rows, length - 31), _meta(2, length), _meta(1, 32), idx,
                                                             idx, 31), [((rows, length), f32), ((rows, 32), f32)]),
        ("vad_walk", lambda: _ops.vad_walk(_meta(2, frames, 513), _meta(512), _meta(2, 1024 * 256),
                                           _meta(4096, dtype=torch.uint8), vi, vf, 1024, 0), []),
        ("vad_trigger", lambda: _ops.vad_trigger(_meta(2, frames), _meta(4096, dtype=torch.uint8), vi, vf, 1024, 0),
         [((2, frames), f32)]),
    ]


def test_every_op_has_a_meta_case():
    registered = {n.split("::")[1] for n in torch._C._dispatch_get_all_op_names() if n.startswith("b200audio::")}
    cases = [name for name, _, _ in _meta_cases()]
    assert len(cases) == len(set(cases))
    assert set(cases) == registered


@pytest.mark.parametrize("case", _meta_cases(), ids=lambda c: c[0])
def test_meta_shapes(case):
    name, call, expected = case
    out = call()
    outs = [] if out is None else list(out) if isinstance(out, tuple) else [out]
    assert [(tuple(t.shape), t.dtype) for t in outs] == expected
    assert all(t.device.type == "meta" for t in outs)


# ---- the rebuild rule of the workspace caches ------------------------------------------------------------------------
class _Counter:
    def __init__(self):
        self.calls = 0

    def __call__(self, *tensors):
        self.calls += 1
        return object()


def test_cache_returns_the_same_value_for_an_unmodified_tensor():
    cache, build, t = StampCache(), _Counter(), torch.ones(4)
    v = cache.get((t, None), build)
    assert cache.get((t, None), build) is v and build.calls == 1


def test_cache_rebuilds_after_an_in_place_edit():
    cache, build, t = StampCache(), _Counter(), torch.ones(4)
    v = cache.get((t,), build)
    t.mul_(2.0)
    assert cache.get((t,), build) is not v and build.calls == 2
    assert cache.get((t,), build) is cache.value and build.calls == 2


def test_cache_rebuilds_for_a_different_tensor():
    cache, build, t = StampCache(), _Counter(), torch.ones(4)
    v = cache.get((t,), build)
    assert cache.get((t.clone(),), build) is not v and build.calls == 2


def test_cache_rebuilds_when_a_none_slot_becomes_a_tensor():
    cache, build, t = StampCache(), _Counter(), torch.ones(4)
    v = cache.get((t, None), build)
    assert cache.get((t, torch.ones(2)), build) is not v and build.calls == 2


def test_cache_passes_the_tensors_to_build():
    cache, t, u = StampCache(), torch.ones(4), torch.zeros(2)
    assert cache.get((t, None, u), lambda *args: args) == (t, None, u)


def test_cache_keeps_the_tensors_alive():
    cache, build = StampCache(), _Counter()
    t = torch.ones(4)
    ref = weakref.ref(t)
    cache.get((t,), build)
    del t
    gc.collect()
    assert ref() is not None
    cache.get((torch.zeros(4),), build)  # a new stamp releases the old tensors
    gc.collect()
    assert ref() is None
