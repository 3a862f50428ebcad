"""The numpy forced-alignment oracle (tests/forced_align_oracle.py) against the reference CPU's paths and scores in
tests/golden/forced_align_ref_cases.npz, merge_tokens against the reference's spans, and the argument checks of the
forced_align C ABI, none of which needs a GPU."""
import ctypes

import numpy as np
import pytest
import torch

import forced_align_oracle as O
from audio_b200 import _build, _lib
from audio_b200.functional import TokenSpan, merge_tokens
from conftest import _load


@pytest.fixture(scope="module")
def ref():
    return _load("forced_align_ref_cases.npz")


def _keys(ref, prefix):
    return sorted(int(k[len(prefix):]) for k in ref if k.startswith(prefix) and k[len(prefix):].isdigit())


def test_oracle_matches_hand_worked_fixtures(ref):
    for i in range(4):
        p, s = O.align(ref[f"fx_{i}_lp"][0], ref[f"fx_{i}_tg"][0], 5)
        assert np.array_equal(p, ref[f"fx_{i}_path"]) and np.array_equal(s, ref[f"fx_{i}_score"]), i


def test_oracle_matches_reference_recipes(ref):
    for i in _keys(ref, "rc_"):
        lp, tg, blank = O.case_inputs(ref[f"rc_{i}"])
        p, s = O.align(lp[0], tg[0], blank)
        assert np.array_equal(p, ref[f"path_{i}"]), i
        assert s.dtype == ref[f"score_{i}"].dtype and np.array_equal(s, ref[f"score_{i}"]), i


def test_oracle_matches_reference_batches(ref):
    for i in _keys(ref, "bt_"):
        lp, tg, tl, ul, blank = O.batch_inputs(ref[f"bt_{i}"])
        p, s = O.align_batch(lp, tg, tl, ul, blank)
        assert np.array_equal(p, ref[f"bpath_{i}"]) and np.array_equal(s, ref[f"bscore_{i}"]), i


def test_oracle_empty_targets_are_all_blank():
    lp = np.log(np.full((7, 4), 0.25, dtype=np.float32))
    p, s = O.align(lp, np.zeros(0, dtype=np.int64), 2)
    assert (p == 2).all() and np.array_equal(s, lp[:, 2])


def test_merge_tokens_matches_reference(ref):
    for i in _keys(ref, "rc_"):
        if f"mt_{i}_token" not in ref:
            continue
        blank = int(ref[f"rc_{i}"][4])
        spans = merge_tokens(torch.from_numpy(ref[f"path_{i}"].astype(np.int64)), torch.from_numpy(ref[f"score_{i}"]),
                             blank=blank)
        assert [x.token for x in spans] == ref[f"mt_{i}_token"].tolist()
        assert [x.start for x in spans] == ref[f"mt_{i}_start"].tolist()
        assert [x.end for x in spans] == ref[f"mt_{i}_end"].tolist()
        assert [x.score for x in spans] == ref[f"mt_{i}_score"].tolist()
        assert [len(x) for x in spans] == (ref[f"mt_{i}_end"] - ref[f"mt_{i}_start"]).tolist()


def test_merge_tokens_validation():
    with pytest.raises(ValueError, match="must be 1D Tensor"):
        merge_tokens(torch.zeros(1, 3, dtype=torch.int64), torch.zeros(3))
    with pytest.raises(ValueError, match="must be the same length"):
        merge_tokens(torch.zeros(3, dtype=torch.int64), torch.zeros(4))
    assert merge_tokens(torch.zeros(0, dtype=torch.int64), torch.zeros(0)) == []
    assert merge_tokens(torch.tensor([0, 3, 3, 0, 3]), torch.tensor([0.0, 1.0, 2.0, 0.0, 4.0])) == [
        TokenSpan(3, 1, 3, 1.5), TokenSpan(3, 4, 5, 4.0)]


def test_forced_align_abi_argument_validation_without_gpu():
    _build.build()  # no-op when the .so is fresh
    lib = _lib.lib()
    fake = ctypes.c_void_p(0x1000)  # never dereferenced: every case below returns before a launch
    out = (ctypes.c_int64 * 11)()

    def desc(**kw):
        d = _lib.ForcedAlignDesc(2, 10, 4, 6, 0, _lib.DTYPE_F32, _lib.INDEX_I64, _lib.INDEX_I64)
        for k, v in kw.items():
            setattr(d, k, v)
        return d

    good = desc()
    ws = lib.b200a_forced_align_workspace_bytes(good)
    assert ws > 2 * 10 * 9 // 4
    for bad in (dict(batch=0), dict(max_t=0), dict(max_l=-1), dict(classes=0), dict(blank=6), dict(blank=-1),
                dict(dtype=3), dict(target_dtype=2), dict(length_dtype=-1)):
        assert lib.b200a_forced_align_workspace_bytes(desc(**bad)) == 0, bad
        rc = lib.b200a_forced_align_run(desc(**bad), fake, fake, fake, fake, fake, fake, fake, ws, None)
        assert rc == _lib.EINVAL, bad
        if "blank" not in bad:  # the check takes any blank
            assert lib.b200a_forced_align_check(desc(**bad), fake, fake, fake, out, fake, ws, None) == _lib.EINVAL
    assert lib.b200a_forced_align_run(None, fake, fake, fake, fake, fake, fake, fake, ws, None) == _lib.EINVAL
    for i in range(7):
        ptrs = [fake] * 7
        ptrs[i] = None
        assert lib.b200a_forced_align_run(good, *ptrs, ws, None) == _lib.EINVAL, i
    assert lib.b200a_forced_align_run(good, fake, fake, fake, fake, fake, fake, fake, ws - 1, None) == _lib.EWORKSPACE
    assert lib.b200a_forced_align_check(good, fake, fake, fake, out, fake, 7, None) == _lib.EWORKSPACE
    assert lib.b200a_forced_align_check(good, fake, None, fake, out, fake, ws, None) == _lib.EINVAL
    assert lib.b200a_forced_align_check(good, fake, fake, fake, None, fake, ws, None) == _lib.EINVAL
    assert lib.b200a_forced_align_check(good, None, fake, fake, out, fake, ws, None) == _lib.EINVAL
    capped = desc(max_l=_lib.FORCED_ALIGN_MAX_L)
    assert lib.b200a_forced_align_workspace_bytes(capped) > 0
    over = desc(max_l=_lib.FORCED_ALIGN_MAX_L + 1)
    assert lib.b200a_forced_align_workspace_bytes(over) == 0
    assert lib.b200a_forced_align_run(over, fake, fake, fake, fake, fake, fake, fake, 1 << 40, None) == \
        _lib.EUNSUPPORTED
