"""forced_align and merge_tokens on the GPU: paths and scores equal (torch.equal) to the reference CPU's
(tests/golden/forced_align_ref_cases.npz) and to the numpy oracle (tests/forced_align_oracle.py), which restates the
reference's walk bit for bit."""
import importlib.util
import os
import re

import numpy as np
import pytest
import torch

import audio_b200.functional as F
import forced_align_oracle as O
from audio_b200 import _lib
from conftest import ROOT, _load

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
TORCH_DTYPES = {np.dtype(np.float32): torch.float32, np.dtype(np.float16): torch.float16,
                np.dtype(np.float64): torch.float64}


@pytest.fixture(scope="module")
def ref():
    return _load("forced_align_ref_cases.npz")


def _keys(ref, prefix):
    return sorted(int(k[len(prefix):]) for k in ref if k.startswith(prefix) and k[len(prefix):].isdigit())


def run(lp, tg, tl=None, ul=None, blank=0):
    to = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(DEV)  # noqa: E731
    p, s = F.forced_align(to(lp), to(tg), to(tl), to(ul), blank)
    assert p.dtype == torch.from_numpy(tg).dtype and s.dtype == TORCH_DTYPES[lp.dtype]
    assert not p.requires_grad and not s.requires_grad
    return p.cpu(), s.cpu()


def equal(got, exp):
    return torch.equal(got, torch.from_numpy(np.ascontiguousarray(exp)).to(got.dtype)) and \
        got.dtype == torch.from_numpy(np.asarray(exp)).dtype


def test_hand_worked_fixtures(ref):
    for i in range(4):
        for dt in (np.float32, np.float64, np.float16):
            lp = ref[f"fx_{i}_lp"].astype(dt)
            p, s = run(lp, ref[f"fx_{i}_tg"], blank=5)
            op, os_ = O.align(lp[0], ref[f"fx_{i}_tg"][0], 5)
            assert torch.equal(p[0], torch.from_numpy(op).to(p.dtype)) and torch.equal(s[0], torch.from_numpy(os_))
            if dt == np.float32:
                assert torch.equal(p[0], torch.from_numpy(ref[f"fx_{i}_path"]).to(p.dtype))
                assert torch.equal(s[0], torch.from_numpy(ref[f"fx_{i}_score"]))


def test_reference_recipes(ref):
    for i in _keys(ref, "rc_"):
        lp, tg, blank = O.case_inputs(ref[f"rc_{i}"])
        p, s = run(lp, tg, blank=blank)
        assert torch.equal(p[0], torch.from_numpy(ref[f"path_{i}"]).to(p.dtype)), i
        assert equal(s[0], ref[f"score_{i}"]), i


def test_ragged_batches(ref):
    for i in _keys(ref, "bt_"):
        lp, tg, tl, ul, blank = O.batch_inputs(ref[f"bt_{i}"])
        for lengths in ((tl, ul), (tl.astype(np.int32), ul.astype(np.int32)), (tl, ul.astype(np.int32))):
            p, s = run(lp, tg, *lengths, blank=blank)
            assert torch.equal(p, torch.from_numpy(ref[f"bpath_{i}"]).to(p.dtype)), i
            assert equal(s, ref[f"bscore_{i}"]), i
        for b in range(lp.shape[0]):
            assert (p[b, tl[b]:] == blank).all() and (s[b, tl[b]:] == 0).all()


def test_empty_target_row_and_oracle_batch():
    lp, tg, tl, ul, blank = O.batch_inputs((50, 7, 120, 40, 29, 0, 0, 1, 0, 1))
    ul[3] = 0
    p, s = run(lp, tg, tl, ul, blank)
    op, os_ = O.align_batch(lp, tg, tl, ul, blank)
    assert torch.equal(p, torch.from_numpy(op).to(p.dtype)) and equal(s, os_)
    assert (p[3] == blank).all() and torch.equal(s[3, : tl[3]], torch.from_numpy(lp[3, : tl[3], blank]))


def test_rows_independent_of_neighbours_and_order():
    lp, tg, tl, ul, blank = O.batch_inputs((51, 9, 200, 60, 32, 0, 1, 1, 0, 0))
    p, s = run(lp, tg, tl, ul, blank)
    perm = np.random.default_rng(0).permutation(9)
    pp, sp = run(lp[perm], tg[perm], tl[perm], ul[perm], blank)
    assert torch.equal(pp, p[perm]) and torch.equal(sp, s[perm])
    for b in (0, 4, 8):
        p1, s1 = run(lp[b: b + 1, : tl[b]], tg[b: b + 1, : ul[b]], blank=blank)
        assert torch.equal(p1[0], p[b, : tl[b]]) and torch.equal(s1[0], s[b, : tl[b]])


@pytest.mark.parametrize("dt", [np.float32, np.float16, np.float64])
def test_every_states_per_thread_width(dt):
    """L from 1 to the cap's neighbourhood walks K = 2 ... 32 states per thread; each equals the oracle."""
    for seed, L in enumerate((1, 2, 255, 256, 300, 511, 512, 1100, 2100, 4200)):
        rng = np.random.default_rng(100 + seed)
        tg = rng.integers(1, 20, size=(1, L))
        if seed % 3 == 2:  # off the classes _emission masks to -inf
            tg[tg % 3 == 2] = 1
        T = L + O.repeats(tg[0]) + int(rng.integers(0, 40))
        lp = O._emission(rng, T, 20, seed % 3, dt)
        p, s = run(lp[None], tg, blank=0)
        op, os_ = O.align(lp, tg[0], 0)
        assert torch.equal(p[0], torch.from_numpy(op)) and torch.equal(s[0], torch.from_numpy(os_)), (L, dt)


def test_cap():
    L = _lib.FORCED_ALIGN_MAX_L
    rng = np.random.default_rng(7)
    tg = rng.integers(1, 32, size=(1, L))
    T = L + O.repeats(tg[0]) + 50
    lp = O._emission(rng, T, 32, 0, np.float32)[None]
    p, s = run(lp, tg)
    op, os_ = O.align(lp[0], tg[0], 0)
    assert torch.equal(p[0], torch.from_numpy(op)) and torch.equal(s[0], torch.from_numpy(os_))
    tg1 = rng.integers(1, 32, size=(1, L + 1))
    with pytest.raises(ValueError, match="above the supported 8191"):
        run(np.zeros((1, 2 * L + 10, 32), dtype=np.float32), tg1)


def test_offsets_beyond_2_31_elements():
    """float16, B = 2, T = 2^19, C = 4096: sequence 1 starts at element 2^31 (8.6 GB on the device)."""
    B, T, C = 2, 1 << 19, 4096
    assert T * C >= 2**31
    x = torch.full((B, T, C), -3.0, dtype=torch.float16, device=DEV)
    rng = np.random.default_rng(3)
    T1 = 300
    lp1 = O._emission(rng, T1, C, 0, np.float16)
    x[1, :T1] = torch.from_numpy(lp1).to(DEV)
    x[0, :, 0] = -0.5
    tg = np.array([[5, 9, 9, 4000], [7, 3000, 12, 12]], dtype=np.int64)
    tl = np.array([T, T1])
    ul = np.array([4, 4])
    p, s = F.forced_align(x, torch.from_numpy(tg).to(DEV), torch.from_numpy(tl).to(DEV), torch.from_numpy(ul).to(DEV))
    op, os_ = O.align(lp1, tg[1], 0)
    assert torch.equal(p[1, :T1].cpu(), torch.from_numpy(op)) and torch.equal(s[1, :T1].cpu(), torch.from_numpy(os_))
    assert (p[1, T1:] == 0).all() and (s[1, T1:] == 0).all()
    spans = F.merge_tokens(p[0], s[0])
    assert [t.token for t in spans] == [5, 9, 9, 4000]
    del x


def test_reruns_bit_identical():
    lp, tg, tl, ul, blank = O.batch_inputs((52, 16, 400, 120, 64, 0, 1, 0, 1, 0))
    first = run(lp, tg, tl, ul, blank)
    for _ in range(3):
        again = run(lp, tg, tl, ul, blank)
        assert torch.equal(first[0], again[0]) and torch.equal(first[1], again[1])


def test_reference_error_strings(ref):
    g = torch.Generator().manual_seed(0)
    lp = torch.rand(1, 5, 6, generator=g).to(DEV)
    il, tl = torch.tensor([5], device=DEV), torch.tensor([4], device=DEV)

    def call(lp=lp, tg=None, il=il, tl=tl, blank=5, dtype=torch.int32):
        tg = torch.tensor([[0, 1, 2, 3]], dtype=dtype, device=DEV) if tg is None else tg.to(DEV)
        return lambda: F.forced_align(lp, tg, il, tl, blank)

    errors = {}
    for dt, name in ((torch.int32, "i32"), (torch.int64, "i64")):
        errors.update({
            f"too_long_{name}": call(tg=torch.tensor([[0, 1, 2, 3, 4, 4]], dtype=dt), tl=torch.tensor([6], device=DEV),
                                     dtype=dt),
            f"blank_in_{name}": call(tg=torch.tensor([[5, 3, 3]], dtype=dt), tl=torch.tensor([3], device=DEV)),
            f"lp_dtype_{name}": call(lp=lp.int(), dtype=dt),
            f"tg_dtype_{name}": call(tg=torch.tensor([[0., 1., 2., 3.]])),
            f"input_lengths_dim_{name}": call(il=torch.ones(3, 5, dtype=torch.int64, device=DEV), dtype=dt),
            f"target_lengths_dim_{name}": call(tl=torch.ones(3, 5, dtype=torch.int64, device=DEV), dtype=dt),
            f"input_length_{name}": call(il=torch.tensor([10000], device=DEV), dtype=dt),
            f"target_length_{name}": call(tl=torch.tensor([10000], device=DEV), dtype=dt),
            f"range_{name}": call(lp=torch.rand(1, 10, 5, generator=g).to(DEV),
                                  tg=torch.tensor([[7, 8, 9, 10]], dtype=dt)),
            f"blank_range_{name}": call(tg=torch.tensor([[1, 3, 3]], dtype=dt), tl=torch.tensor([3], device=DEV),
                                        blank=10000),
        })
    errors.update({
        "empty_targets": call(tg=torch.zeros(1, 0, dtype=torch.int32), tl=torch.tensor([0], device=DEV)),
        "negative_blank": call(tg=torch.tensor([[1, 3, 3]]), tl=torch.tensor([3], device=DEV), blank=-1),
        "lp_contiguous": call(lp=lp.transpose(1, 2).contiguous().transpose(1, 2)),
        "tg_contiguous": call(tg=torch.tensor([[1, 0, 2, 0, 3, 0, 4, 0]], dtype=torch.int32, device=DEV)[:, ::2]),
        "lp_dim": call(lp=lp[0]),
        "tg_dim": call(tg=torch.tensor([1, 2, 3, 4], dtype=torch.int32)),
    })
    assert set(errors) == {k[4:] for k in ref if k.startswith("err_")}
    for k, fn in errors.items():
        want = str(ref[f"err_{k}"])
        with pytest.raises(Exception) as e:  # noqa: PT011
            fn()
        got = f"{type(e.value).__name__}: {e.value}"
        if k.startswith("blank_in"):
            want, got = want.split("Found")[0], got.split("Found")[0]
        assert got == want, k


def test_extra_value_errors():
    lp = torch.zeros(2, 6, 5, device=DEV)
    tg = torch.tensor([[1, 2], [3, 4]], device=DEV)
    full = torch.tensor([6, 6], device=DEV)
    with pytest.raises(ValueError, match="negative"):
        F.forced_align(lp, torch.tensor([[1, -2], [3, 4]], device=DEV))
    with pytest.raises(ValueError, match="at least 1"):
        F.forced_align(lp, tg, torch.tensor([6, 0], device=DEV))
    with pytest.raises(ValueError, match="non-negative"):
        F.forced_align(lp, tg, full, torch.tensor([2, -1], device=DEV))
    # a target past its sequence's length is padding: any value is accepted, and a blank there too
    p, _ = F.forced_align(lp, torch.tensor([[1, 2], [3, 99]], device=DEV), full, torch.tensor([2, 1], device=DEV))
    assert set(p[1].tolist()) <= {0, 3}
    p, _ = F.forced_align(lp, torch.tensor([[1, 2], [3, 0]], device=DEV), full, torch.tensor([2, 1], device=DEV))
    assert set(p[1].tolist()) <= {0, 3}


def test_cpu_tensors_rejected():
    with pytest.raises(RuntimeError, match="no CPU or ATen fallback"):
        F.forced_align(torch.zeros(1, 4, 3), torch.tensor([[1]]))
    with pytest.raises(RuntimeError, match="targets must be a CUDA tensor"):
        F.forced_align(torch.zeros(1, 4, 3, device=DEV), torch.tensor([[1]]))
    with pytest.raises(RuntimeError, match="input_lengths must be a CUDA tensor"):
        F.forced_align(torch.zeros(1, 4, 3, device=DEV), torch.tensor([[1]], device=DEV), torch.tensor([4]))


def test_merge_tokens_on_device_paths(ref):
    for i in _keys(ref, "rc_"):
        if f"mt_{i}_token" not in ref:
            continue
        lp, tg, blank = O.case_inputs(ref[f"rc_{i}"])
        p, s = F.forced_align(torch.from_numpy(lp).to(DEV), torch.from_numpy(tg).to(DEV), blank=blank)
        spans = F.merge_tokens(p[0], s[0], blank=blank)
        assert [(x.token, x.start, x.end, x.score) for x in spans] == list(zip(
            ref[f"mt_{i}_token"].tolist(), ref[f"mt_{i}_start"].tolist(), ref[f"mt_{i}_end"].tolist(),
            ref[f"mt_{i}_score"].tolist())), i


def _bench_inputs():
    """The inputs tools/forced_align_bench.py times, every workload whole, from its own ``inputs``."""
    spec = importlib.util.spec_from_file_location("forced_align_bench", os.path.join(ROOT, "tools",
                                                                                   "forced_align_bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    return [bench.inputs(*w) for w in bench.WORKLOADS.values()]


def test_path_likelihood_matches_torchaudio_cuda():
    try:
        import torchaudio.functional as TF
        TF.forced_align(torch.zeros(1, 2, 3, device=DEV), torch.tensor([[1]], dtype=torch.int32, device=DEV))
    except Exception as e:  # noqa: BLE001
        pytest.skip(f"torchaudio CUDA forced_align unavailable: {e}")
    differ = total = 0
    for lp, tg, tl, ul in _bench_inputs():
        p, s = F.forced_align(lp.to(DEV), tg.to(DEV), tl.to(DEV), ul.to(DEV))
        for b in range(lp.shape[0]):
            T, L = int(tl[b]), int(ul[b])
            rp, rs = TF.forced_align(lp[b: b + 1, :T].to(DEV), tg[b: b + 1, :L].to(DEV), blank=0)
            ours = s[b, :T].double().sum().item()
            theirs = rs[0].double().sum().item()
            assert abs(ours - theirs) <= 1e-4 * abs(ours) + 1e-3, (b, ours, theirs)
            differ += int(not torch.equal(rp[0], p[b, :T]))
            total += 1
    print(f"torchaudio CUDA: {differ} of {total} paths differ from the reference CPU's; likelihoods agree")


def test_strided_and_expanded_lengths():
    """Lengths of any 1-D strides, as the reference takes them: strided columns and expanded scalars give the result
    of the same values passed contiguous."""
    lp, tg, tl, ul, blank = O.batch_inputs((53, 6, 90, 30, 29, 0, 0, 0, 0, 0))
    x, t = torch.from_numpy(lp).to(DEV), torch.from_numpy(tg).to(DEV)
    tl_d, ul_d = torch.from_numpy(tl).to(DEV), torch.from_numpy(ul).to(DEV)
    want = F.forced_align(x, t, tl_d, ul_d, blank)
    pairs = torch.stack([tl_d, ul_d], 1)  # (B, 2): columns with stride 2
    for a, b in ((pairs[:, 0], pairs[:, 1]), (pairs[:, 0], ul_d.int())):
        assert not a.is_contiguous()
        got = F.forced_align(x, t, a, b, blank)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    B, T, L = tg.shape[0], lp.shape[1], tg.shape[1]  # every row at full length: L + R <= 2 L - 1 < T
    want = F.forced_align(x, t, torch.full((B,), T, device=DEV), torch.full((B,), L, device=DEV), blank)
    for dt_t, dt_l in ((torch.int64, torch.int64), (torch.int32, torch.int32), (torch.int64, torch.int32)):
        a = torch.tensor([T], dtype=dt_t, device=DEV).expand(B)  # stride 0: one element behind B entries
        b = torch.tensor([L], dtype=dt_l, device=DEV).expand(B)
        got = F.forced_align(x, t, a, b, blank)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


def test_blank_range_error_before_negative_target():
    """The reference checks the blank's range before it reads any target; the extra negative-target error comes after
    it, also for a blank outside int32."""
    lp = torch.zeros(1, 6, 5, device=DEV)
    tg = torch.tensor([[1, -1]], device=DEV)
    for blank in (5, 2**40, -(2**40)):
        with pytest.raises(RuntimeError, match=re.escape("blank must be within [0, num classes)")):
            F.forced_align(lp, tg, blank=blank)
    with pytest.raises(ValueError, match="negative"):
        F.forced_align(lp, tg, blank=0)
