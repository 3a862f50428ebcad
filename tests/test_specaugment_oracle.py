"""The SpecAugment oracle (tests/specaugment_oracle.py) against the reference's CPU results in
tests/golden/specaugment_ref_cases.npz: values bit for bit, output strides, whether the input itself came back, how much
of the generator each call consumed, and the error strings.  Also the output layouts audio_b200 derives on meta tensors
against the same strides."""
import ast
import os

import numpy as np
import pytest
import torch

import specaugment_oracle as O
from audio_b200 import _masking

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "specaugment_ref_cases.npz")


@pytest.fixture(scope="module")
def ref():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def _cases(ref):
    n = sum(1 for k in ref if k.startswith("case_"))
    return [(i, ast.literal_eval(str(ref[f"case_{i}"]))) for i in range(n)]


def test_fixture_covers_the_paths(ref):
    ops = [c["op"] for _, c in _cases(ref)]
    assert {op[0] for op in ops} == {"iid", "axis", "freq", "time", "spec"}
    assert any(op[0] == "iid" and isinstance(op[2], tuple) for op in ops)  # tensor fill
    assert {op[4] for op in ops if op[0] == "iid"} >= {0.0, 0.2, 1.0}
    assert {op[1] for op in ops if op[0] == "iid"} >= {0, 1, 5, 40}
    assert {int(ref[f"same_{i}"]) for i, _ in _cases(ref)} == {0, 1}


def test_oracle_reproduces_the_reference(ref):
    for i, case in _cases(ref):
        x = O.make_input(case["x"])
        torch.manual_seed(100 + i)
        y = O.run_case(O.ORACLE, case["op"], x)
        nxt = torch.rand(4).numpy()
        want = ref[f"out_{i}"]
        assert y.shape == want.shape, i
        np.testing.assert_array_equal(y.numpy().view(np.uint32), want.view(np.uint32), err_msg=str(case))
        assert y.stride() == tuple(ref[f"stride_{i}"]), (i, case, y.stride())
        assert int(y is x) == int(ref[f"same_{i}"]), case
        np.testing.assert_array_equal(nxt, ref[f"next_{i}"], err_msg=str(case))


def test_oracle_errors(ref):
    k = 0
    while f"err_{k}" in ref:
        case = ast.literal_eval(str(ref[f"errcase_{k}"]))
        with pytest.raises(Exception) as e:
            O.run_case(O.ORACLE, case["op"], O.make_input(case["x"]))
        assert f"{e.type.__name__}: {e.value}" == str(ref[f"err_{k}"])
        k += 1
    assert k >= 8


def _steps(op, x):
    """The (iid, axis) steps audio_b200 launches for a fixture call, and its fill (a float or a 0-d tensor)."""
    name, *a = op
    dim = x.dim()

    def fill(v):
        return torch.tensor(v[1]) if isinstance(v, tuple) else v

    def limit(param, p, axis):
        return _masking._get_mask_param(param, p, x.shape[axis])

    if name in ("iid", "axis"):
        return ([(name == "iid", a[2])] if limit(a[0], a[3], a[2]) >= 1 else []), fill(a[1])
    if name in ("freq", "time"):
        iid, p, v = (a[1], 1.0, a[2]) if name == "freq" else (a[1], a[2], a[3])
        axis = (1 if name == "freq" else 2) + dim - 3
        v = fill(v)
        if not iid and isinstance(v, torch.Tensor):
            v = float(v)
        return ([(iid, axis)] if limit(a[0], p, axis) >= 1 else []), v
    n_t, t_param, n_f, f_param, iid, p, zero = a
    iid = dim > 2 and iid
    steps = [(iid, dim - 1)] * (n_t if limit(t_param, p, dim - 1) >= 1 else 0)
    steps += [(iid, dim - 2)] * (n_f if limit(f_param, p, dim - 2) >= 1 else 0)
    return steps, 0.0 if zero else torch.tensor(0.0)


def test_meta_layout_matches_reference_strides(ref):
    for i, case in _cases(ref):
        x = O.make_input(case["x"])
        steps, fill = _steps(case["op"], x)
        if not steps:
            assert int(ref[f"same_{i}"]) == 1, case
            continue
        shape, stride = _masking._layout(x, steps, fill)
        assert shape == ref[f"out_{i}"].shape, case
        assert stride == tuple(ref[f"stride_{i}"]), (case, stride)
