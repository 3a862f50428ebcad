"""SpecAugment masking on the GPU against tests/specaugment_oracle.py on the same device under the same seed: values bit
for bit, shapes and strides, the input untouched, the same consumption of the CUDA and CPU generators, and gradients."""
import ast
import json
import os

import numpy as np
import pytest
import torch

import specaugment_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "specaugment_ref_cases.npz")


def _ours():
    import audio_b200.functional as F
    import audio_b200.transforms as T

    return O.SimpleNamespace(mask_along_axis_iid=F.mask_along_axis_iid, mask_along_axis=F.mask_along_axis,
                             FrequencyMasking=T.FrequencyMasking, TimeMasking=T.TimeMasking, SpecAugment=T.SpecAugment)


def _bits(t):
    return t.view(torch.int32)


def _run(ns, op, x):
    try:
        return O.run_case(ns, op, x), None
    except Exception as ex:  # noqa: BLE001
        return None, f"{type(ex).__name__}: {ex}"


def check(op, x, seed=0):
    """Run op with audio_b200 and with the oracle from the same seed; compare everything (or the error both raise);
    return both outputs."""
    x0 = x.clone()
    torch.manual_seed(seed)
    y, y_err = _run(_ours(), op, x)
    got_state = torch.cuda.get_rng_state(), torch.get_rng_state()
    torch.manual_seed(seed)
    e, e_err = _run(O.ORACLE, op, x)
    assert torch.equal(got_state[0], torch.cuda.get_rng_state()), f"{op}: CUDA generator consumption differs"
    assert torch.equal(got_state[1], torch.get_rng_state()), f"{op}: CPU generator consumption differs"
    assert y_err == e_err, op
    if e_err is not None:
        return None, None
    assert (y is x) == (e is x), op
    assert y.shape == e.shape and y.stride() == e.stride(), (op, y.stride(), e.stride())
    assert torch.equal(_bits(y), _bits(e)), f"{op}: {(_bits(y) != _bits(e)).sum().item()} elements differ"
    assert torch.equal(_bits(x), _bits(x0)), f"{op}: the input was modified"
    return y, e


def _golden_cases():
    with np.load(GOLDEN) as z:
        n = sum(1 for k in z.files if k.startswith("case_"))
        return [ast.literal_eval(str(z[f"case_{i}"])) for i in range(n)]


@pytest.mark.parametrize("case", _golden_cases(), ids=lambda c: f"{c['op']}-{c['x'].get('view', '')}")
def test_fixture_cases(case):
    check(case["op"], O.make_input(case["x"], DEV), seed=11)


RECIPE = {"shape": (64, 1600, 80), "seed": 21, "view": "t"}  # (B, T, n_mels).transpose(1, 2)
OPS = [
    ("iid", 27, 0.0, 1, 1.0), ("iid", 100, 0.0, 2, 0.2), ("iid", 27, ("t", -0.5), 1, 1.0),
    ("iid", 100, ("t", 0.25), 2, 1.0), ("iid", 2000, 0.0, 2, 1.0), ("iid", 200, 1.0, 1, 1.0),
    ("axis", 27, 0.0, 1, 1.0), ("axis", 100, 0.5, 2, 0.2), ("axis", 3000, 0.0, 2, 1.0),
    ("freq", 27, False, 0.0), ("time", 100, False, 0.2, 0.0), ("freq", 27, True, 0.0), ("time", 100, True, 0.2, 0.0),
    ("spec", 2, 100, 2, 27, True, 1.0, False), ("spec", 2, 100, 2, 27, True, 0.2, False),
    ("spec", 2, 100, 2, 27, False, 1.0, False), ("spec", 2, 100, 2, 27, True, 1.0, True),
    ("spec", 20, 60, 20, 10, True, 1.0, False),  # 40 masks in one launch
    ("spec", 20, 60, 20, 10, False, 1.0, False),
]


@pytest.mark.parametrize("op", OPS, ids=str)
@pytest.mark.parametrize("view", ["t", None, "step"])
def test_recipe_scale(op, view):
    check(op, O.make_input(dict(RECIPE, view=view), DEV), seed=3)


@pytest.mark.parametrize("op", [("iid", 5, 0.0, 3, 1.0), ("iid", 4, ("t", 1.0), 2, 1.0), ("axis", 4, 2.0, 3, 1.0),
                                ("spec", 3, 6, 3, 4, True, 1.0, False), ("spec", 3, 6, 3, 4, False, 1.0, False)],
                         ids=str)
@pytest.mark.parametrize("view", [None, "perm", "t", "step"])
def test_4d(op, view):
    check(op, O.make_input({"shape": (3, 4, 24, 30), "seed": 5, "view": view}, DEV), seed=4)


def test_nan_inputs_and_nan_mean():
    spec = {"shape": (4, 40, 64), "seed": 8, "nan": (0, 77, 1000, 5000)}
    for op in (("iid", 10, 0.0, 2, 1.0), ("axis", 10, 1.0, 1, 1.0), ("spec", 2, 10, 2, 8, True, 1.0, False),
               ("spec", 2, 10, 2, 8, False, 1.0, False)):
        check(op, O.make_input(spec, DEV), seed=5)
    y, _ = check(("spec", 2, 10, 2, 8, True, 1.0, False), O.make_input(spec, DEV), seed=5)
    assert torch.isnan(y).sum() > 4  # the mean is NaN, and so is every masked element


@pytest.mark.parametrize("shape", [(0, 8, 12), (3, 0, 12), (3, 8, 0), (2, 0, 8, 12)])
def test_zero_size(shape):
    x = torch.zeros(shape, device=DEV)
    for op in (("iid", 5, 0.0, x.dim() - 1, 1.0), ("iid", 5, ("t", 1.0), x.dim() - 2, 1.0),
               ("axis", 5, 0.0, x.dim() - 1, 1.0), ("spec", 2, 5, 2, 4, True, 1.0, True),
               ("spec", 2, 5, 2, 4, False, 1.0, True)):
        y, _ = check(op, x, seed=6)
        assert y is None or y.numel() == 0  # the reference cannot pack (-1, 0, T) or (-1, F, 0): both raise


def test_tensor_fill_checks():
    x = torch.randn(2, 8, 12, device=DEV)
    F = _ours()
    with pytest.raises(RuntimeError, match="one-element float32"):
        F.mask_along_axis_iid(x, 5, torch.zeros(2, device=DEV), 2)
    with pytest.raises(RuntimeError, match="one-element float32"):
        F.mask_along_axis_iid(x, 5, torch.zeros((), dtype=torch.float64, device=DEV), 2)
    with pytest.raises(RuntimeError, match="one-element float32"):
        F.mask_along_axis_iid(x, 5, torch.zeros(()), 2)
    with pytest.raises(TypeError, match="float32"):
        F.mask_along_axis_iid(x.double(), 5, 0.0, 2)


def test_above_2_31_elements():
    rows = (1 << 31) // (256 * 256) + 1
    x = torch.randn(rows, 256, 256, device=DEV)
    assert x.numel() > 1 << 31
    for op in (("iid", 100, 0.0, 2, 1.0), ("freq", 100, False, 0.0)):
        xt = x.transpose(1, 2) if op[0] == "freq" else x
        y, e = check(op, xt, seed=7)
        del y, e
        torch.cuda.empty_cache()


def _grad_pair(op, x, g=None, fill_grad=False, seed=9):
    """Gradients of (input, tensor fill) through audio_b200 and the oracle, same draws."""
    grads = []
    for ns in (_ours(), O.ORACLE):
        xi = x.detach().clone().requires_grad_(True)
        fill = torch.tensor(0.75, device=DEV, requires_grad=True) if fill_grad else None
        op_ = tuple(fill if v == "FILL" else v for v in op)
        torch.manual_seed(seed)
        if fill is not None:
            y = (ns.mask_along_axis_iid if op[0] == "iid" else ns.mask_along_axis)(xi, op_[1], fill, op_[3], p=op_[4])
        else:
            y = O.run_case(ns, op_, xi)
        (y.sum() if g is None else (y * g).sum()).backward()
        grads.append((xi.grad, None if fill is None else fill.grad))
    return grads


@pytest.mark.parametrize("op", [("iid", 27, 0.0, 1, 1.0), ("iid", 100, 1.0, 2, 0.2), ("axis", 27, 0.0, 1, 1.0),
                                ("time", 100, False, 0.2, 0.0), ("spec", 2, 100, 2, 27, True, 1.0, True)], ids=str)
def test_input_gradient_exact(op):
    x = O.make_input(dict(RECIPE, shape=(8, 400, 80)), DEV)
    g = torch.randn(8, 80, 400, device=DEV)
    (ga, _), (gb, _) = _grad_pair(op, x, g)
    assert torch.equal(ga, gb)
    (ga, _), (gb, _) = _grad_pair(op, x)  # .sum(): a stride-0 upstream gradient
    assert torch.equal(ga, gb)


@pytest.mark.parametrize("op", [("iid", 27, "FILL", 1, 1.0), ("iid", 100, "FILL", 2, 0.2), ("axis", 27, "FILL", 1, 1.0)],
                         ids=str)
def test_fill_gradient(op):
    x = O.make_input(dict(RECIPE, shape=(8, 400, 80)), DEV)
    g = torch.randn(8, 80, 400, device=DEV)
    (xa, fa), (xb, fb) = _grad_pair(op, x, g, fill_grad=True)
    assert torch.equal(xa, xb)
    assert abs(fa.item() - fb.item()) <= 1e-6 * abs(fb.item()), (fa.item(), fb.item())


@pytest.mark.parametrize("iid", [True, False])
def test_specaugment_gradient_through_mean(iid):
    x = O.make_input(dict(RECIPE, shape=(8, 400, 80)), DEV)
    op = ("spec", 2, 100, 2, 27, iid, 1.0, False)
    (ga, _), (gb, _) = _grad_pair(op, x)
    vals = torch.unique(gb)
    assert vals.numel() <= 2  # 1/N + 1 unmasked, (masked sum)/N masked
    torch.testing.assert_close(ga, gb, rtol=1e-6, atol=0)
    g = torch.randn(8, 80, 400, device=DEV)
    (ga, _), (gb, _) = _grad_pair(op, x, g)
    torch.testing.assert_close(ga, gb, rtol=1e-6, atol=1e-6 * gb.abs().max().item())


def test_backward_is_deterministic_and_once_differentiable():
    T = _ours()
    x = O.make_input(dict(RECIPE, shape=(16, 800, 80)), DEV).requires_grad_(True)
    torch.manual_seed(1)
    y = T.SpecAugment(4, 100, 4, 27)(x)
    g = torch.randn_like(y)
    a = torch.autograd.grad(y, x, g, retain_graph=True)[0]
    b = torch.autograd.grad(y, x, g, retain_graph=True)[0]
    assert torch.equal(_bits(a), _bits(b))
    gx = torch.autograd.grad(y.sum(), x, create_graph=True)[0]
    with pytest.raises(RuntimeError):
        gx.sum().backward()


def test_no_grad_and_detached_paths_match():
    T = _ours()
    x = O.make_input(dict(RECIPE, shape=(4, 200, 80)), DEV)
    torch.manual_seed(2)
    with torch.no_grad():
        a = T.SpecAugment(2, 50, 2, 27)(x.requires_grad_(True))
    torch.manual_seed(2)
    b = T.SpecAugment(2, 50, 2, 27)(x.detach())
    assert not a.requires_grad and torch.equal(_bits(a), _bits(b))


def test_rnnt_features_then_recipe_train_transform(tmp_path):
    from audio_b200.pipelines import RNNTFeatureExtractor

    path = tmp_path / "global_stats.json"
    rng = np.random.default_rng(0)
    path.write_text(json.dumps({"mean": rng.uniform(10, 16, 80).tolist(), "invstddev": rng.uniform(0.2, 0.4, 80).tolist()}))
    ext = RNNTFeatureExtractor(str(path)).to(DEV)
    g = torch.Generator().manual_seed(3)
    lens = [16000 * 3, 16000 * 2 + 123, 16000 * 4, 9000]
    waves = torch.randn(len(lens), max(lens), generator=g) * 0.1
    feats, _ = ext.forward_batch(waves.to(DEV), lens)

    def chain(ns):
        y = feats.transpose(1, 2)
        y = ns.FrequencyMasking(27)(y)
        y = ns.FrequencyMasking(27)(y)
        y = ns.TimeMasking(100, p=0.2)(y)
        y = ns.TimeMasking(100, p=0.2)(y)
        return y.transpose(1, 2)

    torch.manual_seed(42)
    got = chain(_ours())
    state = torch.get_rng_state()
    torch.manual_seed(42)
    want = chain(O.ORACLE)
    assert torch.equal(state, torch.get_rng_state())
    assert got.shape == want.shape and got.stride() == want.stride()
    assert torch.equal(_bits(got), _bits(want))
    assert (got == 0).any()
