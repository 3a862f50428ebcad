"""rnnt_loss / RNNTLoss on the GPU against the float64 oracle (tests/rnnt_loss_oracle.py).

Accuracy bar, per case: the GPU's error against the oracle is at most twice the reference CPU's own error on the same
inputs (stored in tests/golden/rnnt_loss_ref_cases.npz, or measured here with the installed torchaudio's CPU path)
plus a floor -- costs 1e-6 relative and gradients 1e-5 absolute in float32, 1e-3 for both in float16, where the
oracle runs on the float16-rounded logits.  The reference's own error grows with T + U, so a fixed bar would be too
loose for small cases or fail honest long ones.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import audio_b200.functional as F
import audio_b200.transforms as T
import rnnt_loss_oracle as O
from conftest import ROOT, _load

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
FLOOR = {np.float32: (1e-6, 1e-5), np.float16: (1e-3, 1e-3)}


def _torchaudio():
    try:
        import torchaudio.functional as TF
        return TF
    except Exception:  # noqa: BLE001
        return None


@pytest.fixture(scope="module")
def ref():
    return _load("rnnt_loss_ref_cases.npz")


def cuda_inputs(lg, tg, tl, ul, grad=True):
    x = torch.from_numpy(lg).to(DEV).requires_grad_(grad)
    return x, torch.from_numpy(tg).to(DEV), torch.from_numpy(tl).to(DEV), torch.from_numpy(ul).to(DEV)


def gpu_run(lg, tg, tl, ul, blank=-1, clamp=-1.0, fused=True, dy=None):
    x, t, a, b = cuda_inputs(lg, tg, tl, ul)
    c = F.rnnt_loss(x, t, a, b, blank=blank, clamp=clamp, reduction="none", fused_log_softmax=fused)
    c.backward(torch.ones_like(c) if dy is None else dy)
    return c.detach().double().cpu().numpy(), x.grad.double().cpu().numpy()


def ref_errors(lg, tg, tl, ul, blank, clamp, fused, oc, og):
    """The reference CPU's own (cost relative, gradient max-abs) error against the oracle, or None without torchaudio."""
    TF = _torchaudio()
    if TF is None:
        return None
    x = torch.from_numpy(lg).requires_grad_()
    c = TF.rnnt_loss(x, torch.from_numpy(tg), torch.from_numpy(tl), torch.from_numpy(ul), blank=blank, clamp=clamp,
                     reduction="none", fused_log_softmax=fused)
    c.sum().backward()
    return (np.max(np.abs(c.detach().double().numpy() - oc) / np.abs(oc)),
            np.max(np.abs(x.grad.double().numpy() - og)))


def check(lg, tg, tl, ul, blank=-1, clamp=-1.0, fused=True, errs=None, what=""):
    c, g = gpu_run(lg, tg, tl, ul, blank, clamp, fused)
    oc, og = O.rnnt_loss(lg, tg, tl, ul, blank, clamp, fused)
    if errs is None:
        errs = ref_errors(lg, tg, tl, ul, blank, clamp, fused, oc, og)
    if errs is None:  # no reference here: the reference's growth with the DP length, measured at (400, 60, 16)
        errs = (5e-7, 3e-6 * (lg.shape[1] + lg.shape[2]))
    c_floor, g_floor = FLOOR[lg.dtype.type]
    cerr = np.max(np.abs(c - oc) / np.abs(oc))
    gerr = np.max(np.abs(g - og))
    assert cerr <= 2 * errs[0] + c_floor, f"{what}: cost error {cerr:.3e} (reference {errs[0]:.3e})"
    assert gerr <= 2 * errs[1] + g_floor, f"{what}: gradient error {gerr:.3e} (reference {errs[1]:.3e})"
    return c, g


@pytest.mark.parametrize("name", ["B1_T2_U3_D5", "B2_T4_U3_D3", "B1_T10_U3_D4"])
def test_hand_worked_fixtures(ref, name):
    p = f"fx_{name}_"
    c, g = gpu_run(ref[p + "logits"], ref[p + "targets"], ref[p + "tl"], ref[p + "ul"], int(ref[p + "blank"]), -1.0,
                   bool(ref[p + "fused"]))
    np.testing.assert_allclose(c, ref[p + "cost"], rtol=1e-6)
    np.testing.assert_allclose(g, ref[p + "grad"], atol=1e-6)


@pytest.mark.parametrize("i", range(13))
def test_reference_recipes(ref, i):
    rc = ref[f"rc_{i}"]
    lg, tg, tl, ul = O.case_inputs(rc)
    check(lg, tg, tl, ul, int(rc[5]), float(ref[f"clamp_{i}"]), bool(ref[f"fused_{i}"]),
          (float(ref[f"cerr_{i}"]), float(ref[f"gerr_{i}"])), what=f"recipe {i}")
    if f"grad_{i}" in ref:  # and the reference CPU itself, where stored
        c, g = gpu_run(lg, tg, tl, ul, int(rc[5]), float(ref[f"clamp_{i}"]), bool(ref[f"fused_{i}"]))
        tol = 2e-3 if rc[6] else 1e-5
        np.testing.assert_allclose(c, ref[f"cost_{i}"], rtol=tol)
        np.testing.assert_allclose(g, ref[f"grad_{i}"], atol=tol)


@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("blank", [-1, 0, 14])
@pytest.mark.parametrize("clamp", [-1.0, 0.0, 0.02])
def test_values(half, fused, blank, clamp):
    lg, tg, tl, ul = O.case_inputs((100 + blank, 4, 12, 7, 29, blank, int(half), 1.5))
    _, g = check(lg, tg, tl, ul, blank, clamp, fused, what="values")
    if clamp > 0:
        assert np.abs(g).max() <= clamp * (1 + 1e-3)


@pytest.mark.parametrize("reduction", ["none", "mean", "sum"])
def test_reductions(reduction):
    lg, tg, tl, ul = O.case_inputs((200, 5, 10, 6, 33, -1, 0, 1.0))
    x, t, a, b = cuda_inputs(lg, tg, tl, ul)
    loss = F.rnnt_loss(x, t, a, b, reduction=reduction)
    oc, og = O.rnnt_loss(lg, tg, tl, ul)
    exp = {"none": oc, "mean": oc.mean(), "sum": oc.sum()}[reduction]
    np.testing.assert_allclose(loss.detach().double().cpu().numpy(), exp, rtol=1e-5)
    loss.sum().backward()
    scale = 1.0 / len(oc) if reduction == "mean" else 1.0
    np.testing.assert_allclose(x.grad.double().cpu().numpy(), og * scale, atol=1e-5)
    assert loss.dtype == torch.float32


@pytest.mark.parametrize("shape", [
    (3, 1, 5, 7, False),  # T = 1
    (3, 6, 1, 7, False),  # every target_length 0
    (2, 3, 1025, 3, False),  # more cells per diagonal than threads
    (2, 3, 2049, 3, True),
    (3, 5, 4, 1, False),  # V = 1: the only class is the blank
    (3, 5, 4, 3, True),
    (2, 6, 5, 1024, False),
    (2, 6, 5, 1024, True),
    (2, 5, 4, 4097, False),
    (2, 5, 4, 4097, True),
])
def test_shapes(shape):
    B, max_t, max_u, V, half = shape
    lg, tg, tl, ul = O.case_inputs((300 + V + max_u, B, max_t, max_u, V, -1, int(half), 1.0))
    check(lg, tg, tl, ul, what=str(shape))


def test_ragged_padding_is_never_read_and_gets_zero_gradient():
    lg, tg, tl, ul = O.case_inputs((400, 4, 9, 6, 29, -1, 0, 1.0))
    tl[:] = [9, 3, 1, 6]
    ul[:] = [2, 5, 0, 3]
    oc, og = O.rnnt_loss(lg, tg, tl, ul)
    pad = np.ones(lg.shape, bool)
    for b in range(4):
        pad[b, : tl[b], : ul[b] + 1] = False
    lg = lg.copy()
    lg[pad] = np.nan
    c, g = gpu_run(lg, tg, tl, ul)
    np.testing.assert_allclose(c, oc, rtol=1e-5)
    assert (g[pad] == 0).all()
    np.testing.assert_allclose(g, og, atol=1e-5)


def test_nonfinite_cost_is_nan_with_zero_gradient(ref):
    lg, tg, tl, ul = O.case_inputs((30, 3, 6, 4, 5, -1, 0, 1.0))
    lg[1, :, :, 4] = -np.inf
    c, g = gpu_run(lg, tg, tl, ul)
    np.testing.assert_allclose(c, ref["nonfinite_cost"], rtol=1e-5)  # NaN where the reference CPU's cost is NaN
    assert np.isnan(c[1]) and (g[1] == 0).all() and np.isfinite(g).all()
    np.testing.assert_allclose(g, O.rnnt_loss(lg, tg, tl, ul)[1], atol=1e-5)


@pytest.mark.parametrize("fused", [True, False])
def test_clamp_then_scale_with_nonuniform_upstream(fused):
    lg, tg, tl, ul = O.case_inputs((500, 4, 8, 5, 11, -1, 0, 3.0))
    dy = torch.tensor([0.5, -2.0, 3.0, 0.0], device=DEV)
    c, g = gpu_run(lg, tg, tl, ul, clamp=0.05, fused=fused, dy=dy)
    og = O.rnnt_loss(lg, tg, tl, ul, clamp=0.05, fused=fused)[1]
    assert np.abs(og).max() <= 0.05
    np.testing.assert_allclose(g, og * dy.double().cpu().numpy()[:, None, None, None], atol=1e-5)


def _kernel_names(fn):
    names = set()
    for _ in range(10):  # a profiler session now and then drops kernel records: run the deterministic call again
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
        if any("rnnt_alpha_beta_kernel" in n for n in names):
            break
    return {n for n in names if "Memcpy" not in n and "Memset" not in n}


def test_no_gradient_kernel_without_grad():
    lg, tg, tl, ul = O.case_inputs((600, 3, 8, 5, 29, -1, 0, 1.0))
    x, t, a, b = cuda_inputs(lg, tg, tl, ul)

    def no_grad():
        with torch.no_grad():
            F.rnnt_loss(x, t, a, b)

    def with_grad():
        F.rnnt_loss(x, t, a, b).backward()

    names = _kernel_names(no_grad)
    assert any("rnnt_rows_kernel" in n for n in names), names
    assert not any("rnnt_grad_kernel" in n for n in names), names
    x.requires_grad_(False)
    assert not any("rnnt_grad_kernel" in n for n in _kernel_names(no_grad))
    x.requires_grad_(True)
    assert any("rnnt_grad_kernel" in n for n in _kernel_names(with_grad))


def test_reruns_are_bit_identical():
    lg, tg, tl, ul = O.case_inputs((700, 4, 40, 12, 257, -1, 1, 1.0))
    c1, g1 = gpu_run(lg, tg, tl, ul)
    c2, g2 = gpu_run(lg, tg, tl, ul)
    assert np.array_equal(c1, c2) and np.array_equal(g1, g2)


def test_module_matches_functional():
    m = T.RNNTLoss(blank=0, clamp=0.1, reduction="sum", fused_log_softmax=False)
    assert (m.blank, m.clamp, m.reduction, m.fused_log_softmax) == (0, 0.1, "sum", False)
    d = T.RNNTLoss()
    assert (d.blank, d.clamp, d.reduction, d.fused_log_softmax) == (-1, -1.0, "mean", True)
    lg, tg, tl, ul = O.case_inputs((800, 3, 7, 4, 9, 0, 0, 1.0))
    args = cuda_inputs(lg, tg, tl, ul, grad=False)
    assert torch.equal(m(*args), F.rnnt_loss(*args, blank=0, clamp=0.1, reduction="sum", fused_log_softmax=False))


def test_inplace_edit_before_backward_raises():
    lg, tg, tl, ul = O.case_inputs((900, 2, 5, 3, 7, -1, 0, 1.0))
    x, t, a, b = cuda_inputs(lg, tg, tl, ul, grad=False)
    y = x.clone().requires_grad_()
    z = y * 1.0
    loss = F.rnnt_loss(z, t, a, b)
    z.add_(1.0)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        loss.backward()


def test_error_messages(ref):
    lg, tg, tl, ul = (torch.from_numpy(a).to(DEV) for a in O.case_inputs((31, 2, 4, 3, 5, -1, 0, 1.0)))
    base = dict(logits=lg, targets=tg, logit_lengths=tl, target_lengths=ul)
    cases = {
        "reduction": dict(reduction="avg"),
        "dtype_f64": dict(logits=lg.double()),
        "dtype_bf16": dict(logits=lg.bfloat16()),
        "targets_dtype": dict(targets=tg.long()),
        "logit_lengths_dtype": dict(logit_lengths=tl.long()),
        "target_lengths_dtype": dict(target_lengths=ul.long()),
        "logits_contiguous": dict(logits=lg.transpose(1, 2).contiguous().transpose(1, 2)),
        "targets_contiguous": dict(targets=torch.cat([tg, tg], 1)[:, ::2]),
        "logits_dim": dict(logits=lg[0]),
        "targets_dim": dict(targets=tg[0]),
        "logit_lengths_dim": dict(logit_lengths=tl[None]),
        "target_lengths_dim": dict(target_lengths=ul[None]),
        "batch_logit_lengths": dict(logit_lengths=tl[:1]),
        "batch_target_lengths": dict(target_lengths=ul[:1]),
        "batch_targets": dict(targets=tg[:1]),
        "blank": dict(blank=5),
        "input_length": dict(logit_lengths=tl - 1),
        "output_length": dict(target_lengths=ul - 1),
        "target_length": dict(targets=torch.cat([tg, tg], 1)),
    }
    for key, kw in cases.items():
        kind, msg = str(ref[f"err_{key}"]).split(": ", 1)
        with pytest.raises({"ValueError": ValueError, "RuntimeError": RuntimeError}[kind]) as e:
            F.rnnt_loss(**{**base, **kw})
        assert str(e.value) == msg, key
    with pytest.raises(RuntimeError, match="no CPU or ATen fallback"):
        F.rnnt_loss(lg.cpu(), tg, tl, ul)
    for name in ("targets", "logit_lengths", "target_lengths"):
        with pytest.raises(RuntimeError, match=f"logits and {name} must be on the same device"):
            F.rnnt_loss(**{**base, name: base[name].cpu()})
    with pytest.raises(ValueError, match="logit_lengths entry must be at least 1"):
        F.rnnt_loss(lg, tg, torch.tensor([4, 0], dtype=torch.int32, device=DEV), ul)
    bad_u = ul.clone()
    bad_u[ul.argmin()] = -1
    with pytest.raises(ValueError, match="target_lengths entries must be non-negative"):
        F.rnnt_loss(lg, tg, tl, bad_u)
    bad_t = tg.clone()
    bad_t[0, 0] = 5
    with pytest.raises(ValueError, match=r"outside \[0, 5\)"):
        F.rnnt_loss(lg, bad_t, tl, ul)
    # a target past its sequence's length is padding: any value is accepted
    short = torch.tensor([0, int(ul.max())], dtype=torch.int32, device=DEV)
    pad_t = tg.clone()
    pad_t[0, :] = 99
    F.rnnt_loss(lg, pad_t, tl, short)


def test_offsets_beyond_2_31_elements():
    """float16, B = 3, maxT = 1024, maxU = 1025, V = 1024: the last sequence starts past 2^31 elements; about 2 000
    valid rows keep the oracle cheap (about 13 GB on the device)."""
    B, max_t, max_u, V = 3, 1024, 1025, 1024
    tl = np.array([1024, 1, 3], dtype=np.int32)
    ul = np.array([0, 1024, 2], dtype=np.int32)
    assert 2 * max_t * max_u * V > 2**31
    rng = np.random.default_rng(1000)
    tg = rng.integers(0, V - 1, size=(B, max_u - 1)).astype(np.int32)
    x = torch.full((B, max_t, max_u, V), float("nan"), dtype=torch.float16, device=DEV)
    blocks = []
    for b in range(B):
        blk = rng.standard_normal((tl[b], ul[b] + 1, V)).astype(np.float16)
        x[b, : tl[b], : ul[b] + 1] = torch.from_numpy(blk).to(DEV)
        blocks.append(blk)
    x.requires_grad_()
    c = F.rnnt_loss(x, torch.from_numpy(tg).to(DEV), torch.from_numpy(tl).to(DEV), torch.from_numpy(ul).to(DEV),
                    reduction="sum")
    c.backward()
    g = x.grad
    valid = sum(int(tl[b]) * (int(ul[b]) + 1) for b in range(B))
    assert int((g != 0).any(-1).sum()) <= valid and not torch.isnan(g).any()
    total = 0.0
    for b in range(B):
        oc, og = O.sequence(blocks[b].astype(np.float64), tg[b], V - 1, -1.0, True)
        total += oc
        got = g[b, : tl[b], : ul[b] + 1].double().cpu().numpy()
        one = (blocks[b][None], tg[b: b + 1, : ul[b]], tl[b: b + 1], ul[b: b + 1])
        errs = ref_errors(*one, -1, -1.0, True, np.array([oc]), og[None])
        bar = 2 * (errs[1] if errs is not None else 3e-6 * (tl[b] + ul[b] + 1)) + FLOOR[np.float16][1]
        assert np.max(np.abs(got - og)) <= bar, b
    assert abs(float(c) - total) <= 1e-3 * abs(total)
    del x, g, c
    torch.cuda.empty_cache()


@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("fused", [True, False])
def test_against_torchaudio_cuda(half, fused):
    TF = _torchaudio()
    if TF is None:
        pytest.skip("torchaudio is not importable")
    lg, tg, tl, ul = O.case_inputs((1100, 4, 30, 11, 129, -1, int(half), 1.0))
    args = cuda_inputs(lg, tg, tl, ul)
    x2 = args[0].detach().clone().requires_grad_()
    ours = F.rnnt_loss(*args, reduction="sum", fused_log_softmax=fused)
    ours.backward()
    theirs = TF.rnnt_loss(x2, *args[1:], reduction="sum", fused_log_softmax=fused)
    theirs.backward()
    ours, theirs = ours.detach(), theirs.detach()
    # both differ from the float64 oracle by float32 rounding: allow ours its bar and theirs its own error
    oc, og = O.rnnt_loss(lg, tg, tl, ul, fused=fused)
    c_floor, g_floor = FLOOR[lg.dtype.type]
    c_theirs = abs(float(theirs) - oc.sum()) / abs(oc.sum())
    g_theirs = float((x2.grad.double().cpu() - torch.from_numpy(og)).abs().max())
    assert abs(float(ours) - float(theirs)) <= (3 * c_theirs + c_floor) * abs(float(theirs))
    torch.testing.assert_close(args[0].grad.double(), x2.grad.double(), atol=3 * g_theirs + g_floor, rtol=0)


def test_reference_switch_routes_rnntloss_to_torchaudio():
    if _torchaudio() is None:
        pytest.skip("torchaudio is not importable")
    code = (
        "import warnings, torch\n"
        "warnings.simplefilter('ignore')\n"
        "import audio_b200.transforms as T, torchaudio\n"
        "m = T.RNNTLoss(blank=0)\n"
        "ref = m.__dict__['_reference_module']\n"
        "assert isinstance(ref, torchaudio.transforms.RNNTLoss), type(ref)\n"
        "x = torch.randn(2, 4, 3, 5, device='cuda')\n"
        "t = torch.tensor([[1, 2], [3, 4]], dtype=torch.int32, device='cuda')\n"
        "l = torch.tensor([4, 4], dtype=torch.int32, device='cuda')\n"
        "u = torch.tensor([2, 2], dtype=torch.int32, device='cuda')\n"
        "assert torch.equal(m(x, t, l, u), torchaudio.functional.rnnt_loss(x, t, l, u, blank=0))\n"
        "print('routed')\n"
    )
    env = dict(os.environ, B200A_REFERENCE="1")
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "routed" in out.stdout, out.stderr[-2000:]
