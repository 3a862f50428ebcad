"""The float64 RNN-T loss oracle (tests/rnnt_loss_oracle.py) against the reference CPU's costs and gradients stored in
tests/golden/rnnt_loss_ref_cases.npz, and against torchaudio's CPU rnnt_loss when it is importable."""
import numpy as np
import pytest

import rnnt_loss_oracle as O
from conftest import _load

FIXTURES = ("B1_T2_U3_D5", "B2_T4_U3_D3", "B1_T10_U3_D4")


@pytest.fixture(scope="module")
def ref():
    return _load("rnnt_loss_ref_cases.npz")


def _recipes(ref):
    return sorted(int(k[3:]) for k in ref if k.startswith("rc_"))


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_matches_hand_worked_fixtures(ref, name):
    p = f"fx_{name}_"
    c, g = O.rnnt_loss(ref[p + "logits"], ref[p + "targets"], ref[p + "tl"], ref[p + "ul"], int(ref[p + "blank"]),
                       -1.0, bool(ref[p + "fused"]))
    np.testing.assert_allclose(c, ref[p + "cost"], rtol=1e-6)
    np.testing.assert_allclose(g, ref[p + "grad"], atol=1e-6)


def test_oracle_matches_reference_recipes(ref):
    for i in _recipes(ref):
        lg, tg, tl, ul = O.case_inputs(ref[f"rc_{i}"])
        blank, clamp, fused = int(ref[f"rc_{i}"][5]), float(ref[f"clamp_{i}"]), bool(ref[f"fused_{i}"])
        c, g = O.rnnt_loss(lg, tg, tl, ul, blank, clamp, fused, grads=f"grad_{i}" in ref)
        rel = np.max(np.abs(c - ref[f"cost_{i}"]) / np.abs(c))
        assert rel <= float(ref[f"cerr_{i}"]) * 1.01 + 1e-12, (i, rel)
        if f"grad_{i}" in ref:
            assert np.max(np.abs(g - ref[f"grad_{i}"])) <= float(ref[f"gerr_{i}"]) * 1.01 + 1e-12, i


def test_recipe_shapes_and_lengths(ref):
    for i in _recipes(ref):
        rc = ref[f"rc_{i}"]
        lg, tg, tl, ul = O.case_inputs(rc)
        assert lg.shape == tuple(int(v) for v in rc[1:5]) and lg.dtype == (np.float16 if rc[6] else np.float32)
        assert tl.max() == rc[2] and ul.max() + 1 == rc[3] and tl.min() >= 1 and ul.min() >= 0
        assert tg.shape == (rc[1], rc[3] - 1) and ((tg >= 0) & (tg < rc[4])).all()


def test_nonfinite_cost_is_nan_and_its_gradient_zero(ref):
    lg, tg, tl, ul = O.case_inputs((30, 3, 6, 4, 5, -1, 0, 1.0))
    lg[1, :, :, 4] = -np.inf
    c, g = O.rnnt_loss(lg, tg, tl, ul)
    np.testing.assert_allclose(c, ref["nonfinite_cost"], rtol=1e-6)
    assert np.isnan(c[1]) and (g[1] == 0).all() and np.isfinite(g).all() and (g[0] != 0).any()


def test_clamp_is_symmetric():
    lg, tg, tl, ul = O.case_inputs((40, 2, 5, 4, 6, -1, 0, 3.0))
    g = O.rnnt_loss(lg, tg, tl, ul)[1]
    gc = O.rnnt_loss(lg, tg, tl, ul, clamp=0.05)[1]
    assert g.max() > 0.05 and g.min() < -0.05
    np.testing.assert_array_equal(gc, np.clip(g, -0.05, 0.05))


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("blank", [-1, 0, 3])
def test_oracle_against_installed_torchaudio(fused, blank):
    torch = pytest.importorskip("torch")
    try:
        import torchaudio.functional as TF
    except Exception:  # noqa: BLE001
        pytest.skip("torchaudio is not importable")
    lg, tg, tl, ul = O.case_inputs((50 + blank, 3, 9, 6, 7, blank, 0, 1.5))
    x = torch.from_numpy(lg).requires_grad_()
    c = TF.rnnt_loss(x, torch.from_numpy(tg), torch.from_numpy(tl), torch.from_numpy(ul), blank=blank, clamp=0.1,
                     reduction="none", fused_log_softmax=fused)
    c.sum().backward()
    oc, og = O.rnnt_loss(lg, tg, tl, ul, blank, 0.1, fused)
    np.testing.assert_allclose(c.detach().numpy(), oc, rtol=1e-6)
    np.testing.assert_allclose(x.grad.numpy(), og, atol=1e-5)
