"""vad on the GPU against the reference fixture (tests/golden/make_vad_golden.py): output lengths on every case,
measures within twice the reference's own float32 error (the float64 oracle's distance to it) plus 1e-5, the same
decisions for every chunk length, bit-identical reruns, the gradient through the trim, the module, and the errors."""
import ast
import os
import warnings

import numpy as np
import pytest
import torch

import vad_oracle as O

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vad_ref_cases.npz")
DEV = torch.device("cuda")


@pytest.fixture(scope="module")
def ref():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def _case(ref, c):
    return (torch.from_numpy(np.ascontiguousarray(O.case_input(ref, c))).to(DEV), int(ref[f"sr_{c}"]),
            ast.literal_eval(str(ref[f"kw_{c}"])))


def _names(ref):
    return [k[4:] for k in ref if k.startswith("len_")]


def _measure(x, sr, kw, chunk=None):
    from audio_b200 import _filtering

    plan = _filtering.VadPlan(sr, **kw)
    x2 = x.reshape(-1, x.shape[-1])
    trigger, start, meas = plan.run(x2, keep_measures=True, **({} if chunk is None else dict(chunk=chunk)))
    return trigger, start, meas.T.cpu().numpy().astype(np.float64)  # (frames, channels)


def test_output_lengths_and_views(ref):
    import audio_b200.functional as F

    for c in _names(ref):
        x, sr, kw = _case(ref, c)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            y = F.vad(x, sr, **kw)
        assert y.shape[:-1] == x.shape[:-1] and y.shape[-1] == int(ref[f"len_{c}"]), c
        if y.numel():  # a view of the input's last samples (the trim keeps the tail, or the fixed pre-trigger head)
            assert y.untyped_storage().data_ptr() == x.untyped_storage().data_ptr(), c
            lead = x.reshape(-1, x.shape[-1])
            assert torch.equal(y.reshape(-1, y.shape[-1]), lead[:, lead.shape[1] - y.shape[-1]:]) or \
                torch.equal(y.reshape(-1, y.shape[-1]), lead[:, :y.shape[-1]]), c


def test_measures_match_reference(ref):
    for c in _names(ref):
        exp = ref[f"meas_{c}"]
        if exp.shape[0] == 0:
            continue
        x, sr, kw = _case(ref, c)
        trigger, _, got = _measure(x, sr, kw)
        assert got.shape[0] >= exp.shape[0], c
        got = got[:exp.shape[0]]
        spread = np.abs(O.measures(x.cpu().numpy(), sr, dtype=np.float64, **kw)[:exp.shape[0]] - exp).max()
        err = np.abs(got - exp).max()
        assert err <= 2 * spread + 1e-5, (c, err, spread)


@pytest.mark.parametrize("case", ["mono_all", "stereo_all", "long", "burst_before"])
def test_chunk_length_changes_no_decision(ref, case):
    """Any chunk length gives the same trigger frame and start, and measures within the parity bound.  The walk and
    trigger state carries across chunks exactly, but the front end packs two frames into one complex FFT inside a
    launch, so |X| and P of frames next to a chunk edge can differ from a one-chunk run in the last bits."""
    x, sr, kw = _case(ref, case)
    exp = ref[f"meas_{case}"]
    spread = np.abs(O.measures(x.cpu().numpy(), sr, dtype=np.float64, **kw)[:exp.shape[0]] - exp).max()
    frames = O.num_frames(O.constants(sr, **kw), x.shape[-1])
    base = _measure(x, sr, kw, chunk=frames)
    for chunk in (1, 7, 1024):
        got = _measure(x, sr, kw, chunk=chunk)
        assert got[:2] == base[:2], (chunk, got[:2], base[:2])
        assert got[2].shape[0] >= exp.shape[0], chunk
        err = np.abs(got[2][:exp.shape[0]] - exp).max()
        assert err <= 2 * spread + 1e-5, (chunk, err, spread)


def test_reruns_are_bit_identical(ref):
    x, sr, kw = _case(ref, "stereo_all")
    a, b = _measure(x, sr, kw), _measure(x, sr, kw)
    assert a[:2] == b[:2] and np.array_equal(a[2], b[2])


def test_gradient_through_the_trim(ref):
    import audio_b200.functional as F

    x, sr, kw = _case(ref, "stereo")
    x = x.clone().requires_grad_(True)
    y = F.vad(x, sr, **kw)
    g = torch.randn(y.shape, device=DEV, generator=torch.Generator(DEV).manual_seed(3))
    (g * y).sum().backward()
    exp = torch.zeros_like(x)
    exp[..., x.shape[-1] - y.shape[-1]:] = g
    assert torch.equal(x.grad, exp)


def test_module_equals_functional(ref):
    import audio_b200.functional as F
    import audio_b200.transforms as T

    x, sr, _ = _case(ref, "burst_after")
    kw = dict(trigger_level=6.5, allowed_gap=0.1, pre_trigger_time=0.05)
    m = T.Vad(sr, **kw)
    for _ in range(2):  # the second call reuses the module's plan
        assert torch.equal(m(x), F.vad(x, sr, **kw))
    m.trigger_level = 1e9  # a changed attribute is honoured, as the reference reads them at forward
    assert torch.equal(m(x), F.vad(x, sr, **dict(kw, trigger_level=1e9))) and m(x).shape[-1] == 800


def test_errors():
    import audio_b200.functional as F

    x = torch.zeros(2, 16000, device=DEV)
    with pytest.raises(TypeError, match="must be float32"):
        F.vad(x.double(), 16000)
    with pytest.raises(RuntimeError, match="no CPU or ATen fallback"):
        F.vad(x.cpu(), 16000)
    with pytest.raises(RuntimeError, match=r"dft_len_ws = 16384.*capped at 8192"):
        F.vad(torch.zeros(1, 96000, device=DEV), 96000)
