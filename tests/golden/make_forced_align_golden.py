#!/usr/bin/env python
"""Generate tests/golden/forced_align_ref_cases.npz, the forced_align fixture (run once, with torchaudio installed at
the pinned reference version):

    python tests/golden/make_forced_align_golden.py

torchaudio's forced_align runs on the CPU here, the parity target.  Stored:
- ``fx_<i>_*``: the reference's hand-worked emission cases of test_forced_align (blank 5) -- log-probs, targets,
  the reference CPU's paths and scores;
- ``rc_<i>``: seeded batch-1 recipes (tests/forced_align_oracle.py:case_inputs) with the reference CPU's ``path_<i>``
  (int16) and ``score_<i>`` (in the recipe's dtype);
- ``bt_<i>``: seeded ragged batch recipes (batch_inputs) with ``bpath_<i>`` / ``bscore_<i>``, each row the reference
  CPU's alignment of that row alone and the padding frames blank / 0;
- ``mt_<i>_{token,start,end,score}``: merge_tokens of recipe i's path and scores;
- ``err_<key>``: the reference's error strings ("<exception type>: <message>").
"""
import os
import re
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import torchaudio.functional as RF  # noqa: E402

import forced_align_oracle as O  # noqa: E402

EMISSION = [[0.633766, 0.221185, 0.0917319, 0.0129757, 0.0142857, 0.0260553],
            [0.111121, 0.588392, 0.278779, 0.0055756, 0.00569609, 0.010436],
            [0.0357786, 0.633813, 0.321418, 0.00249248, 0.00272882, 0.0037688],
            [0.0663296, 0.643849, 0.280111, 0.00283995, 0.0035545, 0.00331533],
            [0.458235, 0.396634, 0.123377, 0.00648837, 0.00903441, 0.00623107]]
FIXTURES = [([0, 1, 1, 0], 0), ([0, 1, 2, 3, 4], 0), ([3, 3, 3], 1), ([0, 1, 2], 1)]  # targets, tdtype code

RECIPES = [  # (seed, T (0: T = L + R), L, C, blank, dtype, tdtype, kind, heavy); kind per oracle._emission
    (1, 12, 4, 6, 0, 0, 0, 0, 0),
    (2, 0, 5, 6, 0, 0, 1, 0, 0),
    (3, 0, 6, 6, 3, 1, 0, 0, 1),
    (4, 20, 6, 6, 0, 2, 1, 1, 0),
    (5, 20, 8, 6, 5, 0, 0, 1, 1),
    (6, 0, 7, 6, 0, 1, 1, 1, 1),
    (7, 40, 10, 29, 0, 0, 0, 2, 0),
    (8, 40, 10, 29, 28, 1, 1, 2, 0),
    (9, 0, 12, 29, 0, 2, 0, 2, 1),
    (10, 60, 20, 29, 0, 1, 0, 1, 0),
    (11, 80, 25, 1024, 0, 0, 1, 0, 0),
    (12, 80, 25, 1024, 7, 1, 0, 1, 0),
    (13, 0, 30, 1024, 0, 2, 1, 2, 1),
    (14, 120, 40, 29, 0, 0, 0, 0, 1),
    (15, 1, 1, 6, 0, 0, 0, 0, 0),
    (16, 3, 1, 6, 0, 1, 1, 0, 0),
    (17, 3000, 1000, 32, 0, 0, 0, 0, 0),
    (18, 3000, 1000, 32, 0, 1, 1, 1, 0),
]
BATCHES = [  # (seed, B, T, L, C, blank, dtype, tdtype, kind, heavy)
    (40, 4, 30, 10, 6, 0, 0, 0, 0, 0),
    (41, 5, 50, 12, 29, 0, 1, 1, 1, 1),
    (42, 3, 64, 20, 29, 4, 2, 0, 2, 0),
    (43, 6, 300, 80, 32, 0, 0, 1, 0, 1),
]
MERGE = (0, 3, 5, 10, 14)


def ref(lp, tg, blank):
    p, s = RF.forced_align(torch.from_numpy(lp), torch.from_numpy(tg), blank=blank)
    return p[0].numpy(), s[0].numpy()


def err(fn):
    try:
        fn()
    except Exception as e:  # noqa: BLE001
        msg = re.sub(r"^\w+, \S+:\d+, ", "", str(e).splitlines()[0])  # the C++ check's "<function>, <file>:<line>, "
        return f"{type(e).__name__}: {msg}"
    raise AssertionError("expected an error")


def main():
    out = {}
    for i, (tg, tdc) in enumerate(FIXTURES):
        lp = np.log(np.array([EMISSION], dtype=np.float32))
        tg = np.array([tg], dtype=O.TDTYPES[tdc])
        p, s = ref(lp, tg, 5)
        out.update({f"fx_{i}_lp": lp, f"fx_{i}_tg": tg, f"fx_{i}_path": p.astype(np.int16), f"fx_{i}_score": s})
        print("fixture", i, p)
    for i, rc in enumerate(RECIPES):
        lp, tg, blank = O.case_inputs(rc)
        p, s = ref(lp, tg, blank)
        op, os_ = O.align(lp[0], tg[0], blank)
        assert np.array_equal(p, op) and np.array_equal(s, os_), rc
        out.update({f"rc_{i}": np.array(rc, dtype=np.int64), f"path_{i}": p.astype(np.int16), f"score_{i}": s})
        if i in MERGE:
            spans = RF.merge_tokens(torch.from_numpy(p), torch.from_numpy(s), blank=blank)
            out[f"mt_{i}_token"] = np.array([x.token for x in spans], dtype=np.int64)
            out[f"mt_{i}_start"] = np.array([x.start for x in spans], dtype=np.int64)
            out[f"mt_{i}_end"] = np.array([x.end for x in spans], dtype=np.int64)
            out[f"mt_{i}_score"] = np.array([x.score for x in spans], dtype=np.float64)
        print("recipe", i, rc, lp.shape)
    for i, rc in enumerate(BATCHES):
        lp, tg, tl, ul, blank = O.batch_inputs(rc)
        paths = np.full(lp.shape[:2], blank, dtype=np.int16)
        scores = np.zeros(lp.shape[:2], dtype=lp.dtype)
        for b in range(lp.shape[0]):
            p, s = ref(np.ascontiguousarray(lp[b: b + 1, : tl[b]]), np.ascontiguousarray(tg[b: b + 1, : ul[b]]),
                       blank)
            paths[b, : tl[b]] = p
            scores[b, : tl[b]] = s
        op, os_ = O.align_batch(lp, tg, tl, ul, blank)
        assert np.array_equal(paths, op) and np.array_equal(scores, os_), rc
        out.update({f"bt_{i}": np.array(rc, dtype=np.int64), f"bpath_{i}": paths, f"bscore_{i}": scores})
        print("batch", i, rc, tl, ul)

    g = torch.Generator().manual_seed(0)
    lp = torch.rand(1, 5, 6, generator=g)
    il, tl = torch.tensor([5]), torch.tensor([4])

    def call(lp=lp, tg=None, il=il, tl=tl, blank=5, dtype=torch.int32):
        tg = torch.tensor([[0, 1, 2, 3]], dtype=dtype) if tg is None else tg
        return lambda: RF.forced_align(lp, tg, il, tl, blank)

    errors = {}
    for dt, name in ((torch.int32, "i32"), (torch.int64, "i64")):
        errors.update({
            f"too_long_{name}": call(tg=torch.tensor([[0, 1, 2, 3, 4, 4]], dtype=dt), tl=torch.tensor([6]), dtype=dt),
            f"blank_in_{name}": call(tg=torch.tensor([[5, 3, 3]], dtype=dt), tl=torch.tensor([3])),
            f"lp_dtype_{name}": call(lp=lp.int(), dtype=dt),
            f"tg_dtype_{name}": call(tg=torch.tensor([[0., 1., 2., 3.]])),
            f"input_lengths_dim_{name}": call(il=torch.ones(3, 5, dtype=torch.int64), dtype=dt),
            f"target_lengths_dim_{name}": call(tl=torch.ones(3, 5, dtype=torch.int64), dtype=dt),
            f"input_length_{name}": call(il=torch.tensor([10000]), dtype=dt),
            f"target_length_{name}": call(tl=torch.tensor([10000]), dtype=dt),
            f"range_{name}": call(lp=torch.rand(1, 10, 5, generator=g), tg=torch.tensor([[7, 8, 9, 10]], dtype=dt)),
            f"blank_range_{name}": call(tg=torch.tensor([[1, 3, 3]], dtype=dt), tl=torch.tensor([3]), blank=10000),
        })
    errors.update({
        "empty_targets": call(tg=torch.zeros(1, 0, dtype=torch.int32), tl=torch.tensor([0])),
        "negative_blank": call(tg=torch.tensor([[1, 3, 3]]), tl=torch.tensor([3]), blank=-1),
        "lp_contiguous": call(lp=lp.transpose(1, 2).contiguous().transpose(1, 2)),
        "tg_contiguous": call(tg=torch.tensor([[1, 0, 2, 0, 3, 0, 4, 0]], dtype=torch.int32)[:, ::2]),
        "lp_dim": call(lp=lp[0]),
        "tg_dim": call(tg=torch.tensor([1, 2, 3, 4], dtype=torch.int32)),
    })
    for k, fn in errors.items():
        out[f"err_{k}"] = np.array(err(fn))
        print(k, out[f"err_{k}"])
    np.savez_compressed(os.path.join(HERE, "forced_align_ref_cases.npz"), **out)


if __name__ == "__main__":
    main()
