"""The numpy CTC prefix beam search (tests/ctc_decoder_oracle.py) against exact prefix probabilities and hand-worked
cases: frame skipping and a merge with a re-created prefix."""
import numpy as np
import pytest

import ctc_decoder_oracle as O


def _norm(x):
    return x - np.logaddexp.reduce(x, axis=1, keepdims=True)


@pytest.mark.parametrize("T", [1, 2, 3, 4])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_unpruned_scores_are_prefix_probabilities(T, seed):
    lp = _norm(np.random.default_rng(seed).standard_normal((T, 3)) * 2)
    hyps, _ = O.decode(lp, T, 1000, 0.0, oracle_beam=1000)
    exact = O.exact_prefix_scores(lp)
    got = dict(hyps)
    assert set(got) == set(exact)
    for k, v in exact.items():
        assert abs(got[k] - v) <= 1e-12 * max(1.0, abs(v))


def test_frame_skip_collapses_each_beam():
    # V = 3, frames 0 and 2 selected, frame 1 skipped (blank above the threshold)
    lp = np.log(np.array([[0.2, 0.5, 0.3], [0.99, 0.005, 0.005], [0.3, 0.3, 0.4]]))
    hyps, _ = O.decode(lp, 3, 3, np.log(0.95), oracle_beam=3)
    # step 0: "1" (0.5), "2" (0.3), "" (0.2), each collapsed to p_blank = its score since frame 1 is skipped
    # step 1 (frame 2): "1" -> stay 0.5 * 0.3 = 0.15, "11" = 0.5 * 0.3 = 0.15, "12" = 0.5 * 0.4 = 0.2; "2" -> stay
    # 0.3 * 0.3 = 0.09, "21" = 0.09, "22" = 0.3 * 0.4 = 0.12; "" -> stay 0.2 * 0.3 = 0.06, "1" 0.06 (merged: 0.21),
    # "2" 0.2 * 0.4 = 0.08 (merged: 0.09 + 0.08 = 0.17)
    want = {(1,): 0.21, (1, 2): 0.2, (2,): 0.17}
    assert {k: round(float(np.exp(v)), 12) for k, v in hyps} == want


def test_without_skip_repeats_stay_collapsed():
    lp = np.log(np.array([[0.2, 0.5, 0.3], [0.2, 0.5, 0.3]]))
    hyps, _ = O.decode(lp, 2, 1, 0.0)
    # beam 1 keeps "1" alone after step 0, so blank-1 is pruned: 1-1 and 1-blank = 0.25 + 0.1
    assert hyps[0][0] == (1,) and abs(np.exp(hyps[0][1]) - 0.35) < 1e-12


def test_recreated_prefix_merges_with_an_older_beam():
    # beam 2.  Step 0: "1" (0.6) and "" (0.3).  Step 1: "12" = 0.36 and "1" = 0.18 + 0.06 + 0.03 (the merged "" + 1)
    # = 0.27 survive.  Step 2: "1" + 2 re-creates "12", which must merge into the "12" beam of step 1:
    # 0.36 * (0.5 + 0.4) + 0.27 * 0.4 = 0.432, with one "12" hypothesis only.
    lp = np.log(np.array([[0.3, 0.6, 0.1], [0.3, 0.1, 0.6], [0.5, 0.1, 0.4]]))
    hyps, _ = O.decode(lp, 3, 2, 0.0)
    assert [k for k, _ in hyps] == [(1, 2), (1,)]
    assert abs(np.exp(hyps[0][1]) - 0.432) < 1e-12
    assert abs(np.exp(hyps[1][1]) - (0.27 * 0.5 + 0.09 * 0.1)) < 1e-12


def test_margins_and_rows_without_steps():
    lp = np.log(np.full((3, 4), 0.25))
    assert O.decode(lp, 3, 2, np.log(0.1)) == ([], [])
    assert O.decode(lp, 0, 2, 0.0) == ([], [])
    _, margins = O.decode(lp, 3, 2, 0.0)
    assert margins[0] == 0.0  # every entry of a flat row ties
