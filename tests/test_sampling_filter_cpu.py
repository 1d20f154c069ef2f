"""The float64 statement of top-k / nucleus filtering (oracle/sampling.py) that the GPU tests hold the filtered sampler
to: equal to the usual sort-based formulation on tie-free rows, and pinned by hand on the rows where ties, non-finite
values or degenerate sizes decide the answer."""
import math

import numpy as np
import pytest

from oracle.sampling import boundary_margin, keep_mask

INF, NAN = float("inf"), float("nan")

# (name, x, top_k, top_p, expected keep mask).  x is the temperature-scaled row.  tests/test_sampling_filter_gpu.py
# runs the same rows through the kernel.
ADVERSARIAL = [
    ("kth_value_tied", [3.0, 1.0, 2.0, 2.0, 2.0, 0.0], 2, 1.0, [1, 0, 1, 1, 1, 0]),
    ("kth_value_tied_top", [5.0, 5.0, 5.0, 1.0], 1, 1.0, [1, 1, 1, 0]),
    # w = 4, 1, 1, 1, 1, e^-5: the mass above each 0 is 4 < 0.6 Z, so the whole run of equal values is kept ...
    ("top_p_cut_in_run", [math.log(4.0), 0.0, 0.0, 0.0, 0.0, -5.0], 0, 0.6, [1, 1, 1, 1, 1, 0]),
    # ... and at 0.45 Z none of it is, though part of the run would fit in a sort-order cumulative sum
    ("top_p_cut_before_run", [math.log(4.0), 0.0, 0.0, 0.0, 0.0, -5.0], 0, 0.45, [1, 0, 0, 0, 0, 0]),
    ("top_k_then_top_p", [math.log(4.0), 0.0, 0.0, 0.0, 0.0, -5.0], 3, 0.6, [1, 1, 1, 1, 1, 0]),
    ("k_above_n", [0.5, -1.0, 2.0], 10, 1.0, [1, 1, 1]),
    ("k_above_n_top_p", [0.5, -1.0, 2.0], 10, 0.5, [0, 0, 1]),
    ("n_is_1", [0.3], 1, 0.5, [1]),
    ("n_is_1_off", [-7.0], 0, 1.0, [1]),
    ("minus_inf_and_nan", [-INF, 1.0, NAN, 0.5, -INF], 0, 1.0, [0, 1, 0, 1, 0]),
    ("minus_inf_and_nan_k1", [-INF, 1.0, NAN, 0.5, -INF], 1, 1.0, [0, 1, 0, 0, 0]),
    ("minus_inf_and_nan_k_above_finite", [-INF, 1.0, NAN, 0.5, -INF], 3, 0.999, [0, 1, 0, 1, 0]),
    ("plus_inf", [1.0, INF, 2.0, INF, NAN], 0, 1.0, [0, 1, 0, 1, 0]),
    ("plus_inf_filtered", [1.0, INF, 2.0, INF, NAN], 1, 0.5, [0, 1, 0, 1, 0]),
    ("all_minus_inf", [-INF, -INF, -INF, -INF], 2, 0.9, [0, 0, 0, 0]),
    ("all_nan_or_minus_inf", [NAN, -INF, NAN], 0, 1.0, [0, 0, 0]),
    ("signed_zeros_tie", [-0.0, 0.0, -1.0], 1, 1.0, [1, 1, 0]),
]


def sorted_restatement(x, k, p):
    """Sort descending; top-k keeps the first k positions; top-p keeps while the exclusive cumulative softmax of the
    top-k survivors is < p (HF's TopKLogitsWarper then TopPLogitsWarper on a tie-free row)."""
    order = np.argsort(-x, kind="stable")
    s = x[order]
    m = len(s) if not k else min(k, len(s))
    keep = np.zeros(len(s), dtype=bool)
    keep[:m] = True
    if p < 1.0:
        w = np.exp(s[:m] - s[0])
        excl = (np.cumsum(w) - w) / w.sum()
        keep[:m] = excl < p
    out = np.zeros(len(s), dtype=bool)
    out[order[keep]] = True
    return out


@pytest.mark.parametrize("n", [1, 7, 300, 4000])
def test_keep_mask_equals_the_sort_based_formulation_on_tie_free_rows(n):
    rng = np.random.default_rng(n)
    checked = 0
    for inv_temp in (0.7, 1.0, 1.5):
        for scale in (0.5, 3.0):
            # distinct by construction: a shuffled grid of spacing 6 / n, jittered by less than a third of it
            grid = np.linspace(-3.0, 3.0, n) + rng.uniform(-1.0, 1.0, (6, n)) / n
            logits = (rng.permuted(grid, axis=1) * scale).astype(np.float32)
            x = (logits * np.float32(inv_temp)).astype(np.float64)
            assert all(len(np.unique(r)) == n for r in x)
            for k in sorted({0, 1, 5, 50, max(n - 1, 1), n + 3}):
                for p in (0.1, 0.5, 0.9, 0.999, 1.0):
                    got = keep_mask(x, k, p)
                    margin = boundary_margin(x, k, p)
                    for r in range(x.shape[0]):
                        if margin[r] < 1e-9:
                            continue      # the two summation orders may round either way of p * Z
                        assert np.array_equal(got[r], sorted_restatement(x[r], k, p)), (n, inv_temp, k, p, r)
                        checked += 1
    assert checked > 0.99 * 6 * 6 * 5 * len({0, 1, 5, 50, max(n - 1, 1), n + 3})


@pytest.mark.parametrize("name,x,k,p,want", ADVERSARIAL, ids=[a[0] for a in ADVERSARIAL])
def test_keep_mask_on_hand_built_rows(name, x, k, p, want):
    got = keep_mask(np.array(x), k, p)
    assert got.tolist() == [bool(v) for v in want]


def test_keep_mask_shapes_and_off_switches():
    x = np.array([[1.0, 3.0, 2.0], [0.0, -1.0, 5.0]])
    assert keep_mask(x, 0, 1.0).all() and keep_mask(x, None, None).all()
    assert keep_mask(x, 1, 1.0).tolist() == [[False, True, False], [False, False, True]]
    assert keep_mask(x[0], 2).tolist() == [False, True, True]


def test_boundary_margin_is_the_distance_of_the_nearest_cut():
    # w = 4, 1, 1, 1, 1 (Z = 8): cuts at mass above 0 and 4; p Z = 4.8 -> nearest |4 - 4.8| / 8 = 0.1
    x = np.array([math.log(4.0), 0.0, 0.0, 0.0, 0.0])
    assert boundary_margin(x, 0, 0.6)[0] == pytest.approx(0.1)
    assert boundary_margin(x, 0, 0.5)[0] == pytest.approx(0.0, abs=1e-12)    # 0.5 Z = 4: exactly on a cut
    assert math.isinf(boundary_margin(x, 0, 1.0)[0])                           # top-p off: no cut to be near
    assert math.isinf(boundary_margin(np.array([-INF, NAN]), 0, 0.5)[0])
