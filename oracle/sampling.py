"""float64 statement of top-k / nucleus (top-p) filtering of one sampling step (db200_sample_rows_filtered).

x is the already temperature-scaled row (logits * inv_temp, computed in fp32 like the kernel, then widened).  Per row:
  top-k (k >= 1; 0 / None = off): keep x_c >= tau_k, the k-th largest finite x counting multiplicity (ties kept);
  top-p (0 < p <= 1; 1 / None = off): over the top-k survivors K1, w = exp(x - max), Z = sum_K1 w; keep c iff
         A(c) = sum_{j in K1, x_j > x_c} w_j < p * Z   (the mass strictly above c, so ties share one decision).
NaN and -inf are never kept; if +inf is present the +inf entries are the only ones kept; a row with no finite entry
keeps nothing.  Test infrastructure only: nothing in the package imports this module.
"""
import numpy as np


def _rows(x):
    x = np.asarray(x, dtype=np.float64)
    return x.reshape(1, -1) if x.ndim == 1 else x


def _k1_and_cuts(row, top_k, cuts=True):
    """(top-k mask, distinct surviving values in descending order, mass strictly above each, Z), or the mask alone
    (None for the rest) when the row has +inf or no finite entry, or cuts is False."""
    valid = ~np.isnan(row) & (row > -np.inf)
    if np.isposinf(row).any():
        return np.isposinf(row), None, None, None
    if not valid.any():
        return valid, None, None, None
    k1 = valid
    nv = int(valid.sum())
    if top_k and top_k < nv:
        tau = np.partition(row[valid], nv - top_k)[nv - top_k]     # k-th largest, counting multiplicity
        k1 = valid & (row >= tau)
    if not cuts:
        return k1, None, None, None
    vals, inv = np.unique(row[k1], return_inverse=True)       # ascending distinct values
    w = np.exp(row[k1] - vals[-1])
    group = np.bincount(inv, weights=w, minlength=len(vals))[::-1]   # mass of each distinct value, descending
    above = np.concatenate([[0.0], np.cumsum(group)[:-1]])
    return k1, vals[::-1], above, group.sum()


def keep_mask(x, top_k=0, top_p=1.0):
    """bool array shaped like x: the ids the filter keeps in each row."""
    rows = _rows(x)
    top_k = int(top_k or 0)
    top_p = 1.0 if top_p is None else float(top_p)
    out = np.zeros(rows.shape, dtype=bool)
    for r, row in enumerate(rows):
        k1, vals, above, z = _k1_and_cuts(row, top_k, cuts=top_p < 1.0)
        if vals is None:
            out[r] = k1
            continue
        kept_vals = vals[above < top_p * z]
        out[r] = k1 & (row >= kept_vals[-1])
    return out.reshape(np.shape(x))


def boundary_margin(x, top_k=0, top_p=1.0):
    """Per row: min over the candidate top-p cuts (distinct surviving values) of |mass above - p * Z| / Z, the distance
    of the row's decision from a tie; inf where top-p is off or cannot apply.  A kernel that sums the masses with
    relative error e can only disagree with keep_mask on rows whose margin is below about e."""
    rows = _rows(x)
    top_k = int(top_k or 0)
    top_p = 1.0 if top_p is None else float(top_p)
    out = np.full(rows.shape[0], np.inf)
    if top_p >= 1.0:
        return out
    for r, row in enumerate(rows):
        _, vals, above, z = _k1_and_cuts(row, top_k)
        if vals is not None:
            out[r] = np.abs(above - top_p * z).min() / z
    return out
