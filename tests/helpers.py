"""Shared helpers of the test-suite (comparison metrics, minibatch padding like the reference's tests/utils.py)."""
import numpy as np


def to_minibatch(arrays, batch_size=4, target_num=2):
    """tests/utils.py:7-15 of the reference: the real data goes to slot `target_num`, zeros elsewhere."""
    out = []
    for a in arrays:
        a = np.asarray(a)
        b = np.zeros((batch_size,) + a.shape, a.dtype)
        b[target_num] = a
        out.append(b)
    return out


def rel_err(x, ref):
    """max-abs-error / max-abs-reference per tensor (SURVEY.md 8(d) parity gate)."""
    x = np.asarray(x, np.float64)
    ref = np.asarray(ref, np.float64)
    den = np.abs(ref).max()
    if den == 0:
        return float(np.abs(x).max())
    return float(np.abs(x - ref).max() / den)


def elem_err(x, ref, floor=1e-3):
    """per-element gate: max over the elements of |x - ref| / max(|ref|, floor * max|ref|).  `elem_err(x, ref) <= tol`
    holds every component to tol of its own size, and components below floor x the tensor maximum to tol x floor x
    the maximum, so a wrong contribution to a small component cannot hide behind the largest one (rel_err can).  NaN
    anywhere in x gives NaN, which fails every `<=` gate."""
    x = np.asarray(x, np.float64)
    ref = np.asarray(ref, np.float64)
    if x.size == 0:
        return 0.0
    m = np.abs(ref).max()
    if m == 0:
        return float(np.abs(x).max()) if np.isfinite(x).all() else float("nan")
    den = np.maximum(np.abs(ref), floor * m)
    d = np.abs(x - ref) / den
    return float("nan") if np.isnan(d).any() else float(d.max())


def np_(t):
    return t.detach().cpu().numpy()
