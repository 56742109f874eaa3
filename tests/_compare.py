"""Comparison of kernel outputs with the oracle's, shared by the GPU test files."""
import numpy as np


def _canon(x):
    x = np.ascontiguousarray(x)
    if x.dtype.kind == "f":
        x = np.where(np.isnan(x), np.array(np.nan, x.dtype), x)
    return x


def assert_same_bytes(got, want, what=""):
    """Byte-identical after canonicalising NaN payloads: +inf != -inf, 0.0 != -0.0, NaN != any number."""
    got, want = _canon(got), _canon(want)
    assert got.dtype == want.dtype and got.shape == want.shape, f"{what}: {got.dtype}{got.shape} vs {want.dtype}{want.shape}"
    same = (got.view(np.uint8).reshape(got.shape + (-1,)) == want.view(np.uint8).reshape(want.shape + (-1,))).all(-1)
    if not same.all():
        bad = np.argwhere(~same)[:5]
        raise AssertionError(f"{what}: {int((~same).sum())} elements differ, first at {bad.tolist()}: "
                             f"{[got[tuple(i)] for i in bad]} vs {[want[tuple(i)] for i in bad]}")
