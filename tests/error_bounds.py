"""Per-element error bounds shared by the kernel-vs-float64 tests: the unit roundoff of each precision mode, and the
report of the element that exceeds its tolerance the most."""
import numpy as np

U16, U22, U24 = 2.0 ** -11, 2.0 ** -22, 2.0 ** -24   # unit roundoff of fp16, of the hi+lo pair, of fp32
UNIT = {"f32": U24, "f16tc": U16, "f16x3": U22}


def worst(err, tol):
    """Index and values of the element that exceeds its tolerance the most (for the assertion message)."""
    bad = ~(err <= tol)
    ratio = np.where(bad, np.where(np.isfinite(err), err, np.inf) / np.maximum(tol, 1e-300), 0)
    at = np.unravel_index(np.argmax(ratio), err.shape)
    return "%d elements over; worst at %s: err %.4g tol %.4g" % (bad.sum(), at, err[at], tol[at])
