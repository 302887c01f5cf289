"""TEST INFRASTRUCTURE ONLY -- exact 2-D convex hull of float32 points, for the circumference tests.

The hull is taken in xz, as body_measurements.py:165 hands qhull the (x, z) columns.  Andrew's monotone chain runs on
`fractions.Fraction` copies of the float32 coordinates, so every orientation test is exact: collinear points on a hull
edge are dropped, and a set whose hull has zero area (fewer than 3 distinct xz positions, or all of them collinear) is
reported as such instead of being given a perimeter.  Among points that share (x, z), the one that comes first in
(y, z, x) bit order stands for the position, as in csrc/measure.cu.  The perimeter sums the 3-D edge lengths of the
hull's vertices in float64.
"""
from fractions import Fraction

import numpy as np


def _ord_bits(a):
    """Total order on float32 bit patterns (-0 before +0), as ord_bits() in csrc/measure.cu."""
    i = np.asarray(a, np.float32).view(np.int32).astype(np.int64)
    return np.where(i >= 0, i, i ^ 0x7fffffff)


def representatives(pts):
    """Index of one point per distinct (x, z) float value: the first in (y, z, x) bit order."""
    pts = np.asarray(pts, np.float32).reshape(-1, 3)
    best = {}
    for i, (x, y, z) in enumerate(pts.tolist()):
        key = (x, z)                    # float equality: -0.0 and +0.0 share a position
        k = (int(_ord_bits(pts[i, 1])), int(_ord_bits(pts[i, 2])), int(_ord_bits(pts[i, 0])))
        if key not in best or k < best[key][0]:
            best[key] = (k, i)
    return sorted(i for _, i in best.values())


def hull_indices(pts):
    """Counter-clockwise hull vertices (indices into pts) in xz, or None when the hull has zero area."""
    pts = np.asarray(pts, np.float32).reshape(-1, 3)
    idx = representatives(pts)
    key = {i: (Fraction(float(pts[i, 0])), Fraction(float(pts[i, 2]))) for i in idx}
    order = sorted(idx, key=lambda i: key[i])
    if len(order) < 3:
        return None

    def cross(o, a, b):
        (ox, oz), (ax, az), (bx, bz) = key[o], key[a], key[b]
        return (ax - ox) * (bz - oz) - (az - oz) * (bx - ox)

    lower, upper = [], []
    for i in order:
        while len(lower) >= 2 and cross(lower[-2], lower[-1], i) <= 0:
            lower.pop()
        lower.append(i)
    for i in reversed(order):
        while len(upper) >= 2 and cross(upper[-2], upper[-1], i) <= 0:
            upper.pop()
        upper.append(i)
    hull = lower[:-1] + upper[:-1]
    return hull if len(hull) >= 3 else None


def perimeter(pts):
    """float64 sum of the 3-D lengths of the hull's edges; NaN when the xz hull has zero area."""
    pts = np.asarray(pts, np.float32).reshape(-1, 3)
    h = hull_indices(pts)
    if h is None:
        return float('nan')
    p = pts[h].astype(np.float64)
    d = np.roll(p, -1, axis=0) - p
    return float(np.sqrt((d * d).sum(-1)).sum())
