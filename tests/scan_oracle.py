"""Float64 NumPy restatement of the scan queries and the scan fit's distance terms, from their definitions.

    closest_on_faces(p, tri)            squared distance and barycentrics of the closest point of each point on each
                                        triangle: the orthogonal projection when it falls inside, else the nearest of
                                        the three edges (the only candidates on a zero-area triangle)
    closest_points(vertices, faces, points, weights)   brute force over all faces, the smallest face index on a tie
    nearest_points(queries, points, weights)           brute force, the smallest point index on a tie
    scan_loss / scan_loss_grad          sum_i w_i rho(d_i^2) / sum_i w_i at given correspondences, and its vertex gradient
    sq_dist_grad                        sum_i 2 g_i (q_i - p_i) bary_ic at corner c of face_i (the kernel's backward)
    sample_surface                      area-weighted samples of a mesh's surface
"""
import numpy as np


def _segment(ap, ab):
    """Parameter t in [0, 1] of the closest point a + t ab to p (ap = p - a); 0 on a zero-length segment."""
    l2 = (ab * ab).sum(-1)
    t = np.where(l2 > 0, (ap * ab).sum(-1) / np.where(l2 > 0, l2, 1.0), 0.0)
    return np.clip(t, 0.0, 1.0)


def closest_on_faces(p, tri):
    """p (n, 3), tri (F, 3, 3) -> (d2 (n, F), bary (n, F, 3)) of the closest point of each point on each triangle."""
    p = np.asarray(p, np.float64)[:, None, :]
    a, b, c = (np.asarray(tri, np.float64)[None, :, k, :] for k in range(3))
    ab, ac, ap = b - a, c - a, p - a
    # interior: solve the 2x2 Gram system for the projection's (v, w); inside when v, w >= 0 and v + w <= 1
    g00, g01, g11 = (ab * ab).sum(-1), (ab * ac).sum(-1), (ac * ac).sum(-1)
    r0, r1 = (ab * ap).sum(-1), (ac * ap).sum(-1)
    det = g00 * g11 - g01 * g01
    ok = det > 0
    sd = np.where(ok, det, 1.0)
    v = (g11 * r0 - g01 * r1) / sd
    w = (g00 * r1 - g01 * r0) / sd
    inside = ok & (v >= 0) & (w >= 0) & (v + w <= 1)
    # edges ab, ac, bc as (v, w) pairs
    t0, t1, t2 = _segment(ap, ab), _segment(ap, ac), _segment(p - b, c - b)
    cands = [(t0, np.zeros_like(t0)), (np.zeros_like(t1), t1), (1.0 - t2, t2)]

    def d2_of(vv, ww):
        d = ap - ab * vv[..., None] - ac * ww[..., None]
        return (d * d).sum(-1)

    best = d2_of(*cands[0])
    bv, bw = cands[0]
    for cv, cw in cands[1:]:
        e = d2_of(cv, cw)
        take = e < best
        best, bv, bw = np.where(take, e, best), np.where(take, cv, bv), np.where(take, cw, bw)
    d2 = np.where(inside, d2_of(v, w), best)
    vv, ww = np.where(inside, v, bv), np.where(inside, w, bw)
    return d2, np.stack([1.0 - vv - ww, vv, ww], -1)


def closest_points(vertices, faces, points, weights=None, chunk=32):
    """One body: vertices (V, 3), faces (F, 3), points (N, 3).  Returns (face (N,), bary (N, 3), d2 (N,), second (N,)),
    second the smallest float64 squared distance over the other faces (how unique the winner is); a point with weight
    <= 0 gets face -1, zeros."""
    tri = np.asarray(vertices, np.float64)[np.asarray(faces)]
    N = len(points)
    face, bary = np.full(N, -1, np.int64), np.zeros((N, 3))
    d2, second = np.zeros(N), np.zeros(N)
    keep = np.ones(N, bool) if weights is None else np.asarray(weights) > 0
    idx = np.nonzero(keep)[0]
    for s in range(0, len(idx), chunk):
        rows = idx[s:s + chunk]
        e, bc = closest_on_faces(np.asarray(points, np.float64)[rows], tri)
        f = np.argmin(e, 1)                           # the first minimum: the smallest face index on a tie
        r = np.arange(len(rows))
        face[rows], d2[rows], bary[rows] = f, e[r, f], bc[r, f]
        e[r, f] = np.inf
        second[rows] = e.min(1)
    return face, bary, d2, second


def nearest_points(queries, points, weights=None):
    """One body: the nearest point with weight > 0 of each query, (idx (Q,), d2 (Q,), second (Q,)); -1 and 0 without
    one."""
    q, p = np.asarray(queries, np.float64), np.asarray(points, np.float64)
    keep = np.ones(len(p), bool) if weights is None else np.asarray(weights) > 0
    if not keep.any():
        return np.full(len(q), -1), np.zeros(len(q)), np.full(len(q), np.inf)
    pk = np.where(keep[:, None], p, 0.0)
    e = ((q[:, None, :] - pk[None]) ** 2).sum(-1)
    e[:, ~keep] = np.inf
    i = np.argmin(e, 1)
    r = np.arange(len(q))
    d2 = e[r, i]
    e[r, i] = np.inf
    return i, d2, e.min(1)


def rho(e, sigma=None):
    return e if sigma is None else sigma * sigma * e / (sigma * sigma + e)


def _closest(vertices, faces, face, bary):
    tri = np.asarray(vertices, np.float64)[np.asarray(faces)[face]]        # (N, 3, 3)
    return (np.asarray(bary, np.float64)[:, :, None] * tri).sum(1)


def scan_loss(vertices, faces, points, weights, face, bary, sigma=None):
    """sum_i w_i rho(|q_i - p_i|^2) / sum_i w_i over the points with w_i > 0, q_i = sum_c bary_ic x_c of face_i."""
    w = np.asarray(weights, np.float64)
    keep = w > 0
    q = _closest(vertices, faces, np.where(keep, face, 0), bary)
    d2 = ((q - np.where(keep[:, None], points, 0.0)) ** 2).sum(-1)
    return float((np.where(keep, w * rho(d2, sigma), 0.0)).sum() / w[keep].sum())


def sq_dist_grad(vertices, faces, points, face, bary, g):
    """sum_i 2 g_i (q_i - p_i) bary_ic scattered to the vertex at corner c of face_i; points with face < 0 add
    nothing."""
    out = np.zeros(np.shape(vertices), np.float64)
    keep = np.asarray(face) >= 0
    f, bc = np.asarray(face)[keep], np.asarray(bary, np.float64)[keep]
    q = _closest(vertices, faces, f, bc)
    r = 2.0 * np.asarray(g, np.float64)[keep][:, None] * (q - np.asarray(points, np.float64)[keep])
    for c in range(3):
        np.add.at(out, np.asarray(faces)[f, c], bc[:, c:c + 1] * r)
    return out


def scan_loss_grad(vertices, faces, points, weights, face, bary, sigma=None):
    """The gradient of scan_loss with respect to the vertices, face and barycentrics held."""
    w = np.asarray(weights, np.float64)
    keep = w > 0
    q = _closest(vertices, faces, np.where(keep, face, 0), bary)
    d2 = ((q - np.where(keep[:, None], points, 0.0)) ** 2).sum(-1)
    drho = np.ones_like(d2) if sigma is None else sigma ** 4 / (sigma * sigma + d2) ** 2
    g = np.where(keep, w * drho, 0.0) / w[keep].sum()
    return sq_dist_grad(vertices, faces, points, np.where(keep, face, -1), bary, g)


def sample_surface(vertices, faces, n, rng):
    """n area-weighted uniform samples of the mesh's surface: (points (n, 3), face (n,), bary (n, 3))."""
    tri = np.asarray(vertices, np.float64)[np.asarray(faces)]
    area = 0.5 * np.linalg.norm(np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]), axis=1)
    face = rng.choice(len(tri), size=n, p=area / area.sum())
    r1, r2 = np.sqrt(rng.random(n)), rng.random(n)
    bary = np.stack([1 - r1, r1 * (1 - r2), r1 * r2], 1)
    return (bary[:, :, None] * tri[face]).sum(1), face, bary
