"""The silhouette term of the perspective 2D fit restated on the CPU, in float64 where it computes (include/shapy_b200.h,
shapy_silhouette_*, shapy_render_silhouette): the exact squared distance transform (scipy), the contour rule and its
subsampling, pixel-centre rasterisation with an ambiguity band at the edges, the projection (in float32, in the
kernels' order of operations, as the fit sees it), bilinear sampling, brute-force closest points on 2D triangles, and
the term with its analytic gradient.  Imports without a GPU."""
import numpy as np
from scipy import ndimage

Z_NEAR = np.float32(1e-3)
AMBIGUOUS = 1e-3          # px: pixel centres this close to a triangle's edge may go either way in float32


# ------------------------------------------------------------------------------------------------ masks
def edt_sq(mask):
    """(H, W) int64: squared distance from each pixel centre to the nearest person pixel; 0 everywhere without one."""
    m = np.asarray(mask) != 0
    if not m.any():
        return np.zeros(m.shape, np.int64)
    d = ndimage.distance_transform_edt(~m)
    return np.rint(d * d).astype(np.int64)


def dist_f32(mask):
    """The float32 distance the device writes: sqrt of the float32 squared distance, correctly rounded."""
    return np.sqrt(edt_sq(mask).astype(np.float32))


def contour_pixels(mask):
    """(count, 2) int64 (r, c) of the person pixels with a 4-neighbour inside the image that is not a person pixel, in
    raster order."""
    m = np.asarray(mask) != 0
    out = np.zeros_like(m)
    out[:, 1:] |= ~m[:, :-1]
    out[:, :-1] |= ~m[:, 1:]
    out[1:, :] |= ~m[:-1, :]
    out[:-1, :] |= ~m[1:, :]
    return np.argwhere(m & out)


def kept_contour(mask, max_points):
    """(contour (max_points, 3) float32 of (c, r, 0) then zeros, weights (max_points,), count found)."""
    rc = contour_pixels(mask)
    n = len(rc)
    k = -(-n // max_points) if n > max_points else 1
    kept = rc[::k]
    pts = np.zeros((max_points, 3), np.float32)
    w = np.zeros(max_points, np.float32)
    pts[:len(kept), 0], pts[:len(kept), 1] = kept[:, 1], kept[:, 0]
    w[:len(kept)] = 1
    return pts, w, n


# ------------------------------------------------------------------------------------------------ projection
def project_f32(Y, intr, z_near=True):
    """(..., 2) float32 (u, v) of camera-frame points Y (..., 3) with intr (3,) (f, px, py), rounded step by step as
    the kernels do: u = f (Y_x / z) + px, z = max(Y_z, 1e-3) (z_near) or Y_z."""
    Y = np.asarray(Y, np.float32)
    f, px, py = (np.float32(c) for c in intr)
    z = np.maximum(Y[..., 2], Z_NEAR) if z_near else Y[..., 2]
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        return np.stack([f * (Y[..., 0] / z) + px, f * (Y[..., 1] / z) + py], -1).astype(np.float32)


def bilinear(dist, u, v):
    """D, dD/du, dD/dv (float64) of dist (H, W) at (u, v) (arrays) clamped to [0, W-1] x [0, H-1], in the cell
    c0 = min(floor(x), W - 2) (0 for W = 1), likewise r0; the derivative is 0 along an axis where (u, v) is clamped."""
    d = np.asarray(dist, np.float64)
    H, W = d.shape
    u, v = np.asarray(u, np.float64), np.asarray(v, np.float64)
    x, y = np.clip(u, 0, W - 1), np.clip(v, 0, H - 1)
    c0 = np.clip(np.minimum(np.floor(x).astype(np.int64), W - 2), 0, None)
    r0 = np.clip(np.minimum(np.floor(y).astype(np.int64), H - 2), 0, None)
    c1, r1 = np.minimum(c0 + 1, W - 1), np.minimum(r0 + 1, H - 1)
    fx, fy = x - c0, y - r0
    d00, d01, d10, d11 = d[r0, c0], d[r0, c1], d[r1, c0], d[r1, c1]
    top, bot = (1 - fx) * d00 + fx * d01, (1 - fx) * d10 + fx * d11
    D = (1 - fy) * top + fy * bot
    du = np.where((u >= 0) & (u <= W - 1), (1 - fy) * (d01 - d00) + fy * (d11 - d10), 0.0)
    dv = np.where((v >= 0) & (v <= H - 1), bot - top, 0.0)
    return D, du, dv


def cell_of(dist_shape, u, v):
    """The bilinear cell (c0, r0) and the clamping of each (u, v): equal before and after a step means the term is
    one bilinear polynomial along it."""
    H, W = dist_shape
    u, v = np.asarray(u, np.float64), np.asarray(v, np.float64)
    x, y = np.clip(u, 0, W - 1), np.clip(v, 0, H - 1)
    c0 = np.clip(np.minimum(np.floor(x).astype(np.int64), W - 2), 0, None)
    r0 = np.clip(np.minimum(np.floor(y).astype(np.int64), H - 2), 0, None)
    return np.stack([c0, r0, u < 0, u > W - 1, v < 0, v > H - 1], -1)


# ------------------------------------------------------------------------------------------------ rasterisation
def rasterise(Y, faces, intr, H, W):
    """(mask, ambiguous) (H, W) bool of the triangles faces (F, 3) of the camera-frame vertices Y (V, 3): a pixel is
    covered when its centre is inside a triangle whose three vertices have Y_z > 0 by more than AMBIGUOUS px from every
    edge, ambiguous when it is not covered but within AMBIGUOUS px of such a triangle (or of a degenerate one)."""
    Y = np.asarray(Y, np.float32)
    uv = project_f32(Y, intr, z_near=False).astype(np.float64)
    mask = np.zeros((H, W), bool)
    amb = np.zeros((H, W), bool)
    for f in np.asarray(faces):
        if not (Y[f, 2] > 0).all():
            continue
        t = uv[f]
        if not np.isfinite(t).all():
            continue
        lo, hi = t.min(0), t.max(0)
        x0, x1 = max(int(np.ceil(lo[0] - AMBIGUOUS)), 0), min(int(np.floor(hi[0] + AMBIGUOUS)), W - 1)
        y0, y1 = max(int(np.ceil(lo[1] - AMBIGUOUS)), 0), min(int(np.floor(hi[1] + AMBIGUOUS)), H - 1)
        if x0 > x1 or y0 > y1:
            continue
        xs, ys = np.meshgrid(np.arange(x0, x1 + 1, dtype=np.float64), np.arange(y0, y1 + 1, dtype=np.float64))
        area2 = (t[1, 0] - t[0, 0]) * (t[2, 1] - t[0, 1]) - (t[1, 1] - t[0, 1]) * (t[2, 0] - t[0, 0])
        if abs(area2) < 1e-12:
            amb[y0:y1 + 1, x0:x1 + 1] = True
            continue
        sgn = 1.0 if area2 > 0 else -1.0
        sd = []
        for a, b in ((0, 1), (1, 2), (2, 0)):
            e = t[b] - t[a]
            cross = e[0] * (ys - t[a, 1]) - e[1] * (xs - t[a, 0])
            sd.append(sgn * cross / np.hypot(*e))          # > 0 inside, in px from the edge's line
        sd = np.min(sd, 0)
        mask[y0:y1 + 1, x0:x1 + 1] |= sd > AMBIGUOUS
        amb[y0:y1 + 1, x0:x1 + 1] |= np.abs(sd) <= AMBIGUOUS
    return mask, amb & ~mask


# ------------------------------------------------------------------------------------------------ closest points
def closest_2d(points, tris):
    """Brute force, float64: for each point (N, 2) the squared distance to the nearest triangle of tris (F, 3, 2)
    (0 inside one) and the set of minimisers within `tol` is left to the caller: returns (sq_dist (N,), per-point
    per-triangle squared distances (N, F))."""
    p = np.asarray(points, np.float64)[:, None, :]
    t = np.asarray(tris, np.float64)[None]
    a, b, c = t[..., 0, :], t[..., 1, :], t[..., 2, :]

    def seg(p, a, b):
        ab = b - a
        L = (ab * ab).sum(-1)
        s = np.where(L > 0, ((p - a) * ab).sum(-1) / np.where(L > 0, L, 1), 0.0)
        q = a + np.clip(s, 0, 1)[..., None] * ab
        return ((p - q) ** 2).sum(-1)

    d2 = np.minimum(np.minimum(seg(p, a, b), seg(p, b, c)), seg(p, c, a))

    def cr(o, x, y):
        return (x[..., 0] - o[..., 0]) * (y[..., 1] - o[..., 1]) - (x[..., 1] - o[..., 1]) * (y[..., 0] - o[..., 0])
    e0, e1, e2 = cr(a, b, p), cr(b, c, p), cr(c, a, p)
    inside = ((e0 >= 0) & (e1 >= 0) & (e2 >= 0)) | ((e0 <= 0) & (e1 <= 0) & (e2 <= 0))
    d2 = np.where(inside, 0.0, d2)
    return d2.min(1), d2


# ------------------------------------------------------------------------------------------------ the term
def model_to_mask(Y, intr, dist):
    """(1/V) sum_v D(p_v)^2 at the float32 projection with the z_near clamp."""
    uv = project_f32(Y, intr)
    D, _, _ = bilinear(dist, uv[:, 0], uv[:, 1])
    return float((D * D).mean())


def term(Y, intr, dist, contour, contour_w, faces):
    """The unweighted term of one body: model_to_mask + mean over the kept contour pixels of the squared distance to
    the projected mesh (float64 brute force on the float32 projection)."""
    uv = project_f32(Y, intr)
    keep = np.asarray(contour_w) > 0
    s2m = 0.0
    if keep.any():
        d2, _ = closest_2d(np.asarray(contour)[keep, :2], uv[np.asarray(faces)])
        s2m = float(d2.mean())
    return model_to_mask(Y, intr, dist) + s2m


def gradient(Y, intr, dist, g, contour=None, contour_w=None, faces=None, face_idx=None, bary=None):
    """(V, 3) float64 gradient of g * term with respect to Y, D's bilinear gradient and, with the correspondences
    (face_idx (N,), bary (N, 3)) held, the mask -> model half: 2 (q_i - p_i) bary_ic / N at each corner, q_i the held
    closest point on the projected mesh.  The depth is clamped at z_near (no gradient there) as in the kernel."""
    Y = np.asarray(Y, np.float64)
    f, px, py = (float(c) for c in intr)
    V = Y.shape[0]
    uv = project_f32(Y.astype(np.float32), intr).astype(np.float64)
    D, du, dv = bilinear(dist, uv[:, 0], uv[:, 1])
    gu, gv = g * 2 * D * du / V, g * 2 * D * dv / V
    if face_idx is not None:
        keep = (np.asarray(contour_w) > 0) & (np.asarray(face_idx) >= 0)
        n = max(int((np.asarray(contour_w) > 0).sum()), 1)
        F = np.asarray(faces)
        for i in np.nonzero(keep)[0]:
            tri = F[face_idx[i]]
            q = (np.asarray(bary[i], np.float64)[:, None] * uv[tri]).sum(0)
            r = 2 * g * (q - np.asarray(contour[i][:2], np.float64)) / n
            for k in range(3):
                gu[tri[k]] += r[0] * bary[i][k]
                gv[tri[k]] += r[1] * bary[i][k]
    z = np.maximum(Y[:, 2], float(Z_NEAR))
    out = np.zeros_like(Y)
    out[:, 0] = gu * f / z
    out[:, 1] = gv * f / z
    out[:, 2] = np.where(Y[:, 2] > float(Z_NEAR), -(gu * f * Y[:, 0] / z + gv * f * Y[:, 1] / z) / z, 0.0)
    return out


def model_to_mask_f64(Y, intr, dist):
    """model_to_mask with the projection in float64 (for central differences of the oracle's own gradient)."""
    Y = np.asarray(Y, np.float64)
    f, px, py = (float(c) for c in intr)
    z = np.maximum(Y[:, 2], float(Z_NEAR))
    D, _, _ = bilinear(dist, f * Y[:, 0] / z + px, f * Y[:, 1] / z + py)
    return float((D * D).mean())


def iou(a, b):
    a, b = np.asarray(a) != 0, np.asarray(b) != 0
    u = (a | b).sum()
    return 1.0 if u == 0 else float((a & b).sum() / u)
