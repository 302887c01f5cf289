"""TEST INFRASTRUCTURE ONLY -- float64 restatement of the exact circumference derivative of the measurement kernels
(shapy_measure_backward_exact, shapy_measure_jacobian_betas_exact in csrc/measure.cu).

Not a test module.  The hull is the kernels' own walk (oracle/measure_grad_oracle.hull_cycle).  Each hull point's ray
(which of the six rays of isect_points gave its first hit) comes from a float32 restatement of that ray order
(first_ray), so the combinatorics are the kernels'.  The closed-form adjoints (DESIGN.md section 4) are evaluated in
float64:
  edge point  (ray 3-5, triangle edge a -> b)  p = a + s (b - a), s = (h - a_y) / (b_y - a_y)
  line point  (ray 0-2, query edge o + s w)    p = o + s w, s = n.(v0 - o) / n.w, o_y = h
  no hit                                       p constant
and the plane height's adjoint goes to the y components of the landmark face's corners, weighted by its barycentrics.
Mass and height terms are measure_grad_oracle's.
"""
import numpy as np

from oracle import measure_grad_oracle, measure_oracle as mo

PLANES = ('chest', 'waist', 'hips')
F32 = np.float32


def _sub(a, b):
    return [F32(a[i] - b[i]) for i in range(3)]


def _dot(a, b):
    return F32(F32(F32(a[0] * b[0]) + F32(a[1] * b[1])) + F32(a[2] * b[2]))


def _cross(a, b):
    return [F32(F32(a[1] * b[2]) - F32(a[2] * b[1])), F32(F32(a[2] * b[0]) - F32(a[0] * b[2])),
            F32(F32(a[0] * b[1]) - F32(a[1] * b[0]))]


def _ray_hits(orig, d, v0, v1, v2):
    """mmi_device.cuh ray_tri in float32 (no FMA), and the first-hit rule 0 <= t <= 1."""
    e1, e2 = _sub(v1, v0), _sub(v2, v0)
    pvec = _cross(d, e2)
    det = _dot(e1, pvec)
    if abs(float(det)) < 1e-4:
        return False
    inv = F32(F32(1.0) / det)
    tvec = _sub(orig, v0)
    u = F32(_dot(tvec, pvec) * inv)
    if u < 0 or u > 1:
        return False
    qvec = _cross(tvec, e1)
    v = F32(_dot(d, qvec) * inv)
    if v < 0 or F32(u + v) > 1:
        return False
    t = F32(_dot(e2, qvec) * inv)
    return not (t > 1 or t < 0)


def first_ray(Q, T):
    """Which ray gives isect_points its first point (mmi::isect_first_ray): 0-2 query edge i against T, 3-5 T's edge i
    against the query, -1 none.  Q, T (3, 3) float32."""
    Q = [[F32(x) for x in r] for r in np.asarray(Q, F32)]
    T = [[F32(x) for x in r] for r in np.asarray(T, F32)]
    for i in range(3):
        if _ray_hits(Q[i], _sub(Q[(i + 1) % 3], Q[i]), T[0], T[1], T[2]):
            return i
    for i in range(3):
        if _ray_hits(T[i], _sub(T[(i + 1) % 3], T[i]), Q[0], Q[1], Q[2]):
            return 3 + i
    return -1


def point_adjoint(T, Q, ray, h, g):
    """(d (3, 3) corner adjoints, d_h) of one hull point for the upstream vector g, float64."""
    T, Q, g = np.asarray(T, np.float64), np.asarray(Q, np.float64), np.asarray(g, np.float64)
    d = np.zeros((3, 3))
    if ray >= 3:
        i = ray - 3
        j = (i + 1) % 3
        e = T[j] - T[i]
        D = e[1]
        s = (h - T[i][1]) / D
        q = g @ e / D
        d[i] = (1 - s) * g
        d[i, 1] += q * (s - 1)
        d[j] = s * g
        d[j, 1] -= q * s
        return d, q
    if ray < 0:
        return d, 0.0
    o, w = Q[ray].copy(), Q[(ray + 1) % 3] - Q[ray]
    o[1] = h
    e1, e2 = T[1] - T[0], T[2] - T[0]
    n = np.cross(e1, e2)
    s = n @ (T[0] - o) / (n @ w)
    r = T[0] - (o + s * w)
    c = g @ w / (n @ w)
    d[1] = c * np.cross(e2, r)
    d[2] = c * np.cross(r, e1)
    d[0] = c * n - d[1] - d[2]
    return d, g[1] - c * n[1]


def plane_terms(tris, face_idx, bc, max_collisions=4096):
    """The kernel's hull of one plane with each vertex's (face, query half, ray) and its upstream vector
    u_in - u_out (float64): (h float32, [(face, q, ray, g)] in hull order)."""
    bc = np.asarray(bc, F32)
    pts, f, _, cyc = measure_grad_oracle.hull_cycle(tris, face_idx, bc, max_collisions)
    h = F32((tris[face_idx] * bc.reshape(3, 1)).sum(axis=0, dtype=F32)[1])
    # the query half of each point, as hull_cycle derives its codes
    faces, _ = mo.mesh_to_mesh_forward(mo.plane_quad(h)[None], tris[None], max_collisions)
    valid = np.where(faces[0] > 0)[0]
    half = valid // max_collisions
    P = pts.astype(np.float64)
    m = len(cyc)
    out = []
    for j in range(m):
        cur, prev, nxt = cyc[j], cyc[(j - 1) % m], cyc[(j + 1) % m]
        ui = (P[cur] - P[prev]) / np.linalg.norm(P[cur] - P[prev])
        uo = (P[nxt] - P[cur]) / np.linalg.norm(P[nxt] - P[cur])
        Q = mo.plane_quad(h)[half[cur]]
        out.append((int(f[cur]), int(half[cur]), first_ray(Q, tris[f[cur]]), ui - uo))
    return h, out


def exact_grad(v_shaped, faces, grad_out, lm=None):
    """Gradient of (mass, height, chest, waist, hips) . grad_out with respect to v_shaped (V, 3), float64, with the
    exact circumference derivative (mass and height as measure_grad_oracle)."""
    lm = lm or mo.load_landmarks()
    g = np.asarray(grad_out, np.float64)
    v_shaped = np.asarray(v_shaped, F32)
    out = measure_grad_oracle.measure_grad(v_shaped, faces, np.concatenate([g[:2], np.zeros(3)]), lm)
    tris = np.ascontiguousarray(v_shaped[faces])
    for i, name in enumerate(PLANES):
        if g[2 + i] == 0:
            continue
        h, terms = plane_terms(tris, lm[name]['face_idx'], lm[name]['bc'])
        gh = 0.0
        for f, q, ray, gv in terms:
            d, dh = point_adjoint(tris[f], mo.plane_quad(h)[q], ray, float(h), g[2 + i] * gv)
            for k in range(3):
                out[faces[f, k]] += d[k]
            gh += dh
        fl = lm[name]['face_idx']
        for k in range(3):
            out[faces[fl, k], 1] += gh * float(np.float32(lm[name]['bc'][k]))
    return out


def jacobian_betas(v, faces, S, lm=None):
    """(5, NB) float64 Jacobian of (mass, height, chest, waist, hips) with respect to betas at the vertices v (V, 3),
    S the shape basis (V, 3, NB), with the exact circumference derivative."""
    S = np.asarray(S, np.float64)
    return np.stack([np.einsum('vc,vcl->l', exact_grad(v, faces, np.eye(5)[k], lm), S) for k in range(5)])


def line_points_on_hull(v_shaped, faces, lm=None):
    """Number of hull vertices, over the three planes, that are line points (ray 0-2)."""
    lm = lm or mo.load_landmarks()
    tris = np.ascontiguousarray(np.asarray(v_shaped, F32)[faces])
    return sum(sum(1 for t in plane_terms(tris, lm[n]['face_idx'], lm[n]['bc'])[1] if 0 <= t[2] < 3) for n in PLANES)


def circumference_f64(v, faces, face_idx, bc, max_collisions=4096):
    """The float64 forward of one circumference: mmi_oracle_f64's points on the plane at the landmark's float64
    height, the hull's vertices chosen on their float32 copies (oracle/hull_exact), the 3-D edge lengths summed in
    float64."""
    from oracle import hull_exact, mmi_oracle_f64
    tris = np.asarray(v, np.float64)[faces]
    h = float(tris[face_idx, :, 1] @ np.asarray(bc, np.float64))
    q = np.array([[[-1, h, -1], [1, h, -1], [1, h, 1]], [[-1, h, -1], [1, h, 1], [-1, h, 1]]], np.float64)
    fi, bcs = mmi_oracle_f64.mesh_to_mesh_forward(q[None], tris[None], max_collisions)
    valid = np.where(fi[0] > 0)[0]
    pts = (tris[fi[0][valid]] * bcs[0][valid, 0][..., None]).sum(-2)
    idx = hull_exact.hull_indices(pts.astype(F32))
    p = pts[idx]
    return float(np.linalg.norm(np.roll(p, -1, 0) - p, axis=1).sum())
