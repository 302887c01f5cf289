"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the gradient of BodyMeasurements under the reference's autograd.

  compute_mass / compute_height / compute_peripheries backward
      mesh-mesh-intersection/body_measurements/body_measurements.py:137-215 (float32 autograd arithmetic restated)
  point selection: oracle/mmi_oracle.c through oracle/measure_oracle.py; hull: scipy.spatial.ConvexHull (qhull)

Pinned against the reference's own autograd gradients (tests/golden/ref_measure_grad.npz, written by
tools/make_golden.py through oracle/ref_body_measurements.py) in tests/test_measure_grad_cpu.py.
"""
import numpy as np

from oracle import measure_oracle as mo
def _ord_bits(f):
    i = int(np.float32(f).view(np.int32))
    return i if i >= 0 else i ^ 0x7fffffff


def hull_cycle(tris: np.ndarray, face_idx: int, bc, max_collisions=4096):
    """The hull of one slicing plane as the kernels walk it: (points (n,3) float32, faces (n,), bcs (n,3), cycle) with
    `cycle` the hull vertices in order (scipy's qhull on the xz coordinates).  Among points that share (x, z) the
    representative is the first in (y, z, x) bit order, then by (face, query half), as in csrc/measure.cu."""
    from scipy.spatial import ConvexHull
    bc = np.asarray(bc, np.float32)
    vertex = (tris[face_idx] * bc.reshape(3, 1)).sum(axis=0, dtype=np.float32)
    q = mo.plane_quad(np.float32(vertex[1]))
    faces, bcs = mo.mesh_to_mesh_forward(q[None], tris[None], max_collisions)
    faces, bcs = faces[0], bcs[0]
    valid = np.where(faces > 0)[0]
    f = faces[valid]
    b1 = bcs[valid, 0]                                   # the two points of a collision coincide (mmi_oracle.c)
    code = (f << 1) | (valid // max_collisions)
    pts = (tris[f] * b1[..., None]).sum(axis=-2, dtype=np.float32)
    # qhull on the reference's point list, where every point appears twice (body_measurements.py:162-165): its
    # choice of vertices near a straight hull edge depends on the input, not only on the point set
    hull = ConvexHull(np.repeat(pts[:, [0, 2]], 2, axis=0))
    cyc = []
    for h in hull.vertices // 2:
        same = np.where((pts[:, 0] == pts[h, 0]) & (pts[:, 2] == pts[h, 2]))[0]
        key = [(_ord_bits(pts[i, 1]), _ord_bits(pts[i, 2]), _ord_bits(pts[i, 0]), int(code[i])) for i in same]
        cyc.append(int(same[min(range(len(same)), key=key.__getitem__)]))
    return pts, f, b1, cyc


def measure_grad(v_shaped: np.ndarray, faces: np.ndarray, grad_out, lm=None) -> np.ndarray:
    """Gradient of (mass, height, chest, waist, hips) . grad_out with respect to v_shaped (V,3), float64, with the
    reference's autograd semantics (body_measurements.py:137-215): the intersection barycentrics are constants (chosen
    under no_grad), the plane height gets none, sign(0) = 0.  Each hull edge p_i -> p_j of length L adds
    -g (p_j - p_i) / L to p_i and +g (p_j - p_i) / L to p_j, spread to the face's vertices by the point's bc."""
    lm = lm or mo.load_landmarks()
    g = np.asarray(grad_out, np.float64)
    tris = np.ascontiguousarray(v_shaped[faces].astype(np.float32))
    out = np.zeros((v_shaped.shape[0], 3), np.float64)
    t64 = tris.astype(np.float64)
    if g[0] != 0:
        # autograd of compute_mass in float32: out = (|sum_f vol_f| / 6) * 985; each coordinate appears in two of the
        # six products (s x_a y_b) z_c of vol_f, so its two float32 terms add exactly in either order
        x, y, z = tris[..., 0], tris[..., 1], tris[..., 2]
        vol = (-x[:, 2] * y[:, 1] * z[:, 0] + x[:, 1] * y[:, 2] * z[:, 0] + x[:, 2] * y[:, 0] * z[:, 1]
               - x[:, 0] * y[:, 2] * z[:, 1] - x[:, 1] * y[:, 0] * z[:, 2] + x[:, 0] * y[:, 1] * z[:, 2])
        gs = np.float32(np.float32(np.float32(g[0]) * np.float32(mo.DENSITY)) / np.float32(6.0))
        gs = gs * np.float32(np.sign(vol.sum(dtype=np.float32)))
        gt = np.zeros(tris.shape, np.float32)
        for sg, a, b, c in ((-1, 2, 1, 0), (1, 1, 2, 0), (1, 2, 0, 1), (-1, 0, 2, 1), (-1, 1, 0, 2), (1, 0, 1, 2)):
            gz = gs * z[:, c]
            gt[:, a, 0] += sg * (gz * y[:, b])
            gt[:, b, 1] += sg * (gz * x[:, a])
            gt[:, c, 2] += sg * (gs * (x[:, a] * y[:, b]))
        for k in range(3):
            np.add.at(out, faces[:, k], gt[:, k].astype(np.float64))
    if g[1] != 0:
        def land(name):
            return (tris[lm[name]['face_idx']] * np.asarray(lm[name]['bc'], np.float32).reshape(3, 1)).sum(0)
        s = g[1] * np.sign(np.float32(land('head_top')[1]) - np.float32(land('left_heel')[1]))
        for name, sg in (('head_top', 1.0), ('left_heel', -1.0)):
            fi = lm[name]['face_idx']
            for k in range(3):
                out[faces[fi, k], 1] += sg * s * lm[name]['bc'][k]
    for i, name in enumerate(('chest', 'waist', 'hips')):
        if g[2 + i] == 0:
            continue
        pts, f, b1, cyc = hull_cycle(tris, lm[name]['face_idx'], lm[name]['bc'])
        m = len(cyc)
        gi = np.float32(g[2 + i])
        for j in range(m):
            # autograd of (p_b - p_a).pow(2).sum().sqrt() in float32: g / (2 r) * (2 d)
            a, b = cyc[j], cyc[(j + 1) % m]
            d = pts[b] - pts[a]
            r = np.sqrt(np.float32(d[0] * d[0] + d[1] * d[1]) + np.float32(d[2] * d[2]))
            gd = (gi / (np.float32(2.0) * r)) * (np.float32(2.0) * d)
            for pnt, sg in ((a, -1.0), (b, 1.0)):
                for k in range(3):
                    out[faces[f[pnt], k]] += sg * (gd * b1[pnt, k]).astype(np.float64)
    return out
