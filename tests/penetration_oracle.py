"""TEST INFRASTRUCTURE ONLY -- float64 NumPy restatement of the self-penetration term and a brute-force self-collision
oracle.

loss / loss_and_grad: the conical distance-field loss of the reference's DistanceFieldPenetrationLoss
(mesh-mesh-intersection/mesh_mesh_intersection/loss.py, vectorized=True) on vertices (B, V, 3), faces (F, 3) and
(receiver, intruder) rows (B, C, 2), rows with a first index < 0 skipped, with the analytic gradient of the kernel
(shapy_b200/csrc/penetration.cu) in float64.  Pinned against the reference's own loss.py by tests/golden/
ref_penetration.npz and against central differences (tests/test_penetration_cpu.py).

self_collisions: every pair (f, g), f < g, of faces that share no vertex, whose triangles' boxes overlap and that the
11-axis SAT finds intersecting, in (f, g) order, optionally without the ignored part-label pairs.  The predicates are
the plain-C restatement's (oracle/mmi_oracle.c), reached through its all-pairs mmi_oracle_forward with each face as a
query against the whole mesh (query first, as T_f is in the kernel), so they round like the device's.
"""
import numpy as np

from oracle import measure_oracle
from shapy_b200 import synth


def smooth_smplx():
    """The synthetic SMPL-X without its random pose correctives (posedirs, Gaussian per vertex), which crumple a posed
    mesh into hundreds of thousands of spurious intersections: linear blend skinning of the SMPL-X template.  Its
    meshes still intersect widely (the template alone has 8 254 pairs of faces that share no vertex and intersect,
    and a posed body tens of thousands, part-filtered), so they test detection at scale, not a realistic pair count."""
    d = synth.make_smplx()
    d['posedirs'] = d['posedirs'].zero_()
    return d


def _cone(t):
    """t (..., 3, 3) -> dict of the cone's float64 terms (loss.py calc_circumcircle and the unit normal)."""
    x0, x1, x2 = t[..., 0, :], t[..., 1, :], t[..., 2, :]
    N = np.cross(x1 - x0, x2 - x0)
    alpha, beta = x0 - x2, x1 - x2
    nN = np.linalg.norm(N, axis=-1)
    la, lb, lab = np.linalg.norm(alpha, axis=-1), np.linalg.norm(beta, axis=-1), np.linalg.norm(alpha - beta, axis=-1)
    r = lab / (2 * nN) * la * lb
    s = (alpha * alpha).sum(-1)[..., None] * beta - (beta * beta).sum(-1)[..., None] * alpha
    tt = np.cross(alpha, beta)
    y = np.cross(s, tt)
    k = 2 * (N * N).sum(-1)
    return dict(x=(x0, x1, x2), N=N, alpha=alpha, beta=beta, nN=nN, la=la, lb=lb, lab=lab, r=r, s=s, t=tt, y=y, k=k,
                c=y / k[..., None] + x2, n=N / nN[..., None])


def _psi(x, sigma, penalize_outside, linear_max):
    lin = (x <= -sigma) & (x > -linear_max)
    quad = (x > -sigma) & ((x < sigma) if penalize_outside else (x < 0))
    qa = -(1.0 - 2.0 * sigma) / (4.0 * sigma ** 2)
    psi = np.where(lin, -x + 1 - sigma, 0.0) + np.where(quad, qa * x ** 2 - x / (2.0 * sigma) + 0.25 * (3 - 2 * sigma),
                                                         0.0)
    dpsi = np.where(lin, -1.0, 0.0) + np.where(quad, 2 * qa * x - 1 / (2.0 * sigma), 0.0)
    return psi, dpsi


def _points(p, q, sigma, po, lmax):
    """Point terms of points p (n, 3) in cones q (n-batched dict)."""
    d = p - q['c']
    x = (d * q['n']).sum(-1)
    w = d - x[:, None] * q['n']
    m = np.linalg.norm(w, axis=-1)
    D = -q['r'] / sigma * x + q['r'] + 1e-6
    a = m / D
    psi, dpsi = _psi(x, sigma, po, lmax)
    u = (1 - a) * psi
    mask = (a < 1).astype(np.float64)
    phi1 = mask * u * u
    return dict(d=d, x=x, w=w, m=m, D=D, a=a, psi=psi, dpsi=dpsi, u=u, mask=mask, phi1=phi1, phi=phi1 * phi1)


def _rows(vertices, faces, pairs, F):
    b, c = np.nonzero(pairs[:, :, 0] >= 0)
    r, i = pairs[b, c, 0], pairs[b, c, 1]
    ok = (r < F) & (i >= 0) & (i < F)
    return b[ok], r[ok], i[ok]


def loss_and_grad(vertices, faces, pairs, sigma=0.5, penalize_outside=True, linear_max=1000.0, grad_loss=None):
    """float64 loss (B,) and, with grad_loss (B,) (ones when None), its gradient (B, V, 3)."""
    v = np.asarray(vertices, np.float64)
    faces = np.asarray(faces, np.int64)
    pairs = np.asarray(pairs, np.int64)
    B, V = v.shape[:2]
    g_l = np.ones(B) if grad_loss is None else np.asarray(grad_loss, np.float64)
    b, r, i = _rows(v, faces, pairs, faces.shape[0])
    loss = np.zeros(B)
    grad = np.zeros_like(v)
    if b.size == 0:
        return loss, grad
    tri_r, tri_i = v[b[:, None], faces[r]], v[b[:, None], faces[i]]
    cr, ci = _cone(tri_r), _cone(tri_i)
    for cone, pts, cone_v, pts_v in ((cr, tri_i, faces[r], faces[i]), (ci, tri_r, faces[i], faces[r])):
        gc, gn, gr = np.zeros_like(cone['c']), np.zeros_like(cone['n']), np.zeros_like(cone['r'])
        for k in range(3):
            e = _points(pts[:, k], cone, sigma, penalize_outside, linear_max)
            np.add.at(loss, b, e['phi'] ** 2)
            G = g_l[b] * 8 * e['phi'] * e['phi1'] * e['mask'] * e['u']
            G = np.where(G == 0, 0.0, G)
            ga = -e['psi'] * G
            gx = (1 - e['a']) * e['dpsi'] * G
            gm, gD = ga / e['D'], -ga * e['a'] / e['D']
            gr += gD * (1 - e['x'] / sigma)
            gx += gD * (-cone['r'] / sigma)
            with np.errstate(invalid='ignore', divide='ignore'):
                gw = np.where((e['m'] > 0)[:, None], (gm / e['m'])[:, None] * e['w'], 0.0)
            gx -= (gw * cone['n']).sum(-1)
            gn += -e['x'][:, None] * gw + gx[:, None] * e['d']
            gd = gw + gx[:, None] * cone['n']
            np.add.at(grad, (b, pts_v[:, k]), gd)
            gc -= gd
        gx3 = _cone_backward(cone, gc, gn, gr)
        for k in range(3):
            np.add.at(grad, (b, cone_v[:, k]), gx3[k])
    return loss, grad


def _cone_backward(q, gc, gn, gr):
    dot = lambda a, c: (a * c).sum(-1, keepdims=True)  # noqa: E731
    n, N = q['n'], q['N']
    gN = (gn - dot(n, gn) * n) / q['nN'][:, None]
    ab = q['alpha'] - q['beta']
    gr_ = (gr * q['r'])[:, None]
    gab = gr_ / (q['lab'] ** 2)[:, None] * ab
    galpha = gab + gr_ / (q['la'] ** 2)[:, None] * q['alpha']
    gbeta = -gab + gr_ / (q['lb'] ** 2)[:, None] * q['beta']
    gN = gN - gr_ / (q['nN'] ** 2)[:, None] * N
    gy = gc / q['k'][:, None]
    gk = -dot(gc, q['y']) / (q['k'] ** 2)[:, None]
    gN = gN + 4 * gk * N
    gs, gt = np.cross(q['t'], gy), np.cross(gy, q['s'])
    a, bt = q['alpha'], q['beta']
    gbeta = gbeta + dot(a, a) * gs - 2 * dot(a, gs) * bt
    galpha = galpha - dot(bt, bt) * gs + 2 * dot(bt, gs) * a
    galpha = galpha + np.cross(bt, gt)
    gbeta = gbeta + np.cross(gt, a)
    x0, x1, x2 = q['x']
    ge0, ge1 = np.cross(x2 - x0, gN), np.cross(gN, x1 - x0)
    return (-ge0 - ge1 + galpha, ge0 + gbeta, gc + ge1 - galpha - gbeta)


def point_phi_grad(p, tri, sigma, penalize_outside=True, linear_max=1000.0):
    """phi of point p (3,) in the cone of triangle tri (3, 3), float64, and its gradient (4, 3) with respect to p and
    the triangle's three vertices (the rows of the scan LM step's penetration term)."""
    p = np.asarray(p, np.float64)[None]
    q = _cone(np.asarray(tri, np.float64)[None])
    e = _points(p, q, sigma, penalize_outside, linear_max)
    G = 2 * e['phi1'] * e['mask'] * 2 * e['u']
    grad = np.zeros((4, 3))
    if float(G[0]) == 0.0:
        return float(e['phi'][0]), grad
    ga = -e['psi'] * G
    gx = (1 - e['a']) * e['dpsi'] * G
    gm, gD = ga / e['D'], -ga * e['a'] / e['D']
    gr = gD * (1 - e['x'] / sigma)
    gx = gx + gD * (-q['r'] / sigma)
    gw = (gm / e['m'])[:, None] * e['w'] if float(e['m'][0]) > 0 else np.zeros((1, 3))
    gx = gx - (gw * q['n']).sum(-1)
    gn = -e['x'][:, None] * gw + gx[:, None] * e['d']
    gd = gw + gx[:, None] * q['n']
    grad[0] = gd[0]
    for k, g in enumerate(_cone_backward(q, -gd, gn, gr)):
        grad[1 + k] = g[0]
    return float(e['phi'][0]), grad


def loss(vertices, faces, pairs, sigma=0.5, penalize_outside=True, linear_max=1000.0):
    return loss_and_grad(vertices, faces, pairs, sigma, penalize_outside, linear_max)[0]


def soup_faces(F):
    """The faces arange(3F).view(F, 3) under which triangles (B, F, 3, 3) are vertices (B, 3F, 3)."""
    return np.arange(3 * F, dtype=np.int64).reshape(F, 3)


def self_collisions(vertices, faces, part_labels=None, ignored_part_pairs=(), max_hits=256):
    """float32 vertices (V, 3) of one body -> int64 (n, 2) array of (f, g) rows in ascending order."""
    v = np.asarray(vertices, np.float32)
    faces = np.asarray(faces, np.int64)
    F = faces.shape[0]
    tris = np.ascontiguousarray(v[faces], np.float32)                  # (F, 3, 3)
    hit = np.full(F * max_hits, -1, np.int64)
    bcs = np.zeros((F * max_hits, 2, 3), np.float32)
    worst = measure_oracle.lib().mmi_oracle_forward(tris.ctypes.data, tris.ctypes.data, F, F, max_hits,
                                                    hit.ctypes.data, bcs.ctypes.data)
    assert worst <= max_hits, f'a face overlaps {worst} faces: raise max_hits'
    ignored = {(int(a), int(b)) for a, b in ignored_part_pairs} | {(int(b), int(a)) for a, b in ignored_part_pairs}
    hit = hit.reshape(F, max_hits)
    out = []
    for f in range(F):
        fv = set(faces[f].tolist())
        for g in hit[f]:
            if g <= f:                     # -1 padding, the face itself and the pairs counted from the lower face
                continue
            if fv & set(faces[g].tolist()):
                continue
            if part_labels is not None and (int(part_labels[f]), int(part_labels[g])) in ignored:
                continue
            out.append((f, int(g)))
    return np.array(sorted(out), np.int64).reshape(-1, 2)
