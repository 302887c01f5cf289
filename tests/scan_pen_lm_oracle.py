"""TEST INFRASTRUCTURE ONLY -- float64 restatement of the self-penetration rows of the scan LM step
(shapy_fit_lm_scan_penetration_step), building on tests/scan_lm_oracle.py.

pen_rows: the chunk partial sums of one body's penetration rows, in the layout of scan_lm_oracle.rows: each of a
pair's six points (k < 3: vertex k of the intruder in the receiver's cone, k >= 3: vertex k - 3 of the receiver in the
intruder's cone) with phi != 0 is one row, weight w, residual phi, Jacobian sum over the point and the cone's three
vertices of (d phi / d x)^T J_x (tests/penetration_oracle.point_phi_grad).
lm_scan_pen_step: scan_lm_oracle.lm_scan_step with those chunks added, unscaled, to the data rows and the trial loss.
"""
import numpy as np

import penetration_oracle as po
import scan_lm_oracle as so


def pen_rows(verts, jac, faces, pairs, weight, sigma, P):
    verts, jac = np.asarray(verts, np.float32), np.asarray(jac, np.float32)
    faces, pairs = np.asarray(faces, np.int64), np.asarray(pairs, np.int64)
    F, w = faces.shape[0], float(np.float32(weight))
    sg = float(np.float32(sigma))

    def point(i):
        fr, fi = pairs[i // 6]
        if fr < 0 or fr >= F or fi < 0 or fi >= F:
            return 0.0, []
        k = i % 6
        cone, pv = (faces[fr], faces[fi][k]) if k < 3 else (faces[fi], faces[fr][k - 3])
        phi, g = po.point_phi_grad(verts[pv], verts[cone], sg)
        if phi == 0.0:
            return 0.0, []
        vs = [pv] + list(cone)
        j = sum(g[m] @ jac[int(vs[m])].astype(np.float64) for m in range(4))
        return w * (phi * phi), [(w, phi, j)]

    out = []
    n = 6 * pairs.shape[0]
    for c0 in range(0, n, so.CHUNK):
        A, gv, L = np.zeros((P, P)), np.zeros(P), 0.0
        for ls, rws in (point(i) for i in range(c0, min(n, c0 + so.CHUNK))):
            L += ls
            for u, r, j in rws:
                uj = u * j
                A += np.outer(uj, j)
                gv += uj * r
        out.append((np.tril(A), gv, L))
    return out


def lm_scan_pen_step(state, trial, chunks, ns, pen_chunks, weights, V, s2m, m2s, lambda_up, lambda_down, first,
                     **kw):
    """scan_lm_oracle.lm_scan_step with the penetration chunks: they enter the point group scaled by 1 / c_s, so that
    c_s (As + Ap / c_s) = c_s As + Ap (equal up to rounding, the step adds them after the scan terms); s2m > 0."""
    W = so.weight_sum(weights)
    cs = float(np.float32(s2m)) / (W if W > 0.0 else 1.0)
    scaled = [(A / cs, g / cs, L / cs) for A, g, L in pen_chunks]
    return so.lm_scan_step(state, trial, chunks[:ns] + scaled + chunks[ns:], ns + len(scaled), weights, V, s2m, m2s,
                           lambda_up, lambda_down, first, **kw)
