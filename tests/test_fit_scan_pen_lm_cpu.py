"""CPU: the self-penetration rows of the scan LM step (tests/scan_pen_lm_oracle.py) against central differences: each
row's residual is phi of its point and its Jacobian the derivative of phi through the vertices' Jacobian."""
import numpy as np
import pytest

import penetration_oracle as po
import scan_pen_lm_oracle as spo


def _case(seed, C=6):
    rng = np.random.default_rng(seed)
    F = 2 * C
    tris = rng.normal(size=(F, 1, 3)) * 0.01 + rng.normal(size=(F, 3, 3)) * 0.02
    tris[C:] = tris[:C] + rng.normal(size=(C, 3, 3)) * 0.005     # each intruder near its receiver
    verts = tris.reshape(3 * F, 3).astype(np.float32)
    faces = po.soup_faces(F)
    pairs = np.stack([np.arange(C), np.arange(C, F)], 1)
    pairs[-1] = -1                                                 # a skipped row
    return verts, faces, pairs


@pytest.mark.parametrize('sigma', [0.02, 0.005])
def test_point_gradient_matches_central_differences(sigma):
    verts, faces, pairs = _case(1)
    h, checked = 1e-7, 0
    for fr, fi in pairs[:-1]:
        for pv, cone in [(faces[fi][k], faces[fr]) for k in range(3)] + [(faces[fr][k], faces[fi]) for k in range(3)]:
            x = verts.astype(np.float64)
            phi, g = po.point_phi_grad(x[pv], x[cone], sigma)
            if phi == 0.0:
                continue
            vs = [pv] + list(cone)
            fd = np.zeros((4, 3))
            for m in range(4):
                for q in range(3):
                    xp, xm = x.copy(), x.copy()
                    xp[vs[m], q] += h
                    xm[vs[m], q] -= h
                    fd[m, q] = (po.point_phi_grad(xp[pv], xp[cone], sigma)[0] -
                                po.point_phi_grad(xm[pv], xm[cone], sigma)[0]) / (2 * h)
            np.testing.assert_allclose(g, fd, rtol=1e-5, atol=1e-6 * np.abs(fd).max())
            checked += 1
    assert checked >= 6


def test_rows_match_central_differences_through_the_jacobian():
    verts, faces, pairs = _case(2)
    V, P = verts.shape[0], 7
    jac = (np.random.default_rng(3).normal(size=(V, 3, P)) * 0.01).astype(np.float32)
    sigma, w = 0.02, 0.5
    chunks = spo.pen_rows(verts, jac, faces, pairs, w, sigma, P)
    A, g, L = chunks[0]

    def total(theta):
        x = verts.astype(np.float64) + jac.astype(np.float64) @ theta
        loss = 0.0
        for fr, fi in pairs:
            if fr < 0:
                continue
            for pv, cone in [(faces[fi][k], faces[fr]) for k in range(3)] + [(faces[fr][k], faces[fi]) for k in range(3)]:
                loss += w * po.point_phi_grad(x[pv], x[cone], sigma)[0] ** 2
        return loss

    assert L > 0 and np.isclose(L, total(np.zeros(P)), rtol=1e-6)
    # the rows' gradient J^T W r is half the loss's gradient
    h = 1e-6
    fd = np.array([(total(h * e) - total(-h * e)) / (2 * h) for e in np.eye(P)])
    np.testing.assert_allclose(2 * g, fd, rtol=1e-4, atol=1e-7 * np.abs(fd).max())
    # and J^T W J is the Gauss-Newton part of its Hessian: symmetric positive semi-definite
    Af = A + np.tril(A, -1).T
    assert np.linalg.eigvalsh(Af).min() >= -1e-12 * np.abs(Af).max()
