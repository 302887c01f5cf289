"""CPU: tests/scan_lm_oracle.py pinned (its vertex Jacobian against central differences of the float64 forward, its g
against the gradient of the loss with the correspondences held, point-to-plane against point-to-point rows), and the
argument checks of fit_body_to_scan(method='lm')."""
import math

import numpy as np
import pytest
import torch

import lm_harness as H
import scan_lm_oracle as so
from oracle import smplx_oracle
from shapy_b200 import synth


def _model():
    return synth.make_smplx()


def _body(seed, nb):
    g = torch.Generator().manual_seed(seed)
    rot = H.rodrigues(torch.randn(22, 3, generator=g, dtype=torch.float64) * 0.3).numpy()
    return rot, (torch.randn(nb, generator=g) * 0.5).double().numpy(), (torch.randn(3, generator=g) * 0.1).double().numpy()


def _forward(model, rot, betas, transl):
    """(V, 3) float64 posed vertices of oracle/smplx_oracle.py plus transl."""
    J = model['J_regressor'].shape[0]
    full = torch.eye(3, dtype=torch.float64).repeat(1, J, 1, 1)
    full[0, :22] = torch.from_numpy(rot)
    out = smplx_oracle.smplx_forward_full(model, torch.from_numpy(betas)[None], full)
    return out['vertices'][0].numpy() + transl


def _at(model, rot, betas, transl, d):
    """The forward at the parameter offset d = [delta (66) | betas | transl]."""
    nb = len(betas)
    R = np.stack([rot[j] @ H.expm(d[3 * j:3 * j + 3]) for j in range(22)])
    return _forward(model, R, betas + d[66:66 + nb], transl + d[66 + nb:])


def test_vertex_jacobian_matches_central_differences():
    model = _model()
    nb = model['shapedirs'].shape[2]
    rot, betas, transl = _body(1, nb)
    x, jac = so.vertex_jacobian(model, betas, rot, transl)
    assert np.abs(x - _forward(model, rot, betas, transl)).max() < 1e-12
    P = jac.shape[2]
    idx = np.random.default_rng(0).choice(x.shape[0], 64, replace=False)
    h = 1e-6
    for col in list(range(0, 66, 5)) + list(range(66, P)):
        d = np.zeros(P)
        d[col] = h
        fd = (_at(model, rot, betas, transl, d) - _at(model, rot, betas, transl, -d))[idx] / (2 * h)
        assert np.abs(fd - jac[idx, :, col]).max() < 1e-6 * max(1.0, np.abs(jac[:, :, col]).max()), col


def _case(seed, N=300):
    """A body, its oracle vertices and Jacobian, scan points near its surface with held closest points on random
    faces (all interior: barycentrics > 0) and nearest points for every vertex."""
    model = _model()
    nb = model['shapedirs'].shape[2]
    rot, betas, transl = _body(seed, nb)
    x, jac = so.vertex_jacobian(model, betas, rot, transl)
    faces = model['faces_tensor'].numpy().astype(np.int64)
    rng = np.random.default_rng(seed)
    f = rng.integers(0, len(faces), N)
    b = rng.dirichlet([2.0, 2.0, 2.0], N)
    c = np.einsum('nk,nkc->nc', b, x[faces[f]])
    e1, e2 = x[faces[f, 1]] - x[faces[f, 0]], x[faces[f, 2]] - x[faces[f, 0]]
    n = np.cross(e1, e2)
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    pts = c + n * rng.normal(scale=0.01, size=(N, 1))
    w = rng.uniform(0.5, 1.5, N)
    nearest = rng.integers(0, N, x.shape[0])
    return model, rot, betas, transl, x, jac, faces, f, b, pts, w, nearest


@pytest.mark.parametrize('sigma', [math.inf, 0.02])
def test_g_is_the_gradient_with_correspondences_held(sigma):
    model, rot, betas, transl, x, jac, faces, f, b, pts, w, nearest = _case(2)
    P = jac.shape[2]
    chunks = so.rows(x, jac, pts, w, faces, f, b, nearest, sigma, P)
    ns = 1
    W = so.weight_sum(w)
    g = sum(c[1] for c in chunks[:ns]) / W + sum(c[1] for c in chunks[ns:]) / x.shape[0]

    def loss(xv):
        c = np.einsum('nk,nkc->nc', b, xv[faces[f]])
        rho = lambda e: e if math.isinf(sigma) else sigma * sigma * e / (sigma * sigma + e)  # noqa: E731
        return (w * rho(((c - pts) ** 2).sum(1))).sum() / W + rho(((xv - pts[nearest]) ** 2).sum(1)).mean()
    h = 1e-6
    for col in list(range(0, 66, 7)) + list(range(66, P)):
        d = np.zeros(P)
        d[col] = h
        fd = (loss(_at(model, rot, betas, transl, d)) - loss(_at(model, rot, betas, transl, -d))) / (2 * h)
        assert abs(2 * g[col] - fd) < 1e-6 * max(1.0, abs(fd)), col     # g = J^T W r is half the gradient


def test_point_to_plane_and_point_to_point_g_agree_in_the_interior():
    """A point exactly on its face's normal line: the plane row's g equals the three point-to-point rows' g; only A
    differs (the body may slide along the surface)."""
    model, rot, betas, transl, x, jac, faces, f, b, pts, w, _ = _case(3)
    P = jac.shape[2]
    plane = so.rows(x, jac, pts, w, faces, f, b, None, math.inf, P)[0]
    x32, j32 = x.astype(np.float32).astype(np.float64), jac.astype(np.float32).astype(np.float64)   # the rows' inputs
    g_pp, L = np.zeros(P), 0.0
    for i in range(len(w)):
        r = sum(b[i, k] * x32[faces[f[i], k]] for k in range(3)) - pts[i]
        g_pp += w[i] * (sum(b[i, k] * j32[faces[f[i], k]] for k in range(3)).T @ r)
        L += w[i] * (r @ r)
    # the plane rows drop the tangential part of c - p, which is zero up to the fp32 rounding of the vertices
    assert np.abs(plane[1] - g_pp).max() < 1e-5 * np.abs(g_pp).max()
    assert abs(plane[2] - L) < 1e-12 * L
    A_pp = np.zeros((P, P))
    for i in range(len(w)):
        Jm = sum(b[i, k] * j32[faces[f[i], k]] for k in range(3))
        A_pp += w[i] * np.tril(Jm.T @ Jm)
    assert np.abs(plane[0] - A_pp).max() > 1e-3 * np.abs(A_pp).max()       # only the Gauss-Newton matrix differs


def test_method_lm_argument_checks():
    from shapy_b200.fit import fit_body_to_scan

    class _Model:                      # what the checks read before anything reaches the device
        num_betas = 40
        faces_tensor = torch.zeros(10, 3, dtype=torch.long)
        shapedirs = torch.zeros(1)
    with pytest.raises(ValueError, match='method'):
        fit_body_to_scan(_Model(), torch.zeros(1, 4, 3), method='bfgs')
    with pytest.raises(ValueError, match='at most 96'):
        fit_body_to_scan(_Model(), torch.zeros(1, 4, 3), method='lm')
    m = _Model()
    m.num_betas = 10
    with pytest.raises(ValueError, match='robust_sigma'):
        fit_body_to_scan(m, torch.zeros(1, 4, 3), method='lm', robust_sigma=-1.0)
    with pytest.raises(ValueError, match='weights'):
        fit_body_to_scan(m, torch.zeros(1, 4, 3), method='lm', scan_to_model_weight=0.0, model_to_scan_weight=0.0)
