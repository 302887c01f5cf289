"""CPU: the float64 scan oracle (tests/scan_oracle.py) pinned to analytic closest points in the seven Voronoi regions of
a triangle, on a degenerate triangle and on a tie, its gradient to central differences of the exact distance, and the
scan fit's argument checks, the --scan npz reading and the C entry points' limits, which all stop before a launch."""
import math

import numpy as np
import pytest
import torch

import scan_oracle as so

TRI = np.array([[[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]]])


@pytest.mark.parametrize('p, q, bary', [
    ((-1.0, -1.0, 0.5), (0, 0, 0), (1, 0, 0)),            # vertex a
    ((2.0, -0.5, 0.3), (1, 0, 0), (0, 1, 0)),             # vertex b
    ((-0.5, 2.0, -0.2), (0, 1, 0), (0, 0, 1)),            # vertex c
    ((0.5, -1.0, 0.2), (0.5, 0, 0), (0.5, 0.5, 0)),       # edge ab
    ((-1.0, 0.25, 0.0), (0, 0.25, 0), (0.75, 0, 0.25)),   # edge ac
    ((1.0, 1.0, 0.3), (0.5, 0.5, 0), (0, 0.5, 0.5)),      # edge bc
    ((0.2, 0.3, 0.7), (0.2, 0.3, 0), (0.5, 0.2, 0.3)),    # interior
])
def test_voronoi_regions(p, q, bary):
    d2, bc = so.closest_on_faces(np.array([p]), TRI)
    assert math.isclose(d2[0, 0], float(np.sum((np.array(p) - q) ** 2)), rel_tol=1e-14, abs_tol=1e-15)
    assert np.allclose(bc[0, 0], bary, rtol=0, atol=1e-14)
    assert np.allclose(bc[0, 0] @ TRI[0], q, rtol=0, atol=1e-14)


def test_degenerate_triangles():
    """A zero-area triangle is the nearest of its edges (ab, ac, bc; the first on a tie); a point triangle is its
    point."""
    line = np.array([[[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [2.0, 0.0, 0.0]]])
    d2, bc = so.closest_on_faces(np.array([[1.5, 1.0, 0.0]]), line)
    assert math.isclose(d2[0, 0], 1.0, rel_tol=1e-14)
    assert np.allclose(bc[0, 0], (0.25, 0.0, 0.75), atol=1e-14)       # ac and bc tie at (1.5, 0, 0): ac comes first
    pt = np.array([[[0.3, -0.2, 0.1]] * 3])
    d2, bc = so.closest_on_faces(np.array([[1.3, -0.2, 0.1]]), pt)
    assert math.isclose(d2[0, 0], 1.0, rel_tol=1e-14) and np.all(np.isfinite(bc))


def test_tie_goes_to_the_smaller_face_index():
    """Two triangles mirrored about z = 0: the origin is at distance 1 from both, and the first face wins in either
    order."""
    up = [[-1.0, -1.0, 1.0], [1.0, -1.0, 1.0], [0.0, 1.0, 1.0]]
    down = [[-1.0, -1.0, -1.0], [1.0, -1.0, -1.0], [0.0, 1.0, -1.0]]
    v = np.array(up + down)
    for faces in (np.array([[0, 1, 2], [3, 4, 5]]), np.array([[3, 4, 5], [0, 1, 2]])):
        face, bary, d2, second = so.closest_points(v, faces, np.zeros((1, 3)))
        assert face[0] == 0 and d2[0] == 1.0 and second[0] == 1.0


def _random_mesh(rng, n_faces=6):
    v = rng.normal(size=(8, 3))
    faces = np.array([rng.choice(8, 3, replace=False) for _ in range(n_faces)])
    return v, faces


def test_gradient_vs_central_differences():
    """scan_loss_grad at the exact correspondences is the gradient of the exact loss: the float64 closest point
    recomputed at every perturbed mesh, points kept away from region switches."""
    rng = np.random.default_rng(3)
    v, faces = _random_mesh(rng)
    pts = rng.normal(size=(40, 3)) * 1.5
    w = rng.uniform(0.5, 2.0, 40)
    w[5] = 0.0
    pts[5] = np.nan
    for sigma in (None, 0.5):
        def loss(x):
            f, b, _, _ = so.closest_points(x, faces, pts, w)
            return so.scan_loss(x, faces, pts, w, f, b, sigma)
        f, b, _, second = so.closest_points(v, faces, pts, w)
        g = so.scan_loss_grad(v, faces, pts, w, f, b, sigma)
        h = 1e-6
        fd = np.zeros_like(v)
        for i in range(v.shape[0]):
            for c in range(3):
                e = np.zeros_like(v)
                e[i, c] = h
                fd[i, c] = (loss(v + e) - loss(v - e)) / (2 * h)
        assert np.abs(g - fd).max() <= 1e-6 * np.abs(fd).max(), (g, fd)


def test_sq_dist_grad_is_the_sum_of_its_terms():
    rng = np.random.default_rng(4)
    v, faces = _random_mesh(rng)
    pts = rng.normal(size=(10, 3))
    f, b, _, _ = so.closest_points(v, faces, pts)
    g = rng.normal(size=10)
    f[3] = -1
    got = so.sq_dist_grad(v, faces, pts, f, b, g)
    want = np.zeros_like(v)
    for i in range(10):
        if f[i] < 0:
            continue
        q = b[i] @ v[faces[f[i]]]
        for c in range(3):
            want[faces[f[i], c]] += 2 * g[i] * (q - pts[i]) * b[i, c]
    assert np.allclose(got, want, rtol=1e-14, atol=1e-14)


def test_nearest_points_brute_force():
    rng = np.random.default_rng(5)
    q, p = rng.normal(size=(30, 3)), rng.normal(size=(50, 3))
    w = rng.uniform(-1, 1, 50)
    p[w <= 0] = np.nan
    idx, d2, _ = so.nearest_points(q, p, w)
    for i in range(30):
        e = [np.sum((q[i] - p[j]) ** 2) if w[j] > 0 else np.inf for j in range(50)]
        assert idx[i] == int(np.argmin(e)) and d2[i] == min(e)
    idx, d2, _ = so.nearest_points(q, p, np.zeros(50))
    assert (idx == -1).all() and (d2 == 0).all()
    # a tie: two points at the same distance, the smaller index wins
    idx, _, _ = so.nearest_points(np.zeros((1, 3)), np.array([[0, 0, 2.0], [1.0, 0, 0], [-1.0, 0, 0]]))
    assert idx[0] == 1


def test_sample_surface_is_on_the_mesh():
    rng = np.random.default_rng(6)
    v, faces = _random_mesh(rng)
    pts, f, b = so.sample_surface(v, faces, 100, rng)
    assert (b >= 0).all() and np.allclose(b.sum(1), 1.0)
    _, _, d2, _ = so.closest_points(v, faces, pts)
    assert d2.max() <= 1e-24


# ------------------------------------------------------------------------------ checks before any launch
@pytest.fixture(scope='module')
def cpu_model():
    from shapy_b200 import synth
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    return SMPLX(data_struct=synth.make_smplx())


@pytest.mark.parametrize('kw, match', [
    (dict(points=np.zeros((2, 10, 2))), 'points must be'),
    (dict(points=np.zeros((2, 0, 3))), 'points must be'),
    (dict(points=np.zeros((1, 32769, 3))), 'subsample'),
    (dict(weights=np.ones((2, 9))), 'weights must be'),
    (dict(weights=np.full(10, np.nan)), 'finite'),
    (dict(scan_to_model_weight=0.0, model_to_scan_weight=0.0), 'not both 0'),
    (dict(model_to_scan_weight=-1.0), 'scan-to-model'),
    (dict(robust_sigma=0.0), 'robust_sigma'),
    (dict(pose_prior_weight=-1.0), 'pose_prior_weight'),
    (dict(measurements={'height': 1.7}), 'body_measurements'),
    (dict(circumference_derivative='bogus'), 'bogus'),
])
def test_fit_argument_checks(cpu_model, kw, match):
    from shapy_b200.fit import fit_body_to_scan
    kw = dict(kw)
    points = kw.pop('points', np.zeros((2, 10, 3), np.float32))
    with pytest.raises(ValueError, match=match):
        fit_body_to_scan(cpu_model, points, **kw)


def test_cli_scan_npz(tmp_path):
    """--scan reads points (B, N, 3) or (N, 3) and per-point weights, and rejects a malformed file before the model is
    built."""
    from shapy_b200.fit import _load_scan, main
    p = str(tmp_path / 'one.npz')
    np.savez(p, points=np.zeros((100, 3)), weights=np.ones(100))
    pts, w = _load_scan(p)
    assert pts.shape == (1, 100, 3) and pts.dtype == np.float32 and w.shape == (1, 100)
    p = str(tmp_path / 'batch.npz')
    np.savez(p, points=np.zeros((2, 50, 3)))
    pts, w = _load_scan(p)
    assert pts.shape == (2, 50, 3) and w is None
    for name, arrays in (('none', dict(pts=np.zeros((5, 3)))), ('dims', dict(points=np.zeros((5, 2)))),
                         ('weights', dict(points=np.zeros((2, 5, 3)), weights=np.ones(5)))):
        p = str(tmp_path / f'{name}.npz')
        np.savez(p, **arrays)
        with pytest.raises(SystemExit):
            main(['--synthetic', '--scan', p, '--output', str(tmp_path / 'out.npz')])
    with pytest.raises(SystemExit):
        main(['--synthetic', '--scan', p, '--keypoints-2d', p])


def test_c_entry_limits_return_unsupported():
    """F or N past 32768 returns SHAPY_ERR_UNSUPPORTED before any launch or pointer is read; B = 0 or N = 0 is a
    no-op."""
    from shapy_b200 import _lib
    L = _lib.lib()
    unsupported = -3
    rc = L.shapy_closest_points(None, None, 1, 10, 32769, None, 10, None, 0, None, None, None, None, 0, None)
    assert rc == unsupported and b'32768' in L.shapy_last_error()
    assert L.shapy_closest_points(None, None, 1, 10, 20, None, 32769, None, 0, None, None, None, None, 0, None) == \
        unsupported
    assert L.shapy_nearest_points(None, 1, 10, None, 32769, None, None, None, None, 0, None) == unsupported
    assert L.shapy_closest_points_backward(None, None, None, None, 1, 10, 20, None, 32769, None, None, None, None,
                                           None) == unsupported
    assert L.shapy_closest_points(None, None, 0, 10, 20, None, 10, None, 0, None, None, None, None, 0, None) == 0
    assert L.shapy_closest_points(None, None, 3, 10, 20, None, 0, None, 0, None, None, None, None, 0, None) == 0
    assert L.shapy_nearest_points(None, 0, 10, None, 5, None, None, None, None, 0, None) == 0
    assert L.shapy_closest_points_backward(None, None, None, None, 0, 10, 20, None, 5, None, None, None, None,
                                           None) == 0


def test_ops_limits_raise_value_error():
    """The Python wrappers' limits are ValueErrors; on a CPU tensor they refuse to run (there is no CPU path)."""
    from shapy_b200 import ops
    with pytest.raises(RuntimeError, match='CUDA'):
        ops.closest_points(torch.zeros(1, 3, 3), torch.zeros(1, 3, dtype=torch.int32), torch.zeros(1, 4, 3))
