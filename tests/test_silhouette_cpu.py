"""CPU: tests/silhouette_oracle.py pinned on hand-computed cases (a single triangle, a square mask, masks touching each
border) and against brute force and central differences."""
import numpy as np

import silhouette_oracle as so


def test_single_triangle_raster_and_closest_points():
    # f = 1, pp = 0, depth 1: (u, v) = (X, Y).  Inside: c, r >= 1 and c + r <= 4; the centres with c + r = 5 lie on the
    # hypotenuse x + y = 5
    Y = np.array([[0.5, 0.5, 1.0], [4.5, 0.5, 1.0], [0.5, 4.5, 1.0]], np.float32)
    mask, amb = so.rasterise(Y, [[0, 1, 2]], (1.0, 0.0, 0.0), 6, 6)
    assert sorted(map(tuple, np.argwhere(mask))) == [(1, 1), (1, 2), (1, 3), (2, 1), (2, 2), (3, 1)]
    assert sorted(map(tuple, np.argwhere(amb))) == [(1, 4), (2, 3), (3, 2), (4, 1)]
    # the same triangle behind the camera is not drawn
    mask, amb = so.rasterise(Y * np.float32([1, 1, -1]), [[0, 1, 2]], (1.0, 0.0, 0.0), 6, 6)
    assert not mask.any() and not amb.any()
    d2, _ = so.closest_2d([[0.0, 0.0], [3.0, 3.0], [2.0, 2.0], [6.5, 0.5]], Y[None, :, :2])
    np.testing.assert_allclose(d2, [0.5, 0.5, 0.0, 4.0], rtol=0, atol=1e-12)


def test_square_mask():
    m = np.zeros((5, 5), np.uint8)
    m[1:4, 1:4] = 1
    d2 = so.edt_sq(m)
    assert d2[0, 0] == 2 and d2[0, 2] == 1 and d2[2, 2] == 0 and d2[4, 4] == 2 and d2[2, 0] == 1
    assert (so.dist_f32(m) == np.sqrt(d2.astype(np.float32))).all()
    ring = [(1, 1), (1, 2), (1, 3), (2, 1), (2, 3), (3, 1), (3, 2), (3, 3)]
    assert list(map(tuple, so.contour_pixels(m))) == ring
    pts, w, n = so.kept_contour(m, 3)               # k = ceil(8 / 3) = 3: ranks 0, 3, 6
    assert n == 8 and w.tolist() == [1, 1, 1]
    assert pts.tolist() == [[1, 1, 0], [1, 2, 0], [2, 3, 0]]        # (c, r, 0)
    pts, w, n = so.kept_contour(m, 10)
    assert w.tolist() == [1] * 8 + [0, 0] and (pts[8:] == 0).all()


def test_masks_touching_each_border():
    full = np.ones((4, 6), np.uint8)
    assert len(so.contour_pixels(full)) == 0 and (so.edt_sq(full) == 0).all()
    top = np.zeros((4, 6), np.uint8)
    top[:2] = 1                                     # row 0 touches the top border: only row 1 is contour
    assert list(map(tuple, so.contour_pixels(top))) == [(1, c) for c in range(6)]
    assert (so.edt_sq(top)[3] == 4).all()
    for flip in (lambda a: a[::-1], lambda a: a.T, lambda a: a.T[::-1]):   # bottom, left, right
        m = np.ascontiguousarray(flip(top))
        rc = so.contour_pixels(m)
        assert len(rc) == 6 and len(np.unique(rc[:, 0 if m.shape[0] == 6 else 1])) == 6
    empty = np.zeros((3, 3), np.uint8)
    assert (so.edt_sq(empty) == 0).all() and len(so.contour_pixels(empty)) == 0
    one = np.ones((1, 1), np.uint8)
    assert list(map(tuple, so.contour_pixels(one))) == [] and so.edt_sq(one)[0, 0] == 0


def test_edt_against_brute_force():
    rng = np.random.default_rng(0)
    m = (rng.random((23, 31)) < 0.05).astype(np.uint8)
    person = np.argwhere(m)
    rr, cc = np.mgrid[:23, :31]
    brute = ((rr[..., None] - person[:, 0]) ** 2 + (cc[..., None] - person[:, 1]) ** 2).min(-1)
    assert (so.edt_sq(m) == brute).all()


def test_bilinear_and_clamping():
    d = np.array([[0.0, 1.0], [2.0, 4.0]])
    D, du, dv = so.bilinear(d, np.array([0.5, -3.0, 0.25]), np.array([0.5, 0.5, 7.0]))
    np.testing.assert_allclose(D, [1.75, 1.0, 2.5])
    np.testing.assert_allclose(du, [1.5, 0.0, 2.0])              # clamped in u: no u derivative
    np.testing.assert_allclose(dv, [2.5, 2.0, 0.0])


def test_gradient_matches_central_differences():
    rng = np.random.default_rng(1)
    m = np.zeros((60, 50), np.uint8)
    m[15:45, 18:33] = 1
    dist = so.dist_f32(m).astype(np.float64)
    intr = (100.0, 25.0, 30.0)
    Y = np.stack([rng.uniform(-0.4, 0.4, 40), rng.uniform(-0.4, 0.4, 40), rng.uniform(1.5, 2.5, 40)], 1)
    Y[0, 0] = 5.0                                   # projected far outside the image: no u gradient
    g = so.gradient(Y, intr, dist, 1.0)
    assert g[0, 0] == 0.0
    checked = 0
    for _ in range(5):
        dirn = rng.standard_normal(Y.shape)
        h = 1e-6
        a, b = Y + h * dirn, Y - h * dirn
        if not (so.cell_of(dist.shape, *so.project_f32(a, intr).T) ==
                so.cell_of(dist.shape, *so.project_f32(b, intr).T)).all():
            continue
        fd = (so.model_to_mask_f64(a, intr, dist) - so.model_to_mask_f64(b, intr, dist)) / (2 * h)
        np.testing.assert_allclose((g * dirn).sum(), fd, rtol=1e-4, atol=1e-6)
        checked += 1
    assert checked >= 3
