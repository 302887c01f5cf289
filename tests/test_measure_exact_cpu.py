"""CPU: the float64 restatement of the exact circumference derivative (tests/measure_exact_oracle.py) is the derivative
of the measured circumference: against central differences of the float64 forward on seeded synthetic bodies, against
the closed form on a regular n-gon frustum, and under a translation of the whole body.  Plus the argument checks of
the `circumference_derivative` option, which need no GPU."""
import math

import numpy as np
import pytest
import torch

import measure_exact_oracle as meo
import measure_slices as ms
from oracle import lm_oracle
from shapy_b200 import synth

SEEDS = range(9, 17)


@pytest.fixture(scope='module')
def model():
    d = synth.make_smplx()
    return (d['v_template'].double().numpy(), d['shapedirs'].double().numpy(), d['faces_tensor'].numpy(),
            synth.load_landmarks())


def _body(model, seed):
    vt, S, _, _ = model
    beta = (torch.randn(10, generator=torch.Generator().manual_seed(seed)) * 0.5).double().numpy()
    return beta, (vt + S @ beta).astype(np.float32)


@pytest.mark.parametrize('seed', SEEDS)
def test_exact_rows_vs_central_differences(model, seed):
    """Each circumference row within 2 % relative L2 of central differences at step 1e-4 in beta (measured: <= 1e-5);
    the reference rows on the same body are far from it, and the mass and height rows are the reference's."""
    vt, S, faces, lm = model
    beta, v = _body(model, seed)
    J = meo.jacobian_betas(v, faces, S, lm)
    ref = lm_oracle.jacobian_betas(v, faces, S, lm)
    assert np.array_equal(J[:2], ref[:2])
    worst_ref = 0.0
    for k, name in enumerate(meo.PLANES):
        def circ(b):
            return meo.circumference_f64(vt + S @ b, faces, lm[name]['face_idx'], lm[name]['bc'])
        fd = np.array([(circ(beta + 1e-4 * e) - circ(beta - 1e-4 * e)) / 2e-4 for e in np.eye(10)])
        err = np.linalg.norm(J[2 + k] - fd) / np.linalg.norm(fd)
        assert err <= 2e-2, (seed, name, err)
        worst_ref = max(worst_ref, np.linalg.norm(ref[2 + k] - fd) / np.linalg.norm(fd))
    assert worst_ref > 0.1, worst_ref


def _frustum(n=12, r0=0.5, slope=0.2, bc=(0.2, 0.3, 0.5)):
    """A regular n-gon frustum around the chest plane (y = 0), circumradius r0 + slope * y, no vertex on the quad's
    diagonal.  The chest landmark is the marker triangle at x = 5 (outside the quad), all of whose corners lie at
    y = 0, with barycentrics bc."""
    b = ms.Builder()
    b.lm['chest'] = dict(b.lm['chest'], bc=list(bc))
    ys = (-0.5, 0.5)
    ids = [[b.vert(((r0 + slope * y) * math.cos(0.1 + 2 * math.pi * i / n), y,
                    (r0 + slope * y) * math.sin(0.1 + 2 * math.pi * i / n))) for i in range(n)] for y in ys]
    lo, hi = ids
    for i in range(n):
        # each side triangle starts with a lateral edge, so every ring vertex of the slice is the first ray hit of the
        # triangles on both sides of it: the one whose side the quad's diagonal pierces takes that line point instead
        j = (i + 1) % n
        b.f.append((hi[j], lo[j], lo[i]))
        b.f.append((lo[i], hi[i], hi[j]))
    for i in range(1, n - 1):
        b.f.append((lo[0], lo[i], lo[i + 1]))
        b.f.append((hi[0], hi[i + 1], hi[i]))
    return b.mesh(family='frustum')


@pytest.mark.parametrize('n', [6, 12, 40])
def test_frustum_plane_gradient_closed_form(n):
    """The chest of a frustum is 2 n r(h) sin(pi / n): the exact gradient on the landmark's y components is
    bc_k 2 n r' sin(pi / n); the reference semantics give 0 there."""
    slope, bc = 0.2, (0.2, 0.3, 0.5)
    m = _frustum(n, slope=slope, bc=bc)
    go = np.eye(5)[2]
    g = meo.exact_grad(m.verts, m.faces, go, m.lm)
    fl = m.lm['chest']['face_idx']
    want = 2 * n * slope * math.sin(math.pi / n)
    for k in range(3):
        vid = m.faces[fl, k]
        assert abs(g[vid, 1] - bc[k] * want) <= 1e-5 * want, (n, k, g[vid], bc[k] * want)
        assert g[vid, 0] == 0 and g[vid, 2] == 0
    from oracle import measure_grad_oracle
    gr = measure_grad_oracle.measure_grad(m.verts, m.faces, go, m.lm)
    assert not gr[m.faces[fl]].any()


@pytest.mark.parametrize('seed', SEEDS[:4])
def test_translation_gives_zero_sum(model, seed):
    """Moving the whole body up or down moves its slicing planes with it and leaves every circumference unchanged: the
    y components of the exact gradient sum to zero.  Where no hull vertex is a line point (the quad's diagonal
    piercing a face, which stays put in x and z), the x and z components do too."""
    _, _, faces, lm = model
    _, v = _body(model, seed)
    line = meo.line_points_on_hull(v, faces, lm)
    for i in range(3):
        g = meo.exact_grad(v, faces, np.eye(5)[2 + i], lm)
        s, scale = g.sum(0), np.abs(g).sum(0)
        assert abs(s[1]) <= 1e-9 * scale[1], (seed, i, s, scale)
        if line == 0:
            assert (np.abs(s[[0, 2]]) <= 1e-9 * scale[[0, 2]]).all(), (seed, i, s, scale)


def test_unknown_circumference_derivative_raises():
    from shapy_b200.body_measurements import BodyMeasurements, exact_circumferences
    from shapy_b200.fit import fit_betas_to_measurements, fit_body_to_keypoints, main
    assert exact_circumferences('exact') and not exact_circumferences('reference')
    with pytest.raises(ValueError):
        exact_circumferences('finite-difference')
    bm = BodyMeasurements({'landmarks': synth.load_landmarks()})
    with pytest.raises(ValueError):
        bm.forward_vertices(torch.zeros(1, 3, 3), torch.zeros(1, 3, dtype=torch.int32), circumference_derivative='x')
    with pytest.raises(ValueError):
        bm.forward(torch.zeros(1, 1, 3, 3), circumference_derivative=True)
    with pytest.raises(ValueError):
        fit_betas_to_measurements(None, None, {'height': 1.8}, circumference_derivative='Exact')
    with pytest.raises(ValueError):
        fit_body_to_keypoints(None, None, circumference_derivative=None)
    with pytest.raises(SystemExit):
        main(['--synthetic', '--circumference-derivative', 'fd'])
