"""GPU: the exact circumference derivative of the measurement kernel (shapy_measure_backward_exact,
shapy_measure_backward_tris_exact, shapy_measure_jacobian_betas_exact) against its float64 restatement
(tests/measure_exact_oracle.py), the shape backward (J^T consistency), the triangle entry, the reference-mode launches
it must equal bit for bit where it is not about the circumferences, itself (determinism, batch independence) and the
NaN rules."""
import os

import numpy as np
import pytest
import torch

import measure_exact_oracle as meo
import measure_slices as ms
from shapy_b200 import synth

pytestmark = pytest.mark.gpu
NAMES = ('mass', 'height', 'chest', 'waist', 'hips')


def _bits(t):
    return t.contiguous().view(torch.int32)


def _generic(nb):
    d = dict(synth.make_smplx())
    d['shapedirs'] = torch.randn(d['shapedirs'].shape[0], 3, nb, generator=torch.Generator().manual_seed(nb)) * 0.01
    return d


def _setup(d, B, seed):
    from shapy_b200 import ops
    packed = ops.SmplxModel(dict(d), 'cuda')
    faces = d['faces_tensor'].to(torch.int32).cuda()
    betas = torch.randn(B, packed.NB, generator=torch.Generator().manual_seed(seed)).clamp(-2, 2).cuda()
    return ops, packed, faces, ops.make_landmarks(synth.load_landmarks()), ops.smplx_forward_shape(packed, betas)


def _grad(ops, lm, x, faces, go, exact=True, tris=False):
    go = torch.as_tensor(np.asarray(go, np.float32)).cuda()
    if tris:
        return ops.measure_backward(lm, go, triangles=x, exact=exact)
    return ops.measure_backward(lm, go, v_shaped=x, faces_i32=faces, exact=exact)


def _check_rows(J, ref, what):
    """Circumference rows within fp32-grade error of the float64 oracle, relative to each row's norm."""
    for k in range(2, 5):
        err = np.linalg.norm(J[k] - ref[k]) / np.linalg.norm(ref[k])
        assert err <= 1e-4, (what, NAMES[k], err, J[k], ref[k])


@pytest.mark.parametrize('nb', [10, 7])
@pytest.mark.parametrize('B', [1, 64, 4096])
def test_jacobian_vs_oracle_and_reference_mode(nb, B):
    d = synth.make_smplx() if nb == 10 else _generic(nb)
    ops, packed, faces, lm, v = _setup(d, B, seed=200 + B + nb)
    out, jac, status = ops.measure_jacobian_betas(packed, lm, v, faces, exact=True)
    out_r, jac_r, status_r = ops.measure_jacobian_betas(packed, lm, v, faces)
    # the measurements and the mass and height rows are the reference mode's, bit for bit
    assert torch.equal(_bits(out), _bits(out_r)) and int(status.item()) == int(status_r.item())
    assert torch.equal(_bits(jac[:, :2]), _bits(jac_r[:, :2]))
    assert torch.equal(torch.isnan(jac), torch.isnan(jac_r))
    S = d['shapedirs'].double().numpy()
    f_np = d['faces_tensor'].numpy()
    lmd = synth.load_landmarks()
    rows = range(B) if B == 1 else torch.randperm(B, generator=torch.Generator().manual_seed(B))[:6].tolist()
    J, vs = jac.double().cpu().numpy(), v.cpu().numpy()
    checked = 0
    for b in rows:
        if np.isnan(J[b]).any():
            continue
        _check_rows(J[b], meo.jacobian_betas(vs[b], f_np, S, lmd), (nb, B, b))
        checked += 1
    assert checked >= min(len(rows), 4)


def test_golden_bodies_gradient_vs_oracle(golden_dir):
    """The golden bodies through both gradient entries: one-hot circumference cotangents and a mixed one."""
    from shapy_b200 import ops
    g = np.load(os.path.join(golden_dir, 'img00_body.npz'))
    bodies = np.concatenate([g['v_shaped'][None], g['extra_v_shaped']], 0).astype(np.float32)
    faces_np, lmd = g['faces'], synth.load_landmarks()
    lm = ops.make_landmarks(lmd)
    v, f = torch.from_numpy(bodies).cuda(), torch.from_numpy(faces_np).cuda()
    tris = v[:, f.long()].contiguous()
    B, V = bodies.shape[:2]
    for go in [np.eye(5)[i] for i in (2, 3, 4)] + [np.array([0.3, -2.0, 1.5, 0.7, -1.1])]:
        gv = _grad(ops, lm, v, f, np.tile(go, (B, 1))).double().cpu().numpy()
        gt = _grad(ops, lm, tris, f, np.tile(go, (B, 1)), tris=True).double().cpu().numpy()
        for b in range(B):
            want = meo.exact_grad(bodies[b], faces_np, go, lmd)
            scat = np.zeros((V, 3))
            for k in range(3):
                np.add.at(scat, faces_np[:, k], gt[b, :, k])
            for got in (gv[b], scat):
                err = np.abs(got - want).max() / np.abs(want).max()
                assert err <= 2e-5, (list(go), b, err)


def test_transpose_consistency_and_triangle_entry():
    """Row k of the exact Jacobian is the shape backward of the exact gradient for the cotangent e_k; the triangle
    entry's gradient, scattered to the vertices, is the vertex entry's."""
    d = synth.make_smplx()
    ops, packed, faces, lm, v = _setup(d, 64, seed=5)
    _, jac, _ = ops.measure_jacobian_betas(packed, lm, v, faces, exact=True)
    S = d['shapedirs'].double().cuda()
    for k in range(5):
        go = torch.zeros(64, 5, device='cuda')
        go[:, k] = 1.0
        g = ops.measure_backward(lm, go, v_shaped=v, faces_i32=faces, exact=True)
        row = ops.smplx_backward_shape(packed, g)
        scale = torch.einsum('vcl,bvc->bl', S.abs(), g.double().abs())
        nan = torch.isnan(jac[:, k])
        assert torch.equal(nan, torch.isnan(row))
        err = (row.double() - jac[:, k].double()).abs()[~nan]
        assert (err <= 1e-5 * scale[~nan] + 1e-30).all(), (k, float((err / scale[~nan]).max()))
    go = torch.randn(64, 5, generator=torch.Generator().manual_seed(6)).cuda()
    gv = ops.measure_backward(lm, go, v_shaped=v, faces_i32=faces, exact=True)
    gt = ops.measure_backward(lm, go, triangles=v[:, faces.long()].contiguous(), exact=True)
    scat = torch.zeros_like(gv, dtype=torch.float64)
    for k in range(3):
        scat.index_add_(1, faces[:, k].long(), gt[:, :, k].double())
    fin = torch.isfinite(gv).all(2).all(1)
    assert fin.sum() >= 56
    # the two entries add the same fp32 terms in different orders (measured: <= 4e-6 of a body's largest entry)
    assert ((scat - gv.double()).abs()[fin].amax((1, 2)) <= 1e-5 * gv.abs()[fin].amax((1, 2))).all()


def test_mass_and_height_terms_equal_reference_mode():
    d = synth.make_smplx()
    ops, packed, faces, lm, v = _setup(d, 16, seed=7)
    go = np.zeros((16, 5), np.float32)
    go[:, :2] = np.random.default_rng(7).normal(size=(16, 2))
    tris = v[:, faces.long()].contiguous()
    for x, t in ((v, False), (tris, True)):
        a = _grad(ops, lm, x, faces, go, exact=True, tris=t)
        b = _grad(ops, lm, x, faces, go, exact=False, tris=t)
        assert torch.equal(_bits(a), _bits(b)), t


def test_deterministic_and_batch_independent():
    d = synth.make_smplx()
    ops, packed, faces, lm, v = _setup(d, 256, seed=9)
    go = torch.randn(256, 5, generator=torch.Generator().manual_seed(10)).numpy()
    tris = v[:, faces.long()].contiguous()
    for x, t in ((v, False), (tris, True)):
        a, b = _grad(ops, lm, x, faces, go, tris=t), _grad(ops, lm, x, faces, go, tris=t)
        assert torch.equal(_bits(a), _bits(b)), t
        one = _grad(ops, lm, x[100:101].contiguous(), faces, go[100:101], tris=t)
        assert torch.equal(_bits(one[0]), _bits(a[100])), t
    o1, j1, _ = ops.measure_jacobian_betas(packed, lm, v, faces, exact=True)
    o2, j2, _ = ops.measure_jacobian_betas(packed, lm, v, faces, exact=True)
    assert torch.equal(_bits(j1), _bits(j2))
    o3, j3, _ = ops.measure_jacobian_betas(packed, lm, v[77:78].clone(), faces, exact=True)
    assert torch.equal(_bits(j3[0]), _bits(j1[77])) and torch.equal(_bits(o3[0]), _bits(o1[77]))


def test_nan_rows_and_poisoning():
    """A body with every x = 0 slices into collinear points: its circumference rows are NaN and the rest of the
    Jacobian is finite; a non-zero upstream on a NaN circumference poisons the body's gradient, a zero one adds
    nothing; the neighbours are unaffected."""
    d = synth.make_smplx()
    ops, packed, faces, lm, v = _setup(d, 3, seed=8)
    v = v.clone()
    v[1, :, 0] = 0.0
    out, jac, _ = ops.measure_jacobian_betas(packed, lm, v, faces, exact=True)
    assert torch.isnan(out[1, 2:]).all() and torch.isnan(jac[1, 2:]).all()
    assert torch.isfinite(jac[1, :2]).all() and torch.isfinite(jac[[0, 2]]).all()
    go = np.tile([0.3, -2.0, 1.5, 0.7, -1.1], (3, 1))
    g = _grad(ops, lm, v, faces, go)
    assert torch.isnan(g[1]).all() and torch.isfinite(g[[0, 2]]).all()
    go[1, 2:] = 0.0
    g = _grad(ops, lm, v, faces, go)
    assert torch.isfinite(g).all()
    ref = _grad(ops, lm, v, faces, go, exact=False)
    assert torch.equal(_bits(g[1]), _bits(ref[1]))


FAMILIES = {m.meta['family']: m for m in ms.value_families()}


@pytest.mark.parametrize('fam', list(FAMILIES))
def test_constructed_slices_vs_oracle(fam):
    """The constructed slices (tests/measure_slices.py) through the vertex entry, one-hot circumference cotangents."""
    from shapy_b200 import ops
    mesh = FAMILIES[fam]
    lm = ops.make_landmarks(mesh.lm)
    v, f = torch.from_numpy(mesh.verts)[None].cuda(), torch.from_numpy(mesh.faces).cuda()
    out = ops.measure(lm, v_shaped=v, faces_i32=f)[0].cpu().numpy()
    for i in (2, 3, 4):
        go = np.eye(5)[i]
        g = _grad(ops, lm, v, f, go[None])[0].double().cpu().numpy()
        if np.isnan(out[i]):
            assert np.isnan(g).all(), (fam, i)
            continue
        want = meo.exact_grad(mesh.verts, mesh.faces, go, mesh.lm)
        err = np.abs(g - want).max() / max(np.abs(want).max(), 1e-30)
        assert err <= 1e-4, (fam, i, err)


def test_autograd_carries_the_choice():
    """BodyMeasurements.forward_vertices / forward with circumference_derivative='exact' backpropagate the exact
    gradient; the measurements and the no-grad launch are unchanged."""
    from shapy_b200 import _lib
    from shapy_b200.body_measurements import BodyMeasurements
    d = synth.make_smplx()
    ops, packed, faces, lm, v = _setup(d, 4, seed=12)
    bm = BodyMeasurements({'landmarks': synth.load_landmarks()}).cuda()
    go = torch.randn(4, 5, generator=torch.Generator().manual_seed(13)).cuda()
    x = v.clone().requires_grad_(True)
    m = bm.forward_vertices(x, faces, circumference_derivative='exact')['measurements']
    (torch.stack([m[k]['tensor'] for k in NAMES], 1) * go).sum().backward()
    assert torch.equal(_bits(x.grad), _bits(ops.measure_backward(lm, go, v_shaped=v, faces_i32=faces, exact=True)))
    tris = v[:, faces.long()].contiguous()
    t = tris.clone().requires_grad_(True)
    m = bm(t, circumference_derivative='exact')['measurements']
    (torch.stack([m[k]['tensor'] for k in NAMES], 1) * go).sum().backward()
    assert torch.equal(_bits(t.grad), _bits(ops.measure_backward(lm, go, triangles=tris, exact=True)))
    want = ops.measure(lm, v_shaped=v, faces_i32=faces)
    torch.cuda.synchronize()
    n0 = _lib.lib().shapy_launch_count()
    m = bm.forward_vertices(v, faces, circumference_derivative='exact')['measurements']
    assert _lib.lib().shapy_launch_count() - n0 == 1
    for i, k in enumerate(NAMES):
        assert torch.equal(m[k]['tensor'], want[:, i])


def test_argument_errors():
    from shapy_b200 import ops
    d = _generic(17)
    big = ops.SmplxModel(dict(d), 'cuda')
    lm = ops.make_landmarks(synth.load_landmarks())
    faces = d['faces_tensor'].to(torch.int32).cuda()
    with pytest.raises(RuntimeError):
        ops.measure_jacobian_betas(big, lm, torch.zeros(1, big.V, 3, device='cuda'), faces, exact=True)
    with pytest.raises(RuntimeError):
        ops.measure_backward(lm, torch.zeros(2, 4, device='cuda'), v_shaped=torch.zeros(2, big.V, 3, device='cuda'),
                             faces_i32=faces, exact=True)
