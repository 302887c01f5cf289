"""GPU: the scan queries (ops.closest_points, ops.nearest_points, ops.closest_points_backward and
autograd.ClosestPointsFunction) against the float64 brute force of tests/scan_oracle.py on posed synthetic SMPL-X bodies,
their determinism (run to run, alone or in a batch, fresh or refit tree) and their edges."""
import numpy as np
import pytest
import torch

import scan_oracle as so
from shapy_b200 import ops, synth

pytestmark = pytest.mark.gpu

# Bars recorded from the first run on an H100 80GB HBM3 (700 W), with headroom: the distance |d - d64| and the
# position of the returned closest point (metres), and the backward's error relative to its largest entry.
DIST_BAR = 1e-6      # first run: 6.8e-7 (closest points), 1.5e-8 (nearest points)
GRAD_BAR = 5e-7      # first run: 1.9e-7


def _bits(t):
    return t.contiguous().view(torch.int32)


_CACHE = {}


def _model():
    if 'm' not in _CACHE:
        from shapy_b200.human_shape.models.body_models.body_models import SMPLX
        _CACHE['m'] = SMPLX(data_struct=synth.make_smplx()).cuda()
    return _CACHE['m']


def _bodies(B, seed):
    """Posed bodies of the 2D recipe: betas ~ N(0, 1) clipped to 2, raw pose = mean + 0.3 N, a random translation."""
    m = _model()
    gen = torch.Generator().manual_seed(seed)
    betas = torch.randn(B, m.num_betas, generator=gen).clamp(-2, 2).cuda()
    raw = (synth.mean_params()[:132] + 0.3 * torch.randn(B, 132, generator=gen)).cuda()
    transl = (0.3 * torch.randn(B, 3, generator=gen)).cuda()
    with torch.no_grad():
        rot = ops.decode_rot6d(raw)
        return m(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=betas, transl=transl,
                 return_shaped=False)['vertices'].contiguous()


def _points(verts, n, seed):
    """Per body n points: half on the surface, 3/8 up to 5 cm off it, 1/8 far (up to 1 m from the body's centre)."""
    faces = _model().faces_tensor.cpu().numpy()
    rng = np.random.default_rng(seed)
    out = []
    for v in verts.double().cpu().numpy():
        n_s, n_o = n // 2, 3 * n // 8
        s, _, _ = so.sample_surface(v, faces, n_s + n_o, rng)
        d = rng.normal(size=(n_o, 3))
        s[n_s:] += d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(0, 0.05, (n_o, 1))
        far = v.mean(0) + rng.uniform(-1, 1, (n - n_s - n_o, 3))
        out.append(np.concatenate([s, far]))
    return torch.tensor(np.stack(out), dtype=torch.float32).cuda()


@pytest.fixture(scope='module')
def scene():
    v = _bodies(4, 1)
    p = _points(v, 512, 2)
    return v, _model().faces_i32, p


def test_closest_points_vs_float64_brute_force(scene):
    v, faces, p = scene
    face, bary, d2 = ops.closest_points(v, faces, p)
    fn = faces.cpu().numpy()
    worst = {'dist': 0.0, 'face_dist': 0.0, 'point': 0.0}
    unique = same = 0
    for b in range(v.shape[0]):
        vb, pb = v[b].double().cpu().numpy(), p[b].double().cpu().numpy()
        f64, _, d64, second = so.closest_points(vb, fn, pb)
        fk = face[b].cpu().numpy()
        assert ((fk >= 0) & (fk < fn.shape[0])).all()
        dk = np.sqrt(d2[b].double().cpu().numpy())
        worst['dist'] = max(worst['dist'], float(np.abs(dk - np.sqrt(d64)).max()))
        # the float64 distance to the returned face is the float64 minimum
        tri = vb[fn[fk]]
        dkf = np.array([so.closest_on_faces(pb[i:i + 1], tri[i:i + 1])[0][0, 0] for i in range(len(pb))])
        worst['face_dist'] = max(worst['face_dist'], float(np.abs(np.sqrt(dkf) - np.sqrt(d64)).max()))
        # the returned barycentrics give a point at the returned distance from p
        q = (bary[b].double().cpu().numpy()[:, :, None] * tri).sum(1)
        worst['point'] = max(worst['point'], float(np.abs(np.linalg.norm(q - pb, axis=1) - dk).max()))
        assert (bary[b] >= -1e-6).all() and torch.allclose(bary[b].sum(1), torch.ones_like(bary[b, :, 0]), atol=1e-5)
        u = np.sqrt(second) - np.sqrt(d64) > 10 * DIST_BAR
        unique += int(u.sum())
        same += int((fk[u] == f64[u]).sum())
    print(f'[scan] closest points: max |d - d64| {worst["dist"]:.2e}, returned face vs minimum {worst["face_dist"]:.2e}, '
          f'closest point {worst["point"]:.2e} m; faces equal on {same} / {unique} unique minima')
    assert max(worst.values()) <= DIST_BAR
    assert same == unique


def test_nearest_points_vs_brute_force(scene):
    v, _, p = scene
    gen = torch.Generator().manual_seed(3)
    w = (torch.rand(p.shape[:2], generator=gen) + 0.1).cuda()
    w[:, ::10] = 0.0
    pn = p.clone()
    pn[:, ::10] = float('nan')
    idx, d2 = ops.nearest_points(v, pn, w)
    worst, unique, same = 0.0, 0, 0
    for b in range(v.shape[0]):
        i64, d64, second = so.nearest_points(v[b].double().cpu().numpy(), pn[b].double().cpu().numpy(),
                                             w[b].cpu().numpy())
        ik = idx[b].cpu().numpy()
        assert (ik % 10 != 0).all() and (ik >= 0).all()
        worst = max(worst, float(np.abs(np.sqrt(d2[b].double().cpu().numpy()) - np.sqrt(d64)).max()))
        u = np.sqrt(second) - np.sqrt(d64) > 10 * DIST_BAR
        unique += int(u.sum())
        same += int((ik[u] == i64[u]).sum())
    print(f'[scan] nearest points: max |d - d64| {worst:.2e} m; indices equal on {same} / {unique} unique minima')
    assert worst <= DIST_BAR and same == unique


def test_backward_vs_oracle_and_directional_derivatives(scene):
    from shapy_b200.autograd import ClosestPointsFunction
    v, faces, p = scene
    gen = torch.Generator().manual_seed(4)
    g = torch.randn(p.shape[:2], generator=gen).cuda()
    face, bary, _ = ops.closest_points(v, faces, p)
    grad = ops.closest_points_backward(v, faces, p, face, bary, g)
    fn = faces.cpu().numpy()
    worst = 0.0
    for b in range(v.shape[0]):
        want = so.sq_dist_grad(v[b].double().cpu().numpy(), fn, p[b].double().cpu().numpy(), face[b].cpu().numpy(),
                               bary[b].double().cpu().numpy(), g[b].double().cpu().numpy())
        worst = max(worst, float(np.abs(grad[b].double().cpu().numpy() - want).max() / np.abs(want).max()))
    # the autograd function gives the same bits
    vv = v.clone().requires_grad_(True)
    (ClosestPointsFunction.apply(faces, vv, p, None) * g).sum().backward()
    assert torch.equal(_bits(vv.grad), _bits(grad))
    # directional derivatives of L = sum_i g_i d_i^2 on body 0 against central differences of the float64 distance; the
    # step is small enough that no far point's nearest vertex changes between the two sides
    vb, pb, gb = v[0].double().cpu().numpy(), p[0].double().cpu().numpy(), g[0].double().cpu().numpy()
    rng = np.random.default_rng(5)
    h, rel = 1e-6, []
    for _ in range(3):
        dirn = rng.normal(size=vb.shape)
        L = [float((gb * so.closest_points(vb + s * h * dirn, fn, pb)[2]).sum()) for s in (1, -1)]
        fd = (L[0] - L[1]) / (2 * h)
        an = float((grad[0].double().cpu().numpy() * dirn).sum())
        rel.append(abs(an - fd) / abs(fd))
    print(f'[scan] backward vs oracle: max error / max entry {worst:.2e}; directional derivatives vs float64 central '
          f'differences, relative {max(rel):.2e}')
    assert worst <= GRAD_BAR
    assert max(rel) <= 1e-3


def test_bits_run_to_run_alone_in_a_batch_and_refit(scene):
    v, faces, p = scene
    other = _bodies(64, 7)
    pts64 = _points(other, 512, 8)
    rows = [0, 17, 40]
    vb, pb = other.clone(), pts64.clone()
    vb[rows], pb[rows] = v[:3], p[:3]
    gen = torch.Generator().manual_seed(9)
    g = torch.randn(64, 512, generator=gen).cuda()
    a = ops.closest_points(v, faces, p)
    b = ops.closest_points(v, faces, p)
    big = ops.closest_points(vb, faces, pb)
    tree = ops.ScanTree()
    ops.closest_points(other[:4].contiguous(), faces, p, tree=tree)       # built on other poses
    assert tree.key is not None
    refit = ops.closest_points(v, faces, p, tree=tree)                     # refit to these
    for x, y, z, r in zip(a, b, big, refit):
        assert torch.equal(_bits(x), _bits(y))
        assert torch.equal(_bits(x[:3]), _bits(z[rows]))
        assert torch.equal(_bits(x), _bits(r))
    ga = ops.closest_points_backward(v, faces, p, a[0], a[1], g[:4].contiguous())
    gb = ops.closest_points_backward(v, faces, p, a[0], a[1], g[:4].contiguous())
    gbig = ops.closest_points_backward(vb, faces, pb, big[0], big[1], _rows_of(g, rows))
    assert torch.equal(_bits(ga), _bits(gb))
    assert torch.equal(_bits(ga[:3]), _bits(gbig[rows]))
    na = ops.nearest_points(v, p)
    nbig = ops.nearest_points(vb, pb)
    for x, z in zip(na, nbig):
        assert torch.equal(_bits(x[:3]), _bits(z[rows]))


def _rows_of(g, rows):
    """A (64, 512) cotangent whose rows `rows` are the first rows of g (the 4-body batch's)."""
    out = g.clone()
    out[rows] = g[:len(rows)]
    return out


def test_dropped_points_are_never_read_and_empty_batches(scene):
    v, faces, p = scene
    w = torch.ones(p.shape[:2], device='cuda')
    w[:, 3::7] = 0.0
    w[:, 5::11] = -1.0
    drop = w <= 0
    pn = torch.where(drop[..., None], torch.full_like(p, float('nan')), p)
    face, bary, d2 = ops.closest_points(v, faces, pn, w)
    ref = ops.closest_points(v, faces, p)
    assert (face[drop] == -1).all() and (d2[drop] == 0).all() and (bary[drop] == 0).all()
    keep = ~drop
    assert torch.equal(face[keep], ref[0][keep]) and torch.equal(_bits(d2[keep]), _bits(ref[2][keep]))
    g = torch.where(drop, torch.full_like(d2, float('nan')), torch.ones_like(d2))
    grad = ops.closest_points_backward(v, faces, pn, face, bary, g)
    assert bool(torch.isfinite(grad).all())
    # empty batches and point sets launch nothing
    n0 = ops.lib().shapy_launch_count()
    f0, b0, e0 = ops.closest_points(v[:0], faces, p[:0])
    assert f0.shape == (0, 512) and b0.shape == (0, 512, 3)
    f1, b1, e1 = ops.closest_points(v, faces, p[:, :0])
    assert f1.shape == (4, 0) and e1.shape == (4, 0)
    idx, dd = ops.nearest_points(v, p[:, :0])
    assert (idx == -1).all() and (dd == 0).all()
    assert ops.lib().shapy_launch_count() == n0
    gz = ops.closest_points_backward(v, faces, p[:, :0], f1, b1, e1)
    assert bool((gz == 0).all())
    # limits
    with pytest.raises(ValueError, match='32768'):
        ops.closest_points(v, faces, torch.zeros(4, 32769, 3, device='cuda'))
    with pytest.raises(ValueError, match='32768'):
        ops.nearest_points(v, torch.zeros(4, 32769, 3, device='cuda'))
    with pytest.raises(ValueError, match='32768'):
        ops.closest_points(v, torch.zeros(32769, 3, dtype=torch.int32, device='cuda'), p)
