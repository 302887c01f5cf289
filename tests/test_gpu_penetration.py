"""GPU: self-collision detection (ops.self_collisions) against the brute-force oracle of tests/penetration_oracle.py,
pairs and order, on constructed soups and on self-intersecting posed synthetic bodies; its independence of the batch,
the tree and the run; and the penetration loss and gradient against the float64 restatement and the reference's own
loss.py (tests/golden/ref_penetration.npz)."""
import os
import sys

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import penetration_oracle as po
from test_penetration_cpu import hand_built_case
from shapy_b200 import ops, synth
from penetration_oracle import smooth_smplx

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'ref_penetration.npz')
_CACHE = {}


def _rows(pairs, count):
    """The valid rows of one body of ops.self_collisions as an (n, 2) int64 array."""
    n = min(int(count), pairs.shape[0])
    assert (pairs[n:] == -1).all()
    return pairs[:n].cpu().numpy().astype(np.int64)


# SMPL-X body_pose rows (joint - 1): hips 0 / 1, knees 3 / 4, elbows 17 / 18
POSES = {
    'elbows_flexed': {17: [0, -2.6, 0], 18: [0, 2.6, 0]},
    'elbows_half_flexed': {17: [0, -1.6, 0], 18: [0, 1.6, 0]},
    'thigh_crossed': {0: [0, 0, -0.7], 1: [0, 0, 0.2]},
    'knees_and_elbows': {3: [2.4, 0, 0], 4: [2.4, 0, 0], 17: [0, -2.4, 0.5], 18: [0, 2.4, -0.5]},
}


def _bodies():
    if _CACHE:
        return _CACHE
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    m = SMPLX(data_struct=smooth_smplx()).cuda()
    B = len(POSES)
    rot = np.tile(np.eye(3, dtype=np.float32), (B, 22, 1, 1))
    for b, pose in enumerate(POSES.values()):
        for j, aa in pose.items():
            rot[b, 1 + j] = Rotation.from_rotvec(aa).as_matrix()
    rot = torch.tensor(rot).cuda()
    with torch.no_grad():
        v = m(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=torch.zeros(B, m.num_betas, device='cuda'),
              return_shaped=False)['vertices'].contiguous()
    labels = ops.face_parts(m)
    ignored = ops.parent_child_part_pairs(m.parents)
    _CACHE.update(model=m, v=v, faces=m.faces_i32, labels=labels, ignored=ignored, oracle={})
    return _CACHE


def _oracle(c, b, filtered):
    key = (b, filtered)
    if key not in c['oracle']:
        lab = c['labels'].numpy() if filtered else None
        c['oracle'][key] = po.self_collisions(c['v'][b].cpu().numpy(), c['faces'].cpu().numpy(), lab,
                                              c['ignored'] if filtered else (), max_hits=512)
    return c['oracle'][key]


def test_constructed_soups_match_oracle():
    v, faces = hand_built_case()
    vv = torch.tensor(v[None]).cuda()
    ff = torch.tensor(faces, dtype=torch.int32).cuda()
    pairs, count = ops.self_collisions(vv, ff, 8)
    assert _rows(pairs[0], count[0]).tolist() == [[0, 1], [0, 3]]
    pairs, count = ops.self_collisions(vv, ff, 8, part_labels=[0, 1, 0, 2, 3], ignored_part_pairs=[(1, 0)])
    assert _rows(pairs[0], count[0]).tolist() == [[0, 3]]
    # soups of small random triangles, every fourth one sharing a vertex index with the one before
    rng = np.random.default_rng(5)
    B, F = 3, 400
    centres = rng.uniform(0, 1.2, size=(B, F, 1, 3))
    verts = (centres + rng.normal(size=(B, F, 3, 3)) * 0.06).reshape(B, 3 * F, 3).astype(np.float32)
    fc = np.arange(3 * F).reshape(F, 3)
    fc[4::4, 0] = fc[3::4, 2][:fc[4::4].shape[0]]
    ff = torch.tensor(fc, dtype=torch.int32).cuda()
    pairs, count = ops.self_collisions(torch.tensor(verts).cuda(), ff, 4096)
    for b in range(B):
        want = po.self_collisions(verts[b], fc)
        assert 20 < len(want) < 4096
        np.testing.assert_array_equal(_rows(pairs[b], count[b]), want)


@pytest.mark.parametrize('filtered', [False, True])
def test_posed_bodies_match_oracle(filtered):
    c = _bodies()
    kw = dict(part_labels=c['labels'], ignored_part_pairs=c['ignored']) if filtered else {}
    pairs, count = ops.self_collisions(c['v'], c['faces'], 4096, **kw)
    hit = 0
    for b, name in enumerate(POSES):
        want = _oracle(c, b, filtered)
        assert int(count[b]) == len(want), name
        np.testing.assert_array_equal(_rows(pairs[b], count[b]), want[:4096], err_msg=name)
        hit += len(want) > 0
        print(f'{name}: {len(want)} pairs ({"part-filtered" if filtered else "unfiltered"})', file=sys.stderr)
    assert hit >= 3


def test_independent_of_batch_tree_and_run():
    c = _bodies()
    v, faces = c['v'], c['faces']
    pairs, count = ops.self_collisions(v, faces, 2048)
    for b in range(v.shape[0]):
        p1, c1 = ops.self_collisions(v[b:b + 1].contiguous(), faces, 2048)
        assert torch.equal(p1[0], pairs[b]) and int(c1[0]) == int(count[b])
    p2, c2 = ops.self_collisions(v, faces, 2048)
    assert torch.equal(p2, pairs) and torch.equal(c2, count)
    # refit: the tree built on other poses, then refit to these, gives the fresh build's pairs
    tree = ops.ScanTree()
    ops.closest_points(v.flip(0).contiguous(), faces, v[:, :5].contiguous(), tree=tree)
    ops.self_collisions(v.flip(0).contiguous(), faces, 16, tree=tree)
    built_key = tree.key
    p3, c3 = ops.self_collisions(v, faces, 2048, tree=tree)
    assert tree.key == built_key
    assert torch.equal(p3, pairs) and torch.equal(c3, count)


def test_truncation_keeps_the_first_rows():
    c = _bodies()
    pairs, count = ops.self_collisions(c['v'], c['faces'], 4096)
    m = 3
    pt, ct = ops.self_collisions(c['v'], c['faces'], m)
    assert torch.equal(ct, count)
    for b in range(pairs.shape[0]):
        n = min(m, int(count[b]))
        assert torch.equal(pt[b, :n], pairs[b, :n]) and (pt[b, n:] == -1).all()
    assert int(count.max()) > m


def test_too_many_faces_raises():
    v = torch.zeros(1, 3, 3, device='cuda')
    faces = torch.zeros(ops.MAX_SCAN_FACES + 1, 3, dtype=torch.int32, device='cuda')
    faces[:, 1], faces[:, 2] = 1, 2
    with pytest.raises(ValueError):
        ops.self_collisions(v, faces, 4)


def _loss_case():
    c = _bodies()
    pairs, count = ops.self_collisions(c['v'], c['faces'], 1024, part_labels=c['labels'],
                                       ignored_part_pairs=c['ignored'])
    assert int(count.min()) > 0
    return c, pairs


@pytest.mark.parametrize('sigma,pout,lmax', [(0.5, True, 1000.0), (0.005, False, 1000.0), (0.01, True, 0.004)])
def test_loss_and_gradient_match_oracle(sigma, pout, lmax):
    c, pairs = _loss_case()
    v, faces = c['v'], c['faces']
    loss = ops.penetration_forward(v, faces, pairs, sigma, pout, lmax)
    gl = torch.linspace(1.0, -0.5, v.shape[0], device='cuda')
    grad = ops.penetration_backward(v, faces, pairs, gl, sigma, pout, lmax)
    want_l, want_g = po.loss_and_grad(v.double().cpu().numpy(), faces.cpu().numpy(), pairs.cpu().numpy(), sigma, pout,
                                      lmax, grad_loss=gl.double().cpu().numpy())
    assert (want_l > 0).sum() >= 3
    np.testing.assert_allclose(loss.double().cpu().numpy(), want_l, rtol=2e-3, atol=1e-6 * want_l.max())
    g = grad.double().cpu().numpy()
    for b in range(v.shape[0]):
        scale = np.abs(want_g[b]).max() + 1e-30
        assert np.abs(g[b] - want_g[b]).max() <= 5e-3 * scale, b
    assert torch.equal(ops.penetration_forward(v, faces, pairs, sigma, pout, lmax), loss)
    assert torch.equal(ops.penetration_backward(v, faces, pairs, gl, sigma, pout, lmax), grad)
    l1 = ops.penetration_forward(v[1:2].contiguous(), faces, pairs[1:2].contiguous(), sigma, pout, lmax)
    g1 = ops.penetration_backward(v[1:2].contiguous(), faces, pairs[1:2].contiguous(), gl[1:2].contiguous(), sigma,
                                  pout, lmax)
    assert torch.equal(l1[0], loss[1]) and torch.equal(g1[0], grad[1])


def test_mirror_module_matches_reference_golden():
    from shapy_b200.mesh_mesh_intersection_loss import DistanceFieldPenetrationLoss
    z = np.load(GOLDEN)
    idx = torch.tensor(z['collision_idxs']).cuda()
    for k, (sigma, pout, lmax, p2p) in enumerate(z['settings']):
        t = torch.tensor(z['triangles'], dtype=torch.float32).cuda().requires_grad_(True)
        loss = DistanceFieldPenetrationLoss(sigma=sigma, point2plane=bool(p2p), penalize_outside=bool(pout),
                                            linear_max=lmax)(t, idx)
        loss.sum().backward()
        ref_l, ref_g = z[f'loss_{k}'], z[f'grad_{k}']
        np.testing.assert_allclose(loss.detach().double().cpu().numpy(), ref_l, rtol=2e-3, atol=1e-6 * ref_l.max())
        g = t.grad.double().cpu().numpy()
        assert np.abs(g - ref_g).max() <= 5e-3 * np.abs(ref_g).max(), k
    t = torch.tensor(z['triangles'], dtype=torch.float32).cuda()
    assert (DistanceFieldPenetrationLoss()(t, torch.full((3, 4, 2), -1).cuda()) == 0).all()


def test_install_as_reference_registers_the_loss():
    import shapy_b200
    from shapy_b200.mesh_mesh_intersection_loss import DistanceFieldPenetrationLoss as Ours
    shapy_b200.install_as_reference()
    from mesh_mesh_intersection.loss import DistanceFieldPenetrationLoss
    assert DistanceFieldPenetrationLoss is Ours
