"""CPU checks of the self-penetration oracles: the float64 restatement against the reference's own loss.py (golden),
its analytic gradient against central differences, the brute-force self-collision oracle on hand-built cases, and the
host-side helpers of the term."""
import os

import numpy as np
import pytest
import torch

import penetration_oracle as po

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'ref_penetration.npz')


def test_restatement_matches_reference_golden():
    z = np.load(GOLDEN)
    tris, idx = z['triangles'], z['collision_idxs']
    B, F = tris.shape[:2]
    v, faces = tris.reshape(B, 3 * F, 3), po.soup_faces(F)
    for k, (sigma, pout, lmax, _p2p) in enumerate(z['settings']):
        loss, grad = po.loss_and_grad(v, faces, idx, sigma, bool(pout), lmax)
        np.testing.assert_allclose(loss, z[f'loss_{k}'], rtol=1e-12, atol=1e-300)
        ref = z[f'grad_{k}'].reshape(B, 3 * F, 3)
        np.testing.assert_allclose(grad, ref, rtol=1e-9, atol=1e-12 * np.abs(ref).max())
        assert (z[f'loss_{k}'] > 0).all()
    loss, grad = po.loss_and_grad(v, faces, np.full((B, 4, 2), -1))
    assert (loss == z['loss_empty']).all() and not grad.any()


def _active_case(seed):
    rng = np.random.default_rng(seed)
    tris = rng.normal(size=(2, 12, 1, 3)) * 0.05 + rng.normal(size=(2, 12, 3, 3)) * 0.08
    pairs = np.stack([np.stack([np.arange(6), np.arange(6, 12)], -1)] * 2)
    return tris.reshape(2, 36, 3), po.soup_faces(12), pairs


@pytest.mark.parametrize('sigma,pout,lmax', [(0.5, True, 1000.0), (0.05, False, 1000.0), (0.3, True, 0.4)])
def test_gradient_matches_central_differences(sigma, pout, lmax):
    v, faces, pairs = _active_case(3)
    gl = np.array([1.0, -0.7])
    loss, grad = po.loss_and_grad(v, faces, pairs, sigma, pout, lmax, grad_loss=gl)
    assert (loss > 0).all()
    h = 1e-6
    fd = np.zeros_like(v)
    for idx in np.ndindex(*v.shape):
        vp, vm = v.copy(), v.copy()
        vp[idx] += h
        vm[idx] -= h
        fd[idx] = (gl @ po.loss(vp, faces, pairs, sigma, pout, lmax) - gl @ po.loss(vm, faces, pairs, sigma, pout, lmax)) / (2 * h)
    np.testing.assert_allclose(grad, fd, rtol=1e-5, atol=1e-7 * np.abs(fd).max())


def test_zero_area_face_gives_nan():
    v = np.array([[[0, 0, 0], [1, 0, 0], [2, 0, 0], [0, 0, 0.1], [1, 1, 0.1], [0, 1, -0.1]]], np.float64)
    loss = po.loss(v, [[0, 1, 2], [3, 4, 5]], [[[0, 1]]])
    assert np.isnan(loss).all()


def _tri(*pts):
    return np.array(pts, np.float32)


def hand_built_case():
    """Faces 0 and 1 cross; face 2 shares an edge (two vertex indices) with face 0 in its plane; a vertex of face 3 lies
    on face 0's interior (a touching pair: the box and SAT tests are inclusive); face 4 is far from everything."""
    v = np.concatenate([
        _tri([0, 0, 0], [1, 0, 0], [0, 1, 0]),
        _tri([0.2, 0.2, -0.5], [0.3, 0.2, 0.5], [0.2, 0.3, 0.5]),
        _tri([5, 5, 5], [6, 5, 5], [0.5, -0.5, 0]),
        _tri([0.25, 0.22, 0.0], [2.0, 2.0, 2.0], [2.0, 3.0, 2.0]),
        _tri([9, 9, 9], [9.5, 9, 9], [9, 9.5, 9]),
        _tri([0, 0, 0], [1, 0, 0], [0, 0, 0]),
    ])
    faces = np.array([[0, 1, 2], [3, 4, 5], [0, 1, 8], [9, 10, 11], [12, 13, 14]])
    return v, faces


def test_oracle_hand_built_pairs():
    v, faces = hand_built_case()
    assert po.self_collisions(v, faces).tolist() == [[0, 1], [0, 3]]
    # the same edge through copies of its vertices is a pair: the exclusion is by vertex index
    assert po.self_collisions(v, np.array([[0, 1, 2], [3, 4, 5], [15, 16, 8], [9, 10, 11], [12, 13, 14]])).tolist() \
        == [[0, 1], [0, 2], [0, 3]]
    assert po.self_collisions(v, faces, np.array([0, 1, 0, 2, 3]), [(1, 0)]).tolist() == [[0, 3]]
    lifted = v.copy()
    lifted[9, 2] = 1e-3                              # face 3 lifted off face 0: no contact
    assert po.self_collisions(lifted, faces).tolist() == [[0, 1]]


def test_face_parts_and_parent_pairs():
    from shapy_b200 import ops
    w = torch.tensor([[1.0, 0, 0], [0, 1, 0], [0, 0.5, 0.5], [0, 0, 1]])
    faces = torch.tensor([[0, 1, 2], [1, 2, 3], [0, 3, 2]])
    # face 0: (1, 1.5, 0.5) -> 1; face 1: (0, 1.5, 1.5) -> tie -> 1; face 2: (1, 0.5, 1.5) -> 2
    assert ops.face_parts({'lbs_weights': w, 'faces_tensor': faces}).tolist() == [1, 1, 2]
    assert ops.parent_child_part_pairs(torch.tensor([-1, 0, 0, 1])) == [(1, 0), (2, 0), (3, 1)]


def test_mirror_rejects_what_the_reference_cannot_run():
    from shapy_b200.mesh_mesh_intersection_loss import DistanceFieldPenetrationLoss
    t = torch.zeros(1, 2, 3, 3)
    with pytest.raises(NotImplementedError):
        DistanceFieldPenetrationLoss(vectorized=False)(t, torch.zeros(1, 1, 2, dtype=torch.long))
    with pytest.raises(TypeError):
        DistanceFieldPenetrationLoss()(t.double(), torch.zeros(1, 1, 2, dtype=torch.long))
