"""shapy_mmi_forward against the REFERENCE's own CUDA kernel (mesh-mesh-intersection, SURVEY.md 8c).  The reference
operator was run once on these exact inputs (oracle/build_ref.py builds it, oracle/run_ref_mmi.py runs it) and its
collisions are stored as tests/golden/ref_mmi_*.npz: the (body, slot) index, face and barycentrics of every slot it
filled.  The reference is compiled with nvcc's default FMA contraction, shapy_b200's predicates with -fmad=false (to be
bit-equal to the plain-C oracle), so a pair sitting exactly on a tolerance (SAT `CMP`, |det| < 1e-4) may legitimately
fall on different sides: the bars below allow a handful of such pairs and are otherwise exact."""
import os

import numpy as np
import pytest
import torch

from shapy_b200 import synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_reference(name, query):
    """The stored reference result for `query`: faces (B, Q * M) with -1 in empty slots, bcs (B, Q * M, 2, 3)."""
    d = np.load(os.path.join(ROOT, 'tests', 'golden', f'{name}.npz'))
    assert np.array_equal(d['query'], query), 'the inputs differ from those the reference was run on'
    shape = tuple(int(x) for x in d['shape'])
    faces = np.full(shape, -1, np.int64)
    bcs = np.zeros(shape + (2, 3), np.float32)
    idx = tuple(d['idx'].T)
    faces[idx] = d['faces']
    bcs[idx] = d['bcs']
    return faces, bcs


def compare(r, m, max_set_diff, what):
    """r, m: {(query, face): bcs}.  Collision sets equal up to max_set_diff borderline pairs; barycentrics of the common
    pairs equal to 1e-4 for all but 1 % (a borderline ray test flips which edge supplies the point)."""
    diff = set(r) ^ set(m)
    assert len(diff) <= max_set_diff, (what, len(diff), sorted(diff)[:8])
    common = sorted(set(r) & set(m))
    bad = [k for k in common if np.abs(r[k] - m[k]).max() > 1e-4]
    assert len(bad) <= max(1, len(common) // 100), (what, len(bad), len(common), bad[:4])
    return len(common)


def as_dict(faces, bcs, M):
    """{(query, face): bcs (2,3)} of one body."""
    out = {}
    for s in np.nonzero(faces >= 0)[0]:
        out[(int(s) // M, int(faces[s]))] = bcs[s]
    return out


def plane_inputs(golden_dir):
    """(query, target, max_collisions): the chest-plane quad of 4 real bodies against their 20 908 triangles."""
    g = np.load(os.path.join(golden_dir, 'img00_body.npz'))
    lm = synth.load_landmarks()
    bodies = np.concatenate([g['v_shaped'][None], g['extra_v_shaped']], 0).astype(np.float32)
    tris = bodies[:, g['faces']]                                               # (4, F, 3, 3)
    queries = []
    for b in range(bodies.shape[0]):
        h = float((tris[b, lm['chest']['face_idx']] * np.float32(lm['chest']['bc'])[:, None]).sum(0)[1])
        quad = np.float32([[-1, h, -1], [1, h, -1], [1, h, 1], [-1, h, 1]])     # body_measurements.py:90-97
        queries.append(np.stack([quad[[0, 1, 2]], quad[[0, 2, 3]]]))
    return np.stack(queries).astype(np.float32), np.ascontiguousarray(tris), 256


def soup_inputs():
    """(query, target, max_collisions): two seeded triangle soups, ~180 colliding pairs, at most 5 per query."""
    rng = np.random.default_rng(11)
    B, Q, F = 2, 96, 400

    def soup(n, spread, size):
        c = rng.uniform(-spread, spread, (B, n, 1, 3))
        return (c + rng.normal(0, size, (B, n, 3, 3))).astype(np.float32)
    query = soup(Q, 1.0, 0.15)
    return query, soup(F, 1.0, 0.15), 64


def test_plane_queries_on_real_bodies(golden_dir):
    """The hot-path use: the two triangles of a measurement plane against the 20 908 body triangles."""
    from shapy_b200 import ops
    query, tris, M = plane_inputs(golden_dir)
    ref_f, ref_b = run_reference('ref_mmi_plane', query)
    mine_f, mine_b = ops.mesh_to_mesh_forward(torch.from_numpy(query).cuda(), torch.from_numpy(np.ascontiguousarray(tris)).cuda(), M)
    mine_f, mine_b = mine_f.cpu().numpy(), mine_b.cpu().numpy()
    for b in range(query.shape[0]):
        r, m = as_dict(ref_f[b], ref_b[b], M), as_dict(mine_f[b], mine_b[b], M)
        assert compare(r, m, 2, f'body {b}') > 50


def test_random_mesh_against_mesh():
    """General use of the operator: every triangle of one mesh against another."""
    from shapy_b200 import ops
    query, target, M = soup_inputs()
    B = query.shape[0]
    ref_f, ref_b = run_reference('ref_mmi_soup', query)
    mine_f, mine_b = ops.mesh_to_mesh_forward(torch.from_numpy(query).cuda(), torch.from_numpy(target).cuda(), M)
    mine_f, mine_b = mine_f.cpu().numpy(), mine_b.cpu().numpy()
    total = 0
    for b in range(B):
        r, m = as_dict(ref_f[b], ref_b[b], M), as_dict(mine_f[b], mine_b[b], M)
        total += compare(r, m, max(2, len(r) // 100), f'soup {b}')
    assert total > 100
