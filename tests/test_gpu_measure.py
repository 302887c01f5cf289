"""GPU parity of the measurement kernel and the batched LBVH op against the golden img_00.npz values
and the plain-C restatement of the reference operator (oracle/mmi_oracle.c)."""
import os

import numpy as np
import pytest
import torch

from oracle import measure_oracle
from shapy_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def data(golden_dir):
    from shapy_b200 import ops
    g = np.load(os.path.join(golden_dir, 'img00_body.npz'))
    lm = synth.load_landmarks()
    return g, lm, ops


def _bodies(g):
    return np.concatenate([g['v_shaped'][None], g['extra_v_shaped']], 0).astype(np.float32)


def test_golden_measurements(data):
    """The reference's only golden vector: mass 56.868896, height 1.6437092, chest 0.8745367, ..."""
    g, lm, ops = data
    v = torch.from_numpy(g['v_shaped'])[None].cuda()
    f = torch.from_numpy(g['faces']).cuda()
    out = ops.measure(ops.make_landmarks(lm), v_shaped=v, faces_i32=f)[0].cpu().numpy()
    for i, (name, gold) in enumerate(zip(g['meas_names'], g['meas_values'])):
        assert abs(out[i] - gold) / gold < 1e-6, (name, out[i], gold)


def test_vs_oracle_real_bodies_and_point_sets(data):
    g, lm, ops = data
    bodies = _bodies(g)
    v = torch.from_numpy(bodies).cuda()
    f = torch.from_numpy(g['faces']).cuda()
    out, pts, cnt, status = ops.measure(ops.make_landmarks(lm), v_shaped=v, faces_i32=f, return_points=True)
    assert int(status.item()) == 0
    out = out.cpu().numpy()
    for b in range(bodies.shape[0]):
        ref = measure_oracle.measure(bodies[b], g['faces'], lm)
        for i, name in enumerate(('mass', 'height', 'chest', 'waist', 'hips')):
            assert abs(out[b, i] - ref[name]) / abs(ref[name]) < 2e-6, (b, name, out[b, i], ref[name])
        tris = bodies[b][g['faces']]
        for p, name in enumerate(('chest', 'waist', 'hips')):
            _, ref_pts, _ = measure_oracle.periphery(tris, lm[name]['face_idx'], lm[name]['bc'])
            n = int(cnt[b, p])
            mine = pts[b, p, :n].cpu().numpy()
            ref_u = np.unique(ref_pts.round(7), axis=0)      # oracle stores each point twice
            mine_u = np.unique(mine.round(7), axis=0)
            assert mine_u.shape == ref_u.shape and np.abs(mine_u - ref_u).max() < 1e-6, (b, name)


def test_triangles_entry_matches_vertices_entry(data):
    g, lm, ops = data
    bodies = _bodies(g)
    v = torch.from_numpy(bodies).cuda()
    f = torch.from_numpy(g['faces']).cuda()
    a = ops.measure(ops.make_landmarks(lm), v_shaped=v, faces_i32=f)
    tris = v[:, f.long()]
    b = ops.measure(ops.make_landmarks(lm), triangles=tris.contiguous())
    assert torch.equal(a, b)


def test_module_api_and_batch_independence(data):
    """BodyMeasurements.forward(triangles) output structure; 1024 bodies: rows independent of position."""
    g, lm, ops = data
    from shapy_b200.body_measurements import BodyMeasurements
    bm = BodyMeasurements({'landmarks': lm}).cuda()
    bodies = torch.from_numpy(_bodies(g)).cuda()
    f = torch.from_numpy(g['faces']).cuda()
    big = bodies[torch.arange(1024) % 4]
    scale = (1.0 + 0.05 * torch.sin(torch.arange(1024, dtype=torch.float32))).view(-1, 1, 1).cuda()
    big = (big * scale).contiguous()
    m = bm.forward_vertices(big, f)['measurements']
    assert set(m) == {'mass', 'height', 'chest', 'waist', 'hips'} and m['mass']['tensor'].shape == (1024,)
    sub = bm.forward_vertices(big[500:504].contiguous(), f)['measurements']
    for k in m:
        assert torch.equal(m[k]['tensor'][500:504], sub[k]['tensor'])
    # similarity: scaling a body by s scales lengths by s and mass by s^3 (same triangles hit the plane)
    s = 1.05
    one = bodies[:1]
    a = ops.measure(ops.make_landmarks(lm), v_shaped=one, faces_i32=f)[0]
    b = ops.measure(ops.make_landmarks(lm), v_shaped=(one * s).contiguous(), faces_i32=f)[0]
    assert abs(b[0] / a[0] - s ** 3) < 1e-5 and abs(b[1] / a[1] - s) < 1e-6
    assert all(abs(b[i] / a[i] - s) < 2e-3 for i in (2, 3, 4))
    out = bm(big[:2][:, f.long()].contiguous(), compute_mass=False)['measurements']    # triangles entry
    assert 'mass' not in out
    assert torch.equal(out['hips']['tensor'], m['hips']['tensor'][:2])


def _sets(faces, bcs, Q, M):
    out = []
    for q in range(Q):
        fq = faces[q * M:(q + 1) * M]
        bq = bcs[q * M:(q + 1) * M]
        idx = np.where(fq >= 0)[0]
        order = np.argsort(fq[idx], kind='stable')
        out.append((fq[idx][order], bq[idx][order]))
    return out


def test_mmi_op_plane_vs_body(data):
    """The SHAPY call: Q = 2 plane triangles against the 20 908-face body, max_collisions = 256."""
    g, lm, ops = data
    bodies = _bodies(g)
    tris = torch.from_numpy(bodies[:, g['faces']]).cuda().contiguous()
    hs = [float(bodies[b][g['faces'][lm['chest']['face_idx']]][2][1]) for b in range(4)]
    quads = np.stack([measure_oracle.plane_quad(np.float32(h)) for h in hs]).astype(np.float32)
    faces, bcs = ops.mesh_to_mesh_forward(torch.from_numpy(quads).cuda(), tris, max_collisions=256)
    assert faces.dtype == torch.int64 and faces.shape == (4, 512) and bcs.shape == (4, 512, 2, 3)
    rf, rb = measure_oracle.mesh_to_mesh_forward(quads, bodies[:, g['faces']], 256)
    faces, bcs = faces.cpu().numpy(), bcs.cpu().numpy()
    for b in range(4):
        for (f1, b1), (f2, b2) in zip(_sets(faces[b], bcs[b], 2, 256), _sets(rf[b], rb[b], 2, 256)):
            assert np.array_equal(f1, f2)
            assert np.abs(b1 - b2).max() < 1e-6


@pytest.mark.parametrize('Q,F,M', [(1, 1, 4), (5, 2, 4), (64, 500, 32), (300, 3000, 64)])
def test_mmi_op_random_meshes(data, Q, F, M):
    g, lm, ops = data
    rng = np.random.RandomState(Q * 1000 + F)
    B = 3

    def soup(n, size):
        c = rng.uniform(-1, 1, (B, n, 1, 3))
        return (c + rng.normal(0, size, (B, n, 3, 3))).astype(np.float32)
    q, t = soup(Q, 0.15), soup(F, 0.1)
    faces, bcs = ops.mesh_to_mesh_forward(torch.from_numpy(q).cuda(), torch.from_numpy(t).cuda(), max_collisions=M)
    rf, rb = measure_oracle.mesh_to_mesh_forward(q, t, M)
    faces, bcs = faces.cpu().numpy(), bcs.cpu().numpy()
    n_hits = 0
    for b in range(B):
        for qi, ((f1, b1), (f2, b2)) in enumerate(zip(_sets(faces[b], bcs[b], Q, M), _sets(rf[b], rb[b], Q, M))):
            if len(f2) == M:            # overflowing queries keep an arbitrary subset
                assert len(f1) == M
                continue
            assert np.array_equal(f1, f2), (b, qi)
            if len(f1):
                assert np.abs(b1 - b2).max() < 1e-6
            n_hits += len(f1)
    if F >= 500:
        assert n_hits > 0


def test_config4_4096_random_beta_bodies_vs_oracle(data):
    """BASELINE configs[3]: 4 096 clipped-normal betas (seed 3) -> T-pose bodies -> measurements in one launch each;
    64 of the 4 096 rows against the CPU oracle (shape blend restated in numpy, measure_oracle).

    The synthetic shape basis is white noise per vertex, so a few per cent of these bodies are crumpled enough that a
    slicing plane cuts > 1 024 triangles.  That is outside the reference's own domain (its buffers hold 256 collisions
    per query triangle, beyond which mesh_mesh_intersect_cuda_op.cu:551-557 writes out of bounds); the kernel must
    then report NaN + status instead of a truncated circumference.  Every plane with <= 1 024 points must match the
    oracle (run with a capacity large enough never to truncate)."""
    g, lm, ops = data
    smplx = synth.make_smplx()
    packed = ops.SmplxModel(dict(smplx), 'cuda')
    betas = torch.randn(4096, 10, generator=torch.Generator().manual_seed(3)).clamp(-3, 3)
    vs = ops.smplx_forward_shape(packed, betas.cuda())
    faces = smplx['faces_tensor'].to(torch.int32).cuda()
    out, _, cnt, status = ops.measure(ops.make_landmarks(lm), v_shaped=vs, faces_i32=faces, return_points=True, max_points=1024)
    out, cnt = out.cpu().numpy(), cnt.cpu().numpy()
    n_bad = int(np.isnan(out).any(1).sum())
    assert (int(status.item()) != 0) == (n_bad > 0)
    assert n_bad < 0.05 * 4096, n_bad
    assert not np.isnan(out[:, :2]).any()                                      # mass / height never overflow
    rows = list(np.random.default_rng(5).choice(4096, 60, replace=False)) + list(np.nonzero(np.isnan(out).any(1))[0][:4])
    vt = smplx['v_template'].double().numpy()
    S = smplx['shapedirs'].double().numpy()                                    # (V, 3, 10)
    f = smplx['faces_tensor'].numpy()
    checked = 0
    for r in rows:
        ref_v = (vt + S @ betas[r].double().numpy()).astype(np.float32)
        assert np.abs(vs[r].cpu().numpy() - ref_v).max() < 2e-6
        tris = np.ascontiguousarray(ref_v[f])
        assert abs(out[r, 0] - measure_oracle.mass(tris)) / measure_oracle.mass(tris) < 1e-4
        assert abs(out[r, 1] - measure_oracle.height(tris, lm)) / measure_oracle.height(tris, lm) < 1e-4
        for i, name in enumerate(('chest', 'waist', 'hips')):
            val, pts, _ = measure_oracle.periphery(tris, lm[name]['face_idx'], lm[name]['bc'], max_collisions=4096)
            n = len(pts) // 2                                                   # the oracle stores each point twice
            if n > 1024:
                assert np.isnan(out[r, 2 + i]), (int(r), name, n, out[r, 2 + i])
            else:
                assert cnt[r, i] == n, (int(r), name, cnt[r, i], n)
                assert abs(out[r, 2 + i] - val) / abs(val) < 1e-4, (int(r), name, out[r, 2 + i], val)
                checked += 1
    assert checked > 150
