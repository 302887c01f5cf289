"""GPU: the measurement backward (shapy_measure_backward*, shapy_b200.autograd) against the reference's autograd
gradients (golden), the CPU oracle, and itself (entries, determinism, batch independence, the no-grad path)."""
import os

import numpy as np
import pytest
import torch

import measure_slices as ms
from oracle import measure_grad_oracle
from shapy_b200 import synth

pytestmark = pytest.mark.gpu
NAMES = ('mass', 'height', 'chest', 'waist', 'hips')


@pytest.fixture(scope='module')
def data(golden_dir):
    from shapy_b200 import ops
    g = np.load(os.path.join(golden_dir, 'img00_body.npz'))
    bodies = np.concatenate([g['v_shaped'][None], g['extra_v_shaped']], 0).astype(np.float32)
    ref = np.load(os.path.join(golden_dir, 'ref_measure_grad.npz'))
    return ops, bodies, g['faces'], synth.load_landmarks(), ref


def _gold(ref, name, b, V):
    if name == 'mass':
        return ref['mass'][b].astype(np.float64)
    out = np.zeros((V, 3))
    out[ref[f'{name}_{b}_rows']] = ref[f'{name}_{b}_values']
    return out


def _grad(ops, lm, x, faces, go, entry):
    go = torch.as_tensor(np.asarray(go, np.float32)).cuda()
    if entry == 'triangles':
        return ops.measure_backward(ops.make_landmarks(lm), go, triangles=x)
    return ops.measure_backward(ops.make_landmarks(lm), go, v_shaped=x, faces_i32=faces)


@pytest.mark.parametrize('entry', ['vertices', 'triangles'])
def test_golden_bodies_one_hot_and_mixed(data, entry):
    ops, bodies, faces_np, lm, ref = data
    B, V = bodies.shape[:2]
    v = torch.from_numpy(bodies).cuda()
    f = torch.from_numpy(faces_np).cuda()
    x = v[:, f.long()].contiguous() if entry == 'triangles' else v
    gos = [np.eye(5)[i] for i in range(5)] + [np.array([0.3, -2.0, 1.5, 0.7, -1.1])]
    for go in gos:
        g = _grad(ops, lm, x, f, np.tile(go, (B, 1)), entry)
        if entry == 'triangles':          # gather the triangle gradient onto the vertices
            gt = g.double().cpu().numpy()
            g = np.zeros((B, V, 3))
            for k in range(3):
                for b in range(B):
                    np.add.at(g[b], faces_np[:, k], gt[b, :, k])
        else:
            g = g.double().cpu().numpy()
        for b in range(B):
            refs = [go[i] * _gold(ref, n, b, V) for i, n in enumerate(NAMES)]
            want = sum(refs)
            scale = max(np.abs(r).max() for r in refs if np.abs(r).max() > 0)
            err = np.abs(g[b] - want).max() / scale
            assert err <= 1e-5 * max(1, int((go != 0).sum())), (entry, list(go), b, err)


def test_vertex_entry_equals_gathered_triangle_entry(data):
    ops, bodies, faces_np, lm, _ = data
    v = torch.from_numpy(bodies).cuda()
    f = torch.from_numpy(faces_np).cuda()
    go = np.tile([0.3, -2.0, 1.5, 0.7, -1.1], (4, 1))
    gv = _grad(ops, lm, v, f, go, 'vertices')
    gt = _grad(ops, lm, v[:, f.long()].contiguous(), f, go, 'triangles')
    gathered = torch.zeros_like(gv, dtype=torch.float64)
    for k in range(3):
        gathered.index_add_(1, f[:, k].long(), gt[:, :, k].double())
    assert (gathered - gv.double()).abs().max() <= 1e-6 * gv.abs().max()


def test_64_synthetic_bodies_vs_oracle(data):
    ops, _, _, lm, _ = data
    smplx = synth.make_smplx()
    packed = ops.SmplxModel(dict(smplx), 'cuda')
    betas = torch.randn(64, 10, generator=torch.Generator().manual_seed(11)).clamp(-2, 2)
    vs = ops.smplx_forward_shape(packed, betas.cuda())
    faces = smplx['faces_tensor'].to(torch.int32).cuda()
    go = torch.randn(64, 5, generator=torch.Generator().manual_seed(12))
    out = ops.measure(ops.make_landmarks(lm), v_shaped=vs, faces_i32=faces).cpu().numpy()
    g = _grad(ops, lm, vs, faces, go.numpy(), 'vertices').double().cpu().numpy()
    vs_np, f_np = vs.cpu().numpy(), smplx['faces_tensor'].numpy()
    checked = 0
    for b in range(64):
        if np.isnan(out[b]).any():
            assert np.isnan(g[b]).all()
            continue
        ref = measure_grad_oracle.measure_grad(vs_np[b], f_np, go[b].numpy(), lm)
        assert np.abs(g[b] - ref).max() <= 2e-5 * np.abs(ref).max(), b
        checked += 1
    assert checked >= 56


FAMILIES = {m.meta['family']: m for m in ms.value_families() + [ms.exact_count(1025)]}


@pytest.mark.parametrize('entry', ['vertices', 'vertices_global', 'triangles'])
@pytest.mark.parametrize('fam', list(FAMILIES))
def test_slices_every_source(data, fam, entry):
    """Every constructed slice through every source: one-hot upstream gradients against the oracle; where the forward
    is NaN, a non-zero upstream gradient gives an all-NaN body and a zero one adds nothing."""
    ops = data[0]
    mesh = FAMILIES[fam]
    if entry == 'vertices_global':
        mesh = mesh.padded()
    lm = ops.make_landmarks(mesh.lm)
    v = torch.from_numpy(mesh.verts)[None].cuda()
    f = torch.from_numpy(mesh.faces).cuda()
    out = ops.measure(lm, v_shaped=v, faces_i32=f)[0].cpu().numpy()
    V = mesh.verts.shape[0]
    for i in range(5):
        go = np.eye(5)[i][None]
        if entry == 'triangles':
            gt = _grad(ops, mesh.lm, v[:, f.long()].contiguous(), f, go, 'triangles')[0].double().cpu().numpy()
            g = np.zeros((V, 3))
            for k in range(3):
                np.add.at(g, mesh.faces[:, k], gt[:, k])
        else:
            g = _grad(ops, mesh.lm, v, f, go, 'vertices')[0].double().cpu().numpy()
        if np.isnan(out[i]):
            assert np.isnan(g).all(), (fam, entry, i)
            continue
        assert np.isfinite(g).all(), (fam, entry, i)
        ref = measure_grad_oracle.measure_grad(mesh.verts, mesh.faces, np.eye(5)[i], mesh.lm)
        scale = max(np.abs(ref).max(), 1e-30)
        assert np.abs(g - ref).max() <= 1e-5 * scale, (fam, entry, i, np.abs(g - ref).max() / scale)
    # the NaN policy with a zero upstream gradient on the NaN outputs
    if np.isnan(out).any():
        go = np.where(np.isnan(out), 0.0, 1.0)[None]
        g = _grad(ops, mesh.lm, v, f, go, 'vertices')
        assert torch.isfinite(g).all(), (fam, entry)


def test_deterministic_and_batch_independent(data):
    ops, bodies, faces_np, lm, _ = data
    f = torch.from_numpy(faces_np).cuda()
    big = torch.from_numpy(bodies).cuda()[torch.arange(256) % 4]
    big = (big * (1 + 0.03 * torch.sin(torch.arange(256.0))).view(-1, 1, 1).cuda()).contiguous()
    go = torch.randn(256, 5, generator=torch.Generator().manual_seed(4)).numpy()
    for entry in ('vertices', 'triangles'):
        x = big if entry == 'vertices' else big[:, f.long()].contiguous()
        a = _grad(ops, lm, x, f, go, entry)
        b = _grad(ops, lm, x, f, go, entry)
        assert torch.equal(a, b), entry
        one = _grad(ops, lm, x[100:101].contiguous(), f, go[100:101], entry)
        assert torch.equal(one[0], a[100]), entry


def test_drop_in_backward_through_body_measurements(data):
    """The reference's loss (examples/fit_measurements.py) through `from body_measurements import BodyMeasurements`
    after install_as_reference(), with loss.backward()."""
    ops, bodies, faces_np, lm, ref = data
    import shapy_b200
    shapy_b200.install_as_reference()
    from body_measurements import BodyMeasurements
    bm = BodyMeasurements({'landmarks': lm}).cuda()
    v = torch.from_numpy(bodies[:1]).cuda().requires_grad_(True)
    tris = v[:, torch.from_numpy(faces_np).long().cuda()]
    gt = {'height': 1.7, 'mass': 60.0, 'chest': 0.9, 'waist': 0.8, 'hips': 1.0}
    weights = {'height': 100.0, 'mass': 1.0, 'chest': 2000.0, 'waist': 1000.0, 'hips': 1000.0}
    out = bm(tris)['measurements']
    loss = sum((gt[k] - out[k]['tensor']).pow(2).sum() * weights[k] for k in gt)
    loss.backward()
    est = {k: float(out[k]['tensor'][0]) for k in gt}
    V = bodies.shape[1]
    want = sum(-2.0 * weights[k] * (gt[k] - est[k]) * _gold(ref, k, 0, V) for k in gt)
    assert (v.grad[0].double().cpu().numpy() - want).__abs__().max() <= 1e-5 * np.abs(want).max()
    # a double backward raises
    v2 = torch.from_numpy(bodies[:1]).cuda().requires_grad_(True)
    m = bm.forward_vertices(v2, torch.from_numpy(faces_np).cuda())['measurements']['height']['tensor'].sum()
    (g,) = torch.autograd.grad(m, v2, create_graph=True)
    with pytest.raises(RuntimeError):
        g.sum().backward()


def test_no_grad_path_unchanged(data):
    ops, bodies, faces_np, lm, _ = data
    from shapy_b200 import _lib
    from shapy_b200.body_measurements import BodyMeasurements
    bm = BodyMeasurements({'landmarks': lm}).cuda()
    v = torch.from_numpy(bodies).cuda()
    f = torch.from_numpy(faces_np).cuda()
    want = ops.measure(ops.make_landmarks(lm), v_shaped=v, faces_i32=f)
    torch.cuda.synchronize()
    n0 = _lib.lib().shapy_launch_count()
    a = ops.measure(ops.make_landmarks(lm), v_shaped=v, faces_i32=f)
    n1 = _lib.lib().shapy_launch_count()
    m = bm.forward_vertices(v, f)['measurements']
    n2 = _lib.lib().shapy_launch_count()
    with torch.no_grad():
        m2 = bm.forward_vertices(v.clone().requires_grad_(True), f)['measurements']
    assert n2 - n1 == n1 - n0
    for i, k in enumerate(NAMES):
        assert torch.equal(m[k]['tensor'], want[:, i]) and not m[k]['tensor'].requires_grad
        assert torch.equal(m2[k]['tensor'], want[:, i]) and not m2[k]['tensor'].requires_grad
    assert torch.equal(a, want)
