"""The CPU restatement of the measurement gradient (oracle/measure_grad_oracle.measure_grad) against the reference's own
autograd gradients: the stored golden (tests/golden/ref_measure_grad.npz) and, where the reference tree exists, the
reference's body_measurements.py run live."""
import os

import numpy as np
import pytest

from oracle import measure_grad_oracle, ref_body_measurements

NAMES = ('mass', 'height', 'chest', 'waist', 'hips')
# float32 reference vs the float32-faithful oracle: mass, height and hips agree to < 1e-6 of max|g|; the chest and
# waist rows of some bodies differ by up to 1e-5 (the reference accumulates the hull terms in float32, in an order
# the oracle cannot see)
TOL = {'mass': 1e-6, 'height': 1e-6, 'chest': 2e-5, 'waist': 2e-5, 'hips': 2e-5}


def _bodies(golden_dir):
    g = np.load(os.path.join(golden_dir, 'img00_body.npz'))
    return np.concatenate([g['v_shaped'][None], g['extra_v_shaped']], 0).astype(np.float32), g['faces']


def golden_grad(ref, name, b, V):
    if name == 'mass':
        return ref['mass'][b].astype(np.float64)
    out = np.zeros((V, 3))
    out[ref[f'{name}_{b}_rows']] = ref[f'{name}_{b}_values']
    return out


@pytest.mark.parametrize('b', range(4))
def test_oracle_grad_vs_golden(golden_dir, b):
    bodies, faces = _bodies(golden_dir)
    ref = np.load(os.path.join(golden_dir, 'ref_measure_grad.npz'))
    for i, name in enumerate(NAMES):
        go = np.zeros(5)
        go[i] = 1.0
        mine = measure_grad_oracle.measure_grad(bodies[b], faces, go)
        gold = golden_grad(ref, name, b, bodies.shape[1])
        err = np.abs(mine - gold).max() / np.abs(gold).max()
        assert err <= TOL[name], (b, name, err)


@pytest.mark.skipif(not ref_body_measurements.available(), reason='reference tree not available')
def test_oracle_grad_vs_live_reference(golden_dir):
    import torch
    BM, cfg = ref_body_measurements.load()
    bm = BM(cfg)
    bodies, faces = _bodies(golden_dir)
    go = np.array([0.3, -2.0, 1.5, 0.7, -1.1])
    v = torch.from_numpy(bodies[1])[None].clone().requires_grad_(True)
    m = bm(v[:, torch.from_numpy(faces.astype(np.int64))])['measurements']
    sum(float(go[i]) * m[k]['tensor'].sum() for i, k in enumerate(NAMES)).backward()
    ref = v.grad[0].double().numpy()
    mine = measure_grad_oracle.measure_grad(bodies[1], faces, go)
    assert np.abs(mine - ref).max() / np.abs(ref).max() < 2e-5
