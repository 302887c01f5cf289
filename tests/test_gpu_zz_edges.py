"""Edge cases of the public entry points on the GPU: empty batches (torch semantics: empty in, empty out, nothing
launched), batches that straddle the 32-body tiles of the SMPL-X vertex kernel, single-face / no-face collision queries,
and the argument errors the C ABI reports.  The reference never sees an empty batch on its demo path (its DataLoader
drops them); torch modules accept one, so the mirror does too."""
import numpy as np
import pytest
import torch

from oracle import smplx_oracle
from shapy_b200 import synth

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


@pytest.fixture(scope='module')
def env():
    from shapy_b200 import ops
    model = synth.make_smplx()
    packed = ops.SmplxModel({**model, 'use_face_contour': True}, DEV)
    return model, packed, ops


def test_empty_batch_smplx_and_head(env):
    _, packed, ops = env
    z = lambda *s: torch.zeros(*s, device=DEV)  # noqa: E731
    assert ops.decode_rot6d(z(0, 132)).shape == (0, 22, 3, 3)
    out = ops.smplx_forward(packed, z(0, 10), z(0, 22, 3, 3), camera=z(0, 3))
    assert out['vertices'].shape == (0, packed.V, 3) and out['v_shaped'].shape == (0, packed.V, 3)
    assert out['joints'].shape == (0, packed.K, 3) and out['proj_joints'].shape == (0, packed.K, 2)
    assert ops.smplx_forward_shape(packed, z(0, 10)).shape == (0, packed.V, 3)
    W0, b0, W1, b1, W2, b2 = z(16, 8 + 5), z(16), z(16, 16), z(16), z(5, 16), z(5)
    assert ops.head_forward(z(0, 8), W0, b0, W1, b1, W2, b2, z(5)).shape == (3, 0, 5)


def test_empty_batch_measure_and_collisions(env, golden_dir):
    import os
    model, packed, ops = env
    lm = ops.make_landmarks(synth.load_landmarks())
    faces = torch.from_numpy(np.load(os.path.join(golden_dir, 'img00_body.npz'))['faces']).to(DEV)
    out = ops.measure(lm, torch.zeros(0, packed.V, 3, device=DEV), faces)
    assert out.shape == (0, 5) and int(out.status.item()) == 0
    out, pts, cnt, status = ops.measure(lm, torch.zeros(0, packed.V, 3, device=DEV), faces, return_points=True)
    assert pts.shape[0] == 0 and cnt.shape == (0, 3)
    q = torch.zeros(0, 4, 3, 3, device=DEV)
    f, b = ops.mesh_to_mesh_forward(q, torch.zeros(0, 7, 3, 3, device=DEV), max_collisions=8)
    assert f.shape == (0, 32) and f.dtype == torch.int64 and b.shape == (0, 32, 2, 3)
    # a target without faces: every slot reports "no collision"
    f, b = ops.mesh_to_mesh_forward(torch.rand(2, 4, 3, 3, device=DEV), torch.zeros(2, 0, 3, 3, device=DEV), max_collisions=8)
    assert bool((f == -1).all()) and float(b.abs().max()) == 0.0


def test_empty_batch_backbone_attributes_metrics():
    from shapy_b200 import attributes, metrics
    reg = synth.build_synthetic_regressor().to(DEV).eval()
    feats = reg.backbone(torch.zeros(0, 3, 224, 224, device=DEV))[reg.feature_key]
    assert feats.shape[0] == 0 and feats.dim() == 2
    with pytest.raises(RuntimeError, match='multiple of 32'):
        reg.backbone(torch.zeros(1, 3, 200, 224, device=DEV))
    m, f = attributes.B2A(10, 15), attributes.B2A(10, 15)
    out = attributes.b2a_forward(torch.zeros(0, 10, device=DEV), torch.zeros(0, dtype=torch.int32, device=DEV), m, f)
    assert out.shape == (0, 15)
    pe = metrics.PointError(metrics.build_alignment('translation'))
    err = pe(torch.zeros(0, 100, 3, device=DEV), torch.zeros(0, 100, 3, device=DEV))
    assert err.shape == (0, 100)


@pytest.mark.parametrize('B', [31, 32, 64, 65, 97])
def test_lbs_group_boundaries_vs_oracle(env, B):
    """The vertex kernel works on tiles of 32 bodies; every row of a batch that ends just before / on / after a
    group boundary must match the oracle, and must not depend on what else is in the batch."""
    model, packed, ops = env
    g = torch.Generator().manual_seed(100 + B)
    betas = torch.randn(B, 10, generator=g) * 1.5
    raw = torch.randn(B, 132, generator=g) * 0.4 + synth.mean_params()[:132]
    grot, bpose = smplx_oracle.decode_6d(raw[:, :6]), smplx_oracle.decode_6d(raw[:, 6:])
    rot = torch.cat([grot, bpose], 1).to(DEV)
    out = ops.smplx_forward(packed, betas.to(DEV), rot)
    rows = sorted({0, B // 2, B - 1, min(31, B - 1), min(32, B - 1)})
    ref = smplx_oracle.smplx_forward(model, betas[rows], grot[rows], bpose[rows])
    for k in ('vertices', 'v_shaped', 'joints'):
        a, b = out[k][rows].double().cpu(), torch.as_tensor(ref[k]).double()
        assert float((a - b).abs().max()) <= 1e-4 * float(b.abs().max()), k
    # the same bodies alone give bit-identical rows (no cross-body term, deterministic summation order)
    alone = ops.smplx_forward(packed, betas[rows].to(DEV), rot[rows])
    for k in ('vertices', 'v_shaped', 'joints'):
        assert torch.equal(alone[k], out[k][rows]), k


def test_c_abi_argument_errors(env):
    """The C ABI reports bad arguments through its return code and message (no CUDA error, no crash)."""
    import ctypes as C
    from shapy_b200 import _lib
    _, packed, ops = env
    L = _lib.lib()
    rc = L.shapy_smplx_forward(packed.handle, None, None, 22, None, None, 4, None, None, None, None, None, 0, None)
    assert rc != 0 and b'null' in L.shapy_last_error()
    b = torch.zeros(4, 10, device=DEV)
    r = torch.zeros(4, 22, 3, 3, device=DEV)
    rc = L.shapy_smplx_forward(packed.handle, _lib.ptr(b), _lib.ptr(r), 22, None, None, 0, None, None, None, None, None, 0, None)
    assert rc != 0 and b'batch' in L.shapy_last_error()
    rc = L.shapy_smplx_forward(packed.handle, _lib.ptr(b), _lib.ptr(r), 99, None, None, 4, None, None, None, None, None, 0, None)
    assert rc != 0 and b'n_rot' in L.shapy_last_error()
    with pytest.raises(RuntimeError, match='betas must be'):
        ops.smplx_forward(packed, torch.zeros(4, 9, device=DEV), r)
    with pytest.raises(RuntimeError, match='CUDA tensor'):
        ops.smplx_forward(packed, torch.zeros(4, 10), r)
