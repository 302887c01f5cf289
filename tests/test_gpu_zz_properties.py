"""Size-independent properties of the posed SMPL-X path at BASELINE's config-4 batch (4 096 bodies, 128 body tiles of the
SMPL-X vertex kernel), where the oracle is too slow to run:
  * with the rotations fixed, lbs() is affine in the shape coefficients (joints, transforms and posed vertices all are),
  * a rotation applied in front of the global orientation rotates every vertex and joint about the pelvis joint
    (the pelvis transform multiplies every chain from the left; lbs.py:242-295)."""
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
    return model, ops.SmplxModel({**model, 'use_face_contour': True}, DEV), ops


def _rots(g, n):
    raw = torch.randn(n, 132, generator=g) * 0.4 + synth.mean_params()[:132]
    return torch.cat([smplx_oracle.decode_6d(raw[:, :6]), smplx_oracle.decode_6d(raw[:, 6:])], 1)   # (n, 22, 3, 3)


def test_posed_vertices_are_affine_in_beta_at_4096_bodies(env):
    _, packed, ops = env
    g = torch.Generator().manual_seed(11)
    K = 1024
    rot = _rots(g, K)
    b1, b2 = torch.randn(K, 10, generator=g), torch.randn(K, 10, generator=g)
    betas = torch.cat([b1, b2, b1 + b2, torch.zeros(K, 10)], 0).to(DEV)
    out = ops.smplx_forward(packed, betas, torch.cat([rot] * 4, 0).to(DEV))
    for k in ('vertices', 'joints', 'v_shaped'):
        x = out[k].double()
        lhs, rhs = x[2 * K:3 * K], x[:K] + x[K:2 * K] - x[3 * K:]
        assert float((lhs - rhs).abs().max()) < 2e-5, k
    assert bool(torch.isfinite(out['vertices']).all())


def test_global_rotation_equivariance(env):
    _, packed, ops = env
    g = torch.Generator().manual_seed(12)
    B = 256
    rot = _rots(g, B)
    betas = torch.randn(B, 10, generator=g)
    R0 = smplx_oracle.decode_6d(torch.randn(B, 6, generator=g)).view(B, 3, 3)
    rot2 = rot.clone()
    rot2[:, 0] = R0 @ rot[:, 0]
    a = ops.smplx_forward(packed, betas.to(DEV), rot.to(DEV))
    b = ops.smplx_forward(packed, betas.to(DEV), rot2.to(DEV))
    J0 = a['joints'][:, :1].double()                       # the pelvis joint does not move
    assert float((b['joints'][:, :1].double() - J0).abs().max()) < 1e-6
    R = R0.to(DEV).double()
    n_chain = 55                                           # posed chain joints; the landmark entries that follow are vertex sums
    for k, n in (('vertices', None), ('joints', n_chain)):
        x, y = a[k].double()[:, :n], b[k].double()[:, :n]
        want = torch.einsum('bij,bnj->bni', R, x - J0) + J0
        assert float((y - want).abs().max()) < 2e-5, k
    assert torch.equal(a['v_shaped'], b['v_shaped'])       # the T-pose output does not see the pose at all
