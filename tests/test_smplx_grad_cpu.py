"""CPU: the differentiable float64 forward of tests/smplx_grad_ref.py gives the gradients of the reference's own SMPL-X
forward under autograd (tests/golden/ref_smplx_grad.npz, written by tools/make_golden.py from the reference's lbs()),
for betas, expression, every pose rotation, transl and camera, and the same values as the float64 oracle
(oracle.smplx_oracle.smplx_forward_full)."""
import os

import numpy as np
import torch

from oracle import smplx_oracle
from shapy_b200 import synth
from smplx_grad_ref import LEAVES, forward_differentiable, oracle_grads, pattern

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'ref_smplx_grad.npz')


def golden_case():
    g = np.load(GOLDEN)
    model = synth.make_smplx(dtype=torch.float64)
    B, V, K = g['betas'].shape[0], model['v_template'].shape[0], 123
    cot = {k: pattern(g, k, (B, V, 3) if k in ('vertices', 'v_shaped') else (B, K, 2 if k == 'proj_joints' else 3))
           for k in ('vertices', 'joints', 'v_shaped', 'proj_joints')}
    return g, model, cot


def test_oracle_gradients_equal_the_reference_autograd():
    g, model, cot = golden_case()
    grads, _ = oracle_grads(model, cot, g['betas'], g['rot'], expression=g['expression'], transl=g['transl'],
                            camera=g['camera'])
    for k in LEAVES:
        ref = torch.from_numpy(g[f'grad_{k}'])
        got = grads[k]
        assert ref.shape == got.shape, k
        for b in range(ref.shape[0]):
            scale = float(ref[b].abs().max())
            assert scale > 0, (k, b)
            assert float((got[b] - ref[b]).abs().max()) <= 1e-10 * scale, (k, b)
    # the fixture exercises both ends of the dynamic-contour LUT and the camera past softplus' threshold
    assert g['camera'][:, 0].max() > 20 and g['camera'][:, 0].min() < 20


def test_differentiable_forward_equals_the_oracle():
    g, model, _ = golden_case()
    betas, rot, expr = (torch.from_numpy(g[k]) for k in ('betas', 'rot', 'expression'))
    for contour in (True, False):
        ref = smplx_oracle.smplx_forward_full(model, betas, rot, expression=expr, use_face_contour=contour)
        out = forward_differentiable(model, betas.clone().requires_grad_(True), rot, expression=expr,
                                     use_face_contour=contour)
        assert out['vertices'].requires_grad
        for k in ('vertices', 'joints', 'v_shaped'):
            assert torch.equal(out[k].detach(), ref[k]), (k, contour)
