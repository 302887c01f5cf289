"""GPU quality: the silhouette term in the perspective Adam fit on the synthetic SMPL-X.  The perspective recipe of
tests/test_gpu_fit_lm_kp2d_persp.py with 64 bodies (beta*, pose, t* with t_z* in [2, 4] m, f = 1000, pp = (500, 500)),
masks 1000 x 1000 rendered from the true posed mesh by render_silhouette (pinned to the oracle by
tests/test_gpu_silhouette.py), both fits from the recipe's perturbed start for Adam's default iteration count:
(a) keypoints only, (b) keypoints and silhouettes."""
import time

import pytest
import torch

import lm_harness as harness
from test_gpu_fit_lm_kp2d_persp import _problem

pytestmark = pytest.mark.gpu

F, PP = harness.F, harness.PP
B, SIZE = 64, 1000


def run(weight=None, seed=61):
    """{'a': report, 'b': report} of the two fits; weight None is the default silhouette_weight."""
    from shapy_b200 import ops, synth
    from shapy_b200.fit import SILHOUETTE_WEIGHT, fit_body_to_keypoints_2d
    module = harness.smplx_module()
    packed = module.packed()
    x, _, init, tstar, bstar = _problem(module, B, seed=seed)
    intr = torch.tensor([F, *PP]).repeat(B, 1).cuda()
    # the recipe's truth: _problem keeps the true raw pose at mean + 0.3 N(0, 1) before the start's noise
    gen = torch.Generator().manual_seed(seed)
    torch.randn(B, module.num_betas, generator=gen)
    raw_true = synth.mean_params()[:132] + 0.3 * torch.randn(B, 132, generator=gen)
    with torch.no_grad():
        rot = ops.decode_rot6d(raw_true.cuda())
        v_true = module(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=bstar, transl=tstar,
                        return_shaped=False)['vertices'].contiguous()
        masks = ops.render_silhouette(v_true, module.faces_i32, intr, SIZE, SIZE)
        t_true = ops.smplx_forward_shape(packed, bstar)
    kw = dict(focal_length=F, principal_point=PP)
    w = SILHOUETTE_WEIGHT if weight is None else weight
    out = {}
    for name, extra in (('a', {}), ('b', dict(silhouettes=masks, silhouette_weight=w))):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fit_body_to_keypoints_2d(module, x, init=dict(init), **kw, **extra)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        with torch.no_grad():
            v = module(global_rot=r['global_rot_mat'], body_pose=r['body_pose_mat'], betas=r['betas'],
                       transl=r['transl'], return_shaped=False)['vertices'].contiguous()
            rend = ops.render_silhouette(v, module.faces_i32, intr, SIZE, SIZE)
            iou = (rend & masks).sum((1, 2)).float() / (rend | masks).sum((1, 2)).float()
            v2v = (v - v_true).norm(dim=-1).mean(1)
            ts = ops.smplx_forward_shape(packed, r['betas'])
            d = ts - t_true
            tpose = (d - d.mean(1, keepdim=True)).norm(dim=-1).mean(1)
            rms = (r['proj_joints'] - x).pow(2).sum(-1).mean(1).sqrt()
        out[name] = {'iou': float(iou.median()), 'v2v_mm': 1e3 * float(v2v.median()),
                     'tpose_v2v_mm': 1e3 * float(tpose.median()),
                     'beta_err': float((r['betas'] - bstar).norm(dim=1).median()),
                     'rms_px': float(rms.median()), 'wall_s': wall}
        if name == 'b':
            assert torch.allclose(r['silhouette_iou'], iou, atol=0, rtol=0)
            assert bool(torch.isfinite(r['silhouette']).all())
    return out


# First run on an H100 80GB HBM3 (700 W), README "Silhouettes": (a) / (b) median IoU 0.657 / 0.719, posed v2v 380 /
# 299 mm, T-pose v2v 31.2 / 44.7 mm, |beta - beta*| 3.91 / 5.62, 2D RMS 60.4 / 61.8 px.  Bars just past (b)'s.
BARS = {'iou': 0.71, 'v2v_mm': 310.0, 'tpose_v2v_mm': 46.0, 'beta_err': 5.8, 'rms_px': 63.0}


def test_quality_64_bodies_keypoints_vs_keypoints_and_silhouettes():
    rep = run()
    print('fit_silhouette_64', rep)
    b = rep['b']
    assert b['iou'] >= BARS['iou']
    for k in ('v2v_mm', 'tpose_v2v_mm', 'beta_err', 'rms_px'):
        assert b[k] <= BARS[k], (k, b[k])
    assert b['iou'] > rep['a']['iou']
