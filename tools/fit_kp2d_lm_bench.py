"""Times the Levenberg-Marquardt fit of pose, shape and camera to 2D keypoints on the seeded synthetic SMPL-X model.

    python tools/fit_kp2d_lm_bench.py [--reps 5] [--out fit_kp2d_lm_bench.json]

Per batch size (64 and 4096 bodies), n_rot = 22, with CUDA events, arms alternating within every rep, [min, max] over
the reps of the mean time per call (microseconds):
  step_3d     shapy_fit_lm_keypoints_step (3D keypoints)
  step_2d     shapy_fit_lm_keypoints_2d_step, Geman-McClure loss, pose and betas priors on
  lm_iter_2d  one 2D LM iteration: keypoint Jacobian + 2D step
  adam_iter   one Adam iteration of fit_body_to_keypoints_2d: decoder + forward with the camera, backward, optimiser
Then the time to quality of LM (50 iterations) against Adam (600) on the 256 bodies of
tests/test_gpu_fit_lm_keypoints_2d.py: wall time, median loss, the fraction within 2e-3 2D RMS (crop frame), the
median 2D RMS and the median root-aligned 3D joint error.  The card's name, power limit and SM clocks are read in the
same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests'))
from tools.fit_lm_bench import card, time_arms  # noqa: E402


def _us(t):
    return {k: [round(v[0] * 1e3, 1), round(v[1] * 1e3, 1)] for k, v in t.items()}


def clocks():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=clocks.sm,clocks.max.sm,power.limit', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def kernels(B, reps):
    from shapy_b200 import ops, synth
    from shapy_b200.autograd import Rot6dFunction
    from shapy_b200.fit import LM_DOWN, LM_UP
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    module = SMPLX(data_struct=synth.make_smplx(), use_face_contour=True).cuda()
    packed = module.packed()
    gen = torch.Generator().manual_seed(B)
    raw = (synth.mean_params()[:132] + 0.3 * torch.randn(B, 132, generator=gen)).cuda()
    rot = ops.decode_rot6d(raw)
    betas = torch.randn(B, 10, generator=gen).clamp(-2, 2).cuda()
    transl = torch.zeros(B, 3, device='cuda')
    cam = torch.tensor([1.0, 0.0, 0.0], device='cuda').repeat(B, 1)
    K = packed.K
    kp, jac = ops.smplx_keypoint_jacobian(packed, betas, rot, transl)
    tg = (kp + 0.01 * torch.randn(B, K, 3, generator=gen).cuda()).contiguous()
    tg2 = (torch.nn.functional.softplus(cam[:, :1, None]) * kp[..., :2] +
           0.01 * torch.randn(B, K, 2, generator=gen).cuda()).contiguous()
    w = torch.ones(B, K, device='cuda')
    mk = lambda: {'rot': rot.clone(), 'betas': betas.clone(), 'keypoints': kp.clone(), 'jac': jac.clone(),  # noqa: E731
                  'loss': torch.zeros(B, device='cuda'), 'lambda': torch.ones(B, device='cuda'),
                  'accepted': torch.zeros(B, dtype=torch.int32, device='cuda')}
    s3, s2 = dict(mk(), transl=transl.clone()), dict(mk(), camera=cam.clone())
    t3 = {'rot': rot.clone(), 'betas': betas.clone(), 'transl': transl.clone()}
    t2 = {'rot': rot.clone(), 'betas': betas.clone(), 'camera': cam.clone()}
    anchor = rot.clone()

    def step2():
        ops.fit_lm_keypoints_2d_step(s2, t2, tg2, w, 0.05, 1.0, 0.01, LM_UP, LM_DOWN, False, kp, jac,
                                     pose_anchor=anchor)

    def iter2():
        k, j = ops.smplx_keypoint_jacobian(packed, t2['betas'], t2['rot'])
        ops.fit_lm_keypoints_2d_step(s2, t2, tg2, w, 0.05, 1.0, 0.01, LM_UP, LM_DOWN, False, k, j, pose_anchor=anchor)

    params = {'r': raw.clone().requires_grad_(True), 'b': betas.clone().requires_grad_(True),
              'c': cam.clone().requires_grad_(True)}
    opt = torch.optim.Adam(list(params.values()), lr=0.05)

    def adam():                                    # the body of fit_body_to_keypoints_2d's Adam loop, least squares
        opt.zero_grad(set_to_none=True)
        r = Rot6dFunction.apply(params['r'])
        out = module(global_rot=r[:, :1], body_pose=r[:, 1:], betas=params['b'], camera=params['c'],
                     return_shaped=False)
        ((out['proj_joints'] - tg2).pow(2).sum(-1) * w).sum().backward()
        opt.step()

    arms = {'step_3d': lambda: ops.fit_lm_keypoints_step(s3, t3, tg, w, LM_UP, LM_DOWN, False, kp, jac),
            'step_2d': step2, 'lm_iter_2d': iter2, 'adam_iter': adam}
    return {'B': B, 'us': _us(time_arms(arms, 20 if B <= 64 else 3, reps))}


def time_to_quality():
    from shapy_b200.fit import fit_body_to_keypoints_2d
    from shapy_b200.metrics import PointError, build_alignment
    from lm_harness import smplx_module
    from test_gpu_fit_lm_keypoints_2d import RMS_THRESHOLD, _problem, _rms2d
    module = smplx_module()
    x, joints, init = _problem(module, 256)
    for m in ('lm', 'adam'):                                     # warm-up
        fit_body_to_keypoints_2d(module, x, init=init, method=m, iterations=2)
    pe = PointError(build_alignment('root'))
    out = {}
    for name, kw in (('lm_50', dict(method='lm')), ('adam_600', dict(method='adam'))):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = fit_body_to_keypoints_2d(module, x, init=init, **kw)
        torch.cuda.synchronize()
        sec = time.perf_counter() - t0
        rms = _rms2d(res, x)
        pe(res['keypoints'].contiguous(), joints)
        out[name] = {'seconds': round(sec, 4), 'median_loss': float(res['loss'].median()),
                     'frac_rms2d': round(float((rms < RMS_THRESHOLD).float().mean()), 4),
                     'median_rms2d': float(rms.median()), 'median_root_mpjpe_m': float(pe.last_mean.median())}
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--reps', type=int, default=5)
    p.add_argument('--out', default=None)
    a = p.parse_args()
    res = {'card': card(), 'clocks_before': clocks(), 'kernels': [kernels(B, a.reps) for B in (64, 4096)],
           'time_to_quality': time_to_quality(), 'clocks_after': clocks()}
    s = json.dumps(res)
    print(s)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(s + '\n')


if __name__ == '__main__':
    main()
