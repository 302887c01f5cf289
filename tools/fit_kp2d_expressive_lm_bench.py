"""Times the whole-body 2D keypoint Levenberg-Marquardt pieces against the 22-joint ones on the seeded synthetic
SMPL-X (weak-perspective camera, Geman-McClure loss, pose and betas priors on, later steps).

    python tools/fit_kp2d_expressive_lm_bench.py [--reps 5] [--out fit_kp2d_expressive_lm_bench.json]

Per batch size (64 and 4096 bodies), with CUDA events, arms alternating within every rep, [min, max] over the reps of
the mean time per call (microseconds):
  jac_79 / jac_188        shapy_smplx_keypoint_jacobian at n_rot = 22 (P = 79) / _expr at n_rot = 55, NE = 10 (P = 188)
  kp2d_step_79            shapy_fit_lm_keypoints_2d_step at P = 79
  wide_step_79            shapy_fit_lm_keypoints_2d_expressive_step on the same P = 79 problem: both entries run the
                          one single-image 2D step kernel, so the two arms time the same kernel through two entries
  wide_step_188           shapy_fit_lm_keypoints_2d_expressive_step at P = 188
  iter_79 / iter_188      one LM iteration (Jacobian + step) at P = 79 / at P = 188
The card's name, power limit and SM clocks are read in the same run; nothing is set.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.fit_kp2d_lm_bench import _us, clocks  # noqa: E402
from tools.fit_lm_bench import card, time_arms  # noqa: E402


def kernels(B, reps, packed):
    from shapy_b200 import ops, synth
    from shapy_b200.fit import LM_DOWN, LM_UP
    gen = torch.Generator().manual_seed(B)
    ident = torch.tensor([1.0, 0.0, 0.0, 1.0, 0.0, 0.0])
    raw = torch.cat([synth.mean_params()[:132] + 0.3 * torch.randn(B, 132, generator=gen),
                     ident.repeat(B, 33) + 0.2 * torch.randn(B, 198, generator=gen)], 1).cuda()
    rot55 = ops.decode_rot6d(raw).contiguous()
    rot22 = rot55[:, :22].contiguous()
    betas = torch.randn(B, 10, generator=gen).clamp(-2, 2).cuda()
    expr = torch.randn(B, 10, generator=gen).cuda()
    cam = torch.tensor([1.0, 0.0, 0.0], device='cuda').repeat(B, 1)
    kp22, jac22 = ops.smplx_keypoint_jacobian(packed, betas, rot22)
    kp55, jac55 = ops.smplx_keypoint_jacobian(packed, betas, rot55, expr=expr)
    K = packed.K
    noise = torch.randn(B, K, 2, generator=gen).cuda()
    s0 = torch.nn.functional.softplus(cam[:, :1, None])
    tg22 = (s0 * kp22[..., :2] + 0.01 * noise).contiguous()
    tg55 = (s0 * kp55[..., :2] + 0.01 * noise).contiguous()
    w = torch.ones(B, K, device='cuda')

    def fresh(rot, kp, jac, ne):
        s = {'rot': rot.clone(), 'betas': betas.clone(), 'camera': cam.clone(), 'keypoints': kp.clone(),
             'jac': jac.clone(), 'loss': torch.zeros(B, device='cuda'), 'lambda': torch.ones(B, device='cuda'),
             'accepted': torch.zeros(B, dtype=torch.int32, device='cuda'), 'expression': expr[:, :ne].clone()}
        t = {'rot': rot.clone(), 'betas': betas.clone(), 'camera': cam.clone(), 'expression': expr[:, :ne].clone()}
        return s, t

    st = {'kp2d79': fresh(rot22, kp22, jac22, 0), 'wide79': fresh(rot22, kp22, jac22, 0),
          'wide188': fresh(rot55, kp55, jac55, 10)}
    terms = (0.05, 1.0, 0.01)

    def step(name, k, j):
        s, t = st[name]
        if name == 'kp2d79':
            ops.fit_lm_keypoints_2d_step(s, t, tg22, w, *terms, LM_UP, LM_DOWN, False, k, j, pose_anchor=s['rot'])
        else:
            tg = tg22 if name == 'wide79' else tg55
            ops.fit_lm_keypoints_2d_expressive_step(s, t, tg, w, *terms, 0.001, LM_UP, LM_DOWN, False, k, j,
                                                    pose_anchor=s['rot'])

    def iteration(name):
        t = st[name][1]
        if name == 'wide188':
            k, j = ops.smplx_keypoint_jacobian(packed, t['betas'], t['rot'], expr=t['expression'])
        else:
            k, j = ops.smplx_keypoint_jacobian(packed, t['betas'], t['rot'])
        step(name, k, j)

    arms = {'jac_79': lambda: ops.smplx_keypoint_jacobian(packed, betas, rot22),
            'jac_188': lambda: ops.smplx_keypoint_jacobian(packed, betas, rot55, expr=expr),
            'kp2d_step_79': lambda: step('kp2d79', kp22, jac22),
            'wide_step_79': lambda: step('wide79', kp22, jac22),
            'wide_step_188': lambda: step('wide188', kp55, jac55),
            'iter_79': lambda: iteration('kp2d79'),
            'iter_188': lambda: iteration('wide188')}
    t = time_arms(arms, 20 if B <= 64 else 3, reps)
    return {'B': B, 'us': _us(t)}


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--reps', type=int, default=5)
    p.add_argument('--out', default=None)
    a = p.parse_args()
    from shapy_b200 import ops, synth
    packed = ops.SmplxModel(dict(synth.make_smplx()), 'cuda')
    res = {'card': card(), 'clocks_before': clocks(), 'kernels': [kernels(B, a.reps, packed) for B in (64, 4096)],
           'clocks_after': clocks()}
    s = json.dumps(res)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(s + '\n')


if __name__ == '__main__':
    main()
