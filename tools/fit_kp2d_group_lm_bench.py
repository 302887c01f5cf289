"""Times the grouped 2D keypoint Levenberg-Marquardt fit (one betas per group of images) on the seeded synthetic SMPL-X.

    python tools/fit_kp2d_group_lm_bench.py [--reps 5] [--out fit_kp2d_group_lm_bench.json]

Per batch size (64 and 4096 images), n_rot = 22, with CUDA events, arms alternating within every rep, [min, max] over
the reps of the mean time per call (microseconds), Geman-McClure loss, pose and betas priors on, later steps:
  kp2d_step      shapy_fit_lm_keypoints_2d_step (one betas per image)
  g{n}_step      shapy_fit_lm_keypoints_2d_groups_step with groups of n = 1, 4, 16 images (three launches)
  kp2d_iter      one 2D LM iteration: keypoint Jacobian + step
  g{n}_iter      one grouped LM iteration: keypoint Jacobian + the grouped step
Then the time to quality of 50 LM iterations on the 64 identities x 4 views of tests/test_gpu_fit_lm_kp2d_groups.py:
per image and grouped, with and without known height and mass.  The card's name, power limit and SM clocks are read in
the same run; nothing is set.
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests'))
from tools.fit_kp2d_lm_bench import _us, clocks  # noqa: E402
from tools.fit_kp_meas_lm_bench import _model  # noqa: E402
from tools.fit_lm_bench import card, time_arms  # noqa: E402

GROUP_SIZES = (1, 4, 16)


def kernels(B, reps, module):
    from shapy_b200 import ops, synth
    from shapy_b200.fit import LM_DOWN, LM_UP
    packed = module.packed()
    gen = torch.Generator().manual_seed(B)
    raw = (synth.mean_params()[:132] + 0.3 * torch.randn(B, 132, generator=gen)).cuda()
    rot = ops.decode_rot6d(raw)
    betas = torch.randn(B, 10, generator=gen).clamp(-2, 2).cuda()
    cam = torch.tensor([1.0, 0.0, 0.0], device='cuda').repeat(B, 1)
    K = packed.K
    kp, jac = ops.smplx_keypoint_jacobian(packed, betas, rot)
    tg = (torch.nn.functional.softplus(cam[:, :1, None]) * kp[..., :2] +
          0.01 * torch.randn(B, K, 2, generator=gen).cuda()).contiguous()
    w = torch.ones(B, K, device='cuda')
    anchor = rot.clone()
    sigma, pw, bw = 0.05, 1.0, 0.01
    ks = {'rot': rot.clone(), 'betas': betas.clone(), 'camera': cam.clone(), 'keypoints': kp.clone(),
          'jac': jac.clone(), 'loss': torch.zeros(B, device='cuda'), 'lambda': torch.ones(B, device='cuda'),
          'accepted': torch.zeros(B, dtype=torch.int32, device='cuda')}
    kt = {'rot': rot.clone(), 'betas': betas.clone(), 'camera': cam.clone()}

    def step2(k=kp, j=jac):
        ops.fit_lm_keypoints_2d_step(ks, kt, tg, w, sigma, pw, bw, LM_UP, LM_DOWN, False, k, j, pose_anchor=anchor)

    def iter2():
        step2(*ops.smplx_keypoint_jacobian(packed, kt['betas'], kt['rot']))

    arms = {'kp2d_step': step2, 'kp2d_iter': iter2}
    for n in GROUP_SIZES:
        G = B // n
        off = torch.arange(0, B + 1, n, dtype=torch.int32)
        gb = betas[::n].contiguous()
        gs = dict(ks, betas=gb.clone(), loss=torch.zeros(G, device='cuda'),
                  accepted=torch.zeros(G, dtype=torch.int32, device='cuda'), **{'lambda': torch.ones(G, device='cuda')})
        gt = {'rot': rot.clone(), 'betas': gb.clone(), 'image_betas': gb.repeat_interleave(n, 0).contiguous(),
              'camera': cam.clone()}
        ws = ops.fit_lm_groups_workspace(B, G, 22, 10, 'cuda')

        def stepg(k=kp, j=jac, gs=gs, gt=gt, off=off, ws=ws):
            ops.fit_lm_keypoints_2d_groups_step(gs, gt, tg, w, sigma, pw, bw, LM_UP, LM_DOWN, False, k, j, off, ws,
                                                pose_anchor=anchor)

        def iterg(stepg=stepg, gt=gt):
            stepg(*ops.smplx_keypoint_jacobian(packed, gt['image_betas'], gt['rot']))

        arms[f'g{n}_step'], arms[f'g{n}_iter'] = stepg, iterg
    t = time_arms(arms, 20 if B <= 64 else 3, reps)
    return {'B': B, 'us': _us(t)}


def time_to_quality(module, bm):
    from shapy_b200.fit import fit_body_to_keypoints_2d
    from lm_harness import quality_groups as quality
    from test_gpu_fit_lm_kp2d_groups import _problem
    p = _problem(module, bm, 64)
    gm = {k: p['tg'][k] for k in ('height', 'mass')}
    arms = (('per_image_lm_50', {}, False),
            ('grouped_lm_50', dict(groups=p['groups']), True),
            ('per_image_height_mass_lm_50', dict(body_measurements=bm,
                                                 measurements={k: v[p['groups']] for k, v in gm.items()}), False),
            ('grouped_height_mass_lm_50', dict(groups=p['groups'], body_measurements=bm, measurements=gm), True))
    out = {}
    for name, kw, grouped in arms:
        fit_body_to_keypoints_2d(module, p['x'], init=p['init'], method='lm', iterations=2, **kw)    # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = fit_body_to_keypoints_2d(module, p['x'], init=p['init'], method='lm', **kw)
        torch.cuda.synchronize()
        sec = time.perf_counter() - t0
        q = quality(module, bm, p, res, grouped)
        out[name] = {'seconds': round(sec, 4), **{k: round(v, 4) for k, v in q.items()}}
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--reps', type=int, default=5)
    p.add_argument('--out', default=None)
    a = p.parse_args()
    module, bm = _model()
    res = {'card': card(), 'clocks_before': clocks(), 'kernels': [kernels(B, a.reps, module) for B in (64, 4096)],
           'time_to_quality': time_to_quality(module, bm), 'clocks_after': clocks()}
    s = json.dumps(res)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(s + '\n')


if __name__ == '__main__':
    main()
