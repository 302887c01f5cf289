"""Times the stacked 2D keypoint + measurement Levenberg-Marquardt fit on the seeded synthetic SMPL-X model.

    python tools/fit_kp2d_meas_lm_bench.py [--reps 5] [--out fit_kp2d_meas_lm_bench.json]

Per batch size (64 and 4096 bodies), n_rot = 22, with CUDA events, arms alternating within every rep, [min, max] over
the reps of the mean time per call (microseconds), Geman-McClure loss, pose and betas priors on:
  kp2d_step      shapy_fit_lm_keypoints_2d_step
  kp2dm_step     shapy_fit_lm_keypoints_2d_measurements_step (same keypoints, plus the five measurements)
  kp2d_iter      one keypoint-only 2D LM iteration: keypoint Jacobian + step (2 launches)
  kp2dm_iter     one stacked 2D LM iteration: keypoint Jacobian, forward_shape, measurement Jacobian, step (4 launches)
Then the time to quality of 50 LM iterations on the 256 bodies of tests/test_gpu_fit_lm_kp2d_meas.py (seed 41, perturbed
start): keypoints only, + known height and mass, + all five measurements at their default weights with the 'reference'
and the 'exact' circumference rows, for all keypoints and for the 22 posed body joints only: wall time, the shares with
height < 1 mm, mass < 1 %, every circumference < 0.5 % and 2D RMS < 2e-3 (crop frame), the median |beta - beta*| and
the median root-aligned 3D joint error.  The card's name, power limit and SM clocks are read in the same run; nothing
is set.
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
from tools.fit_kp_meas_lm_bench import NAMES, _model  # noqa: E402
from tools.fit_lm_bench import card, time_arms  # noqa: E402


def kernels(B, reps, module, bm):
    from shapy_b200 import ops, synth
    from shapy_b200.fit import LM_DOWN, LM_UP, _measurement_terms
    packed, faces, lm = module.packed(), module.faces_i32, bm.landmarks()
    gen = torch.Generator().manual_seed(B)
    raw = (synth.mean_params()[:132] + 0.3 * torch.randn(B, 132, generator=gen)).cuda()
    rot = ops.decode_rot6d(raw)
    betas = torch.randn(B, 10, generator=gen).clamp(-2, 2).cuda()
    cam = torch.tensor([1.0, 0.0, 0.0], device='cuda').repeat(B, 1)
    K = packed.K
    kp, jac = ops.smplx_keypoint_jacobian(packed, betas, rot)
    ops.face_incidence(faces)
    meas, mjac, _ = ops.measure_jacobian_betas(packed, lm, ops.smplx_forward_shape(packed, betas), faces)
    tg = (torch.nn.functional.softplus(cam[:, :1, None]) * kp[..., :2] +
          0.01 * torch.randn(B, K, 2, generator=gen).cuda()).contiguous()
    mt, mw = _measurement_terms({k: (meas[:, i] * 1.01).contiguous() for i, k in enumerate(NAMES)}, None, B, 'cuda')
    mt, mw = mt.contiguous(), mw.contiguous()
    w = torch.ones(B, K, device='cuda')
    anchor = rot.clone()
    sigma, pw, bw = 0.05, 1.0, 0.01

    def fresh(with_meas):
        s = {'rot': rot.clone(), 'betas': betas.clone(), 'camera': cam.clone(), 'keypoints': kp.clone(),
             'jac': jac.clone(), 'loss': torch.zeros(B, device='cuda'), 'lambda': torch.ones(B, device='cuda'),
             'accepted': torch.zeros(B, dtype=torch.int32, device='cuda')}
        if with_meas:
            s.update(meas=meas.clone(), meas_jac=mjac.clone())
        return s, {'rot': rot.clone(), 'betas': betas.clone(), 'camera': cam.clone()}

    (ks, kt), (ms, mtr) = fresh(False), fresh(True)

    def step2(k=kp, j=jac):
        ops.fit_lm_keypoints_2d_step(ks, kt, tg, w, sigma, pw, bw, LM_UP, LM_DOWN, False, k, j, pose_anchor=anchor)

    def step2m(k=kp, j=jac, m=meas, mj=mjac):
        ops.fit_lm_keypoints_2d_measurements_step(ms, mtr, tg, w, sigma, pw, bw, mt, mw, LM_UP, LM_DOWN, False, k, j,
                                                  m, mj, pose_anchor=anchor)

    def iter2():
        step2(*ops.smplx_keypoint_jacobian(packed, kt['betas'], kt['rot']))

    def iter2m():
        k, j = ops.smplx_keypoint_jacobian(packed, mtr['betas'], mtr['rot'])
        m, mj, _ = ops.measure_jacobian_betas(packed, lm, ops.smplx_forward_shape(packed, mtr['betas']), faces)
        step2m(k, j, m, mj)

    t = time_arms({'kp2d_step': step2, 'kp2dm_step': step2m, 'kp2d_iter': iter2, 'kp2dm_iter': iter2m},
                  20 if B <= 64 else 3, reps)
    return {'B': B, 'us': _us(t)}


def time_to_quality(module, bm):
    from shapy_b200.fit import fit_body_to_keypoints_2d
    from lm_harness import N_ROT, quality_2d as quality
    from test_gpu_fit_lm_kp2d_meas import _problem
    p = _problem(module, bm, 256)
    hm = {k: p['tg'][k] for k in ('height', 'mass')}
    arms = (('kp2d_lm_50', {}),
            ('kp2d_height_mass_lm_50', dict(body_measurements=bm, measurements=hm)),
            ('kp2d_meas5_reference_lm_50', dict(body_measurements=bm, measurements=p['tg'])),
            ('kp2d_meas5_exact_lm_50', dict(body_measurements=bm, measurements=p['tg'],
                                            circumference_derivative='exact')))
    out = {}
    for which in ('all', 'body'):
        w = torch.ones(p['x'].shape[1], device='cuda')
        if which == 'body':
            w[N_ROT:] = 0.0
        for name, kw in arms:
            fit_body_to_keypoints_2d(module, p['x'], w, init=p['init'], method='lm', iterations=2, **kw)   # warm-up
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = fit_body_to_keypoints_2d(module, p['x'], w, init=p['init'], method='lm', **kw)
            torch.cuda.synchronize()
            sec = time.perf_counter() - t0
            q = quality(module, bm, p, res, w)
            fin = torch.isfinite(res['loss'])
            out[f'{which}/{name}'] = {'seconds': round(sec, 4), 'finite_loss': round(float(fin.float().mean()), 4),
                                      'median_loss': float(res['loss'][fin].median()),
                                      **{k: round(v, 4) for k, v in q.items()}}
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--reps', type=int, default=5)
    p.add_argument('--out', default=None)
    a = p.parse_args()
    module, bm = _model()
    res = {'card': card(), 'clocks_before': clocks(), 'kernels': [kernels(B, a.reps, module, bm) for B in (64, 4096)],
           'time_to_quality': time_to_quality(module, bm), 'clocks_after': clocks()}
    s = json.dumps(res)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(s + '\n')


if __name__ == '__main__':
    main()
