"""Times the perspective 2D keypoint Levenberg-Marquardt step against the weak-perspective one on the seeded synthetic
SMPL-X.

    python tools/fit_kp2d_persp_lm_bench.py [--reps 5] [--out fit_kp2d_persp_lm_bench.json]

Per batch size (64 and 4096 bodies), n_rot = 22, with CUDA events, arms alternating within every rep, [min, max] over
the reps of the mean time per call (microseconds), Geman-McClure loss, pose and betas priors on, later steps:
  kp2d_step / kp2dm_step      shapy_fit_lm_keypoints_2d_step / _measurements_step (weak perspective)
  persp_step / perspm_step    shapy_fit_lm_keypoints_2d_perspective_step / _measurements_step
  *_iter                      one LM iteration: keypoint Jacobian + step (+ forward_shape and the measurement
                              Jacobian with measurements)
The card's name, power limit and SM clocks are read in the same run; nothing is set.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.fit_kp2d_lm_bench import _us, clocks  # noqa: E402
from tools.fit_kp_meas_lm_bench import _model  # noqa: E402
from tools.fit_lm_bench import card, time_arms  # noqa: E402

NAMES = ('mass', 'height', 'chest', 'waist', 'hips')


def kernels(B, reps, module, bm):
    from shapy_b200 import ops, synth
    from shapy_b200.fit import LM_DOWN, LM_UP, _measurement_terms, _project
    packed, faces, lm = module.packed(), module.faces_i32, bm.landmarks()
    gen = torch.Generator().manual_seed(B)
    raw = (synth.mean_params()[:132] + 0.3 * torch.randn(B, 132, generator=gen)).cuda()
    rot = ops.decode_rot6d(raw)
    betas = torch.randn(B, 10, generator=gen).clamp(-2, 2).cuda()
    cam = torch.tensor([1.0, 0.0, 0.0], device='cuda').repeat(B, 1)
    tr = torch.tensor([0.0, 0.2, 3.0], device='cuda').repeat(B, 1)
    intr = torch.tensor([1000.0, 500.0, 500.0], device='cuda').repeat(B, 1)
    K = packed.K
    kp, jac = ops.smplx_keypoint_jacobian(packed, betas, rot)
    ops.face_incidence(faces)
    meas, mjac, _ = ops.measure_jacobian_betas(packed, lm, ops.smplx_forward_shape(packed, betas), faces)
    noise = torch.randn(B, K, 2, generator=gen).cuda()
    tgw = (torch.nn.functional.softplus(cam[:, :1, None]) * kp[..., :2] + 0.01 * noise).contiguous()
    tgp = (_project(kp + tr[:, None], intr) + 2.0 * noise).contiguous()
    mt, mw = _measurement_terms({k: (meas[:, i] * 1.01).contiguous() for i, k in enumerate(NAMES)}, None, B, 'cuda')
    mt, mw = mt.contiguous(), mw.contiguous()
    w = torch.ones(B, K, device='cuda')
    anchor = rot.clone()

    def fresh(last, x, with_meas):
        s = {'rot': rot.clone(), 'betas': betas.clone(), last: x.clone(), 'keypoints': kp.clone(), 'jac': jac.clone(),
             'loss': torch.zeros(B, device='cuda'), 'lambda': torch.ones(B, device='cuda'),
             'accepted': torch.zeros(B, dtype=torch.int32, device='cuda')}
        if with_meas:
            s.update(meas=meas.clone(), meas_jac=mjac.clone())
        return s, {'rot': rot.clone(), 'betas': betas.clone(), last: x.clone()}

    st = {('w', m): fresh('camera', cam, m) for m in (False, True)}
    st.update({('p', m): fresh('transl', tr, m) for m in (False, True)})

    def step(kind, with_meas, k=kp, j=jac, m=meas, mj=mjac):
        s, t = st[kind, with_meas]
        if kind == 'w':
            head, terms = (s, t, tgw, w), (0.05, 1.0, 0.01)
            fn = ops.fit_lm_keypoints_2d_measurements_step if with_meas else ops.fit_lm_keypoints_2d_step
        else:
            head, terms = (s, t, tgp, w, intr), (10.0, 1.0, 0.01)
            fn = (ops.fit_lm_keypoints_2d_perspective_measurements_step if with_meas else
                  ops.fit_lm_keypoints_2d_perspective_step)
        if with_meas:
            fn(*head, *terms, mt, mw, LM_UP, LM_DOWN, False, k, j, m, mj, pose_anchor=anchor)
        else:
            fn(*head, *terms, LM_UP, LM_DOWN, False, k, j, pose_anchor=anchor)

    def iteration(kind, with_meas):
        t = st[kind, with_meas][1]
        k, j = ops.smplx_keypoint_jacobian(packed, t['betas'], t['rot'])
        if with_meas:
            m, mj, _ = ops.measure_jacobian_betas(packed, lm, ops.smplx_forward_shape(packed, t['betas']), faces)
            step(kind, True, k, j, m, mj)
        else:
            step(kind, False, k, j)

    arms = {}
    for kind, name in (('w', 'kp2d'), ('p', 'persp')):
        for m in (False, True):
            n = name + ('m' if m else '')
            arms[n + '_step'] = lambda kind=kind, m=m: step(kind, m)
            arms[n + '_iter'] = lambda kind=kind, m=m: iteration(kind, m)
    t = time_arms(arms, 20 if B <= 64 else 3, reps)
    return {'B': B, 'us': _us(t)}


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--reps', type=int, default=5)
    p.add_argument('--out', default=None)
    a = p.parse_args()
    module, bm = _model()
    res = {'card': card(), 'clocks_before': clocks(), 'kernels': [kernels(B, a.reps, module, bm) for B in (64, 4096)],
           'clocks_after': clocks()}
    s = json.dumps(res)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(s + '\n')


if __name__ == '__main__':
    main()
