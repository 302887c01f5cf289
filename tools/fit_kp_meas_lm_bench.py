"""Times the stacked keypoint + measurement Levenberg-Marquardt fit on the seeded synthetic SMPL-X model.

    python tools/fit_kp_meas_lm_bench.py [--reps 5] [--out fit_kp_meas_lm_bench.json]

Per batch size (64 and 4096 bodies), n_rot = 22, with CUDA events, arms alternating within every rep, [min, max] over
the reps of the mean time per call (microseconds):
  kp_step        shapy_fit_lm_keypoints_step
  kpm_step       shapy_fit_lm_keypoints_measurements_step (same keypoints, plus the five measurements and rho)
  kp_iter        one keypoint-only LM iteration: keypoint Jacobian + step
  kpm_iter       one stacked LM iteration: keypoint Jacobian, forward_shape, measurement Jacobian, step
Then the time to quality of 50 LM iterations, keypoint-only against keypoints + known height and mass and against
keypoints + all five measurements (default weights), on the 256 bodies of tests/test_gpu_fit_lm_kp_meas.py (seed 31,
mean-pose start) for both keypoint sets (all keypoints; only the 22 posed body joints): wall time, the share within
1 cm keypoint RMS, the measurement shares (height < 1 mm, every circumference < 0.5 %, mass < 1 %) and the median
|beta - beta*|.  The card's name, power limit and max SM clock are
read in the same run.
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.fit_lm_bench import card, time_arms  # noqa: E402

NAMES = ('mass', 'height', 'chest', 'waist', 'hips')


def _us(t):
    return {k: [round(v[0] * 1e3, 1), round(v[1] * 1e3, 1)] for k, v in t.items()}


def _model():
    from shapy_b200 import synth
    from shapy_b200.body_measurements import BodyMeasurements
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    return (SMPLX(data_struct=synth.make_smplx(), use_face_contour=True).cuda(),
            BodyMeasurements({'landmarks': synth.load_landmarks()}).cuda())


def kernels(B, reps, module, bm):
    from shapy_b200 import ops, synth
    from shapy_b200.fit import LM_DOWN, LM_UP, _measurement_terms
    packed, faces, lm = module.packed(), module.faces_i32, bm.landmarks()
    gen = torch.Generator().manual_seed(B)
    raw = (synth.mean_params()[:132] + 0.3 * torch.randn(B, 132, generator=gen)).cuda()
    rot = ops.decode_rot6d(raw)
    betas = torch.randn(B, 10, generator=gen).clamp(-2, 2).cuda()
    transl = torch.zeros(B, 3, device='cuda')
    K = packed.K
    kp, jac = ops.smplx_keypoint_jacobian(packed, betas, rot, transl)
    ops.face_incidence(faces)
    meas, mjac, _ = ops.measure_jacobian_betas(packed, lm, ops.smplx_forward_shape(packed, betas), faces)
    tg = (kp + 0.01 * torch.randn(B, K, 3, generator=gen).cuda()).contiguous()
    mt, mw = _measurement_terms({k: (meas[:, i] * 1.01).contiguous() for i, k in enumerate(NAMES)}, None, B, 'cuda')
    w = torch.ones(B, K, device='cuda')
    rho = 0.01

    def fresh(with_meas):
        s = {'rot': rot.clone(), 'betas': betas.clone(), 'transl': transl.clone(), 'keypoints': kp.clone(),
             'jac': jac.clone(), 'loss': torch.zeros(B, device='cuda'), 'lambda': torch.ones(B, device='cuda'),
             'accepted': torch.zeros(B, dtype=torch.int32, device='cuda')}
        if with_meas:
            s.update(meas=meas.clone(), meas_jac=mjac.clone())
        return s, {'rot': rot.clone(), 'betas': betas.clone(), 'transl': transl.clone()}

    (ks, kt), (ms, mtr) = fresh(False), fresh(True)

    def kp_step():
        ops.fit_lm_keypoints_step(ks, kt, tg, w, LM_UP, LM_DOWN, False, kp, jac)

    def kpm_step():
        ops.fit_lm_keypoints_measurements_step(ms, mtr, tg, w, mt, mw, rho, LM_UP, LM_DOWN, False, kp, jac, meas, mjac)

    def kp_iter():
        k, j = ops.smplx_keypoint_jacobian(packed, kt['betas'], kt['rot'], kt['transl'])
        ops.fit_lm_keypoints_step(ks, kt, tg, w, LM_UP, LM_DOWN, False, k, j)

    def kpm_iter():
        k, j = ops.smplx_keypoint_jacobian(packed, mtr['betas'], mtr['rot'], mtr['transl'])
        m, mj, _ = ops.measure_jacobian_betas(packed, lm, ops.smplx_forward_shape(packed, mtr['betas']), faces)
        ops.fit_lm_keypoints_measurements_step(ms, mtr, tg, w, mt, mw, rho, LM_UP, LM_DOWN, False, k, j, m, mj)

    t = time_arms({'kp_step': kp_step, 'kpm_step': kpm_step, 'kp_iter': kp_iter, 'kpm_iter': kpm_iter},
                  20 if B <= 64 else 3, reps)
    return {'B': B, 'us': _us(t)}


def time_to_quality(module, bm):
    from shapy_b200 import ops, synth
    from shapy_b200.fit import fit_body_to_keypoints
    gen = torch.Generator().manual_seed(31)
    bstar = torch.randn(256, 10, generator=gen).clamp(-2, 2).cuda()
    raw = synth.mean_params()[:132] + 0.3 * torch.randn(256, 132, generator=gen)
    with torch.no_grad():
        r = ops.decode_rot6d(raw.cuda())
        kp = module(global_rot=r[:, :1], body_pose=r[:, 1:], betas=bstar)['joints'][:].clone()
        m = bm.forward_vertices(module.forward_shape(betas=bstar)['v_shaped'], module.faces_i32)['measurements']
    tg = {k: m[k]['tensor'].clone() for k in NAMES}
    tgt = torch.stack([tg[k] for k in NAMES], 1)
    ok = torch.isfinite(tgt).all(1)
    mean = synth.mean_params().cuda()
    init = {'global_rot': mean[:6].expand(256, 6), 'body_pose': mean[6:132].expand(256, 126)}
    kw_meas = dict(body_measurements=bm, measurements=tg)
    kw_hm = dict(body_measurements=bm, measurements={k: tg[k] for k in ('height', 'mass')})
    out = {}
    for which in ('all', 'body'):
        w = torch.ones(kp.shape[1], device='cuda')
        if which == 'body':
            w[22:] = 0.0
        for name, kw in (('kp_lm_50', {}), ('kp_height_mass_lm_50', kw_hm), ('kp_meas5_lm_50', kw_meas)):
            fit_body_to_keypoints(module, kp, w, init=init, method='lm', iterations=2, **kw)     # warm-up
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = fit_body_to_keypoints(module, kp, w, init=init, method='lm', **kw)
            torch.cuda.synchronize()
            sec = time.perf_counter() - t0
            with torch.no_grad():
                mm = bm.forward_vertices(module.forward_shape(betas=res['betas'])['v_shaped'],
                                         module.faces_i32)['measurements']
            meas = torch.stack([mm[k]['tensor'] for k in NAMES], 1)
            rms = ((res['keypoints'] - kp).pow(2).sum(-1) * w).sum(1).div(w.sum()).sqrt()
            rel = ((meas - tgt).abs() / tgt.abs())[ok]
            out[f'{which}/{name}'] = {
                'seconds': round(sec, 4), 'median_loss': float(res['loss'].median()),
                'frac_rms_1cm': round(float((rms < 1e-2).float().mean()), 4),
                'height_1mm': round(float(((meas[:, 1] - tgt[:, 1]).abs()[ok] < 1e-3).float().mean()), 4),
                'circ_0.5pct': round(float((rel[:, 2:] < 5e-3).all(1).float().mean()), 4),
                'mass_1pct': round(float((rel[:, 0] < 1e-2).float().mean()), 4),
                'median_beta_err': round(float((res['betas'] - bstar).norm(dim=1).median()), 4)}
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--reps', type=int, default=5)
    p.add_argument('--out', default=None)
    a = p.parse_args()
    module, bm = _model()
    res = {'card': card(), 'kernels': [kernels(B, a.reps, module, bm) for B in (64, 4096)],
           'time_to_quality': time_to_quality(module, bm)}
    s = json.dumps(res)
    print(s)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(s + '\n')


if __name__ == '__main__':
    main()
