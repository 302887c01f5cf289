"""Times the exact circumference derivative against the reference semantics, and measures what it does to the fits.

    python tools/measure_exact_bench.py [--reps 5] [--out measure_exact_bench.json]

On the seeded synthetic SMPL-X model, per batch size (64 and 4096 bodies), with CUDA events, arms alternating within
every rep, [min, max] over the reps of the mean time per call (microseconds):
  jacobian_{reference,exact}   shapy_measure_jacobian_betas[_exact]
  backward_{reference,exact}   the staged (vertex) backward, shapy_measure_backward[_exact], random cotangent
  betas_iter_{reference,exact} one LM iteration of fit_betas_to_measurements (forward_shape, Jacobian, step)
  kpm_iter_{reference,exact}   one LM iteration of fit_body_to_keypoints with measurements (keypoint Jacobian,
                               forward_shape, measurement Jacobian, step)
Then fit quality on 256 bodies, in each mode: LM(50) and Adam(400) of betas to all five measurements (the recipe of
tests/test_gpu_fit_lm.py), and LM(50) and Adam(600) of all keypoints + all five measurements at their default weights
(tests/test_gpu_fit_lm_kp_meas.py), plus the keypoint-only LM for comparison; the README table's columns: wall time,
median loss, share within 1 cm keypoint RMS, height < 1 mm, every circumference < 0.5 %, mass < 1 %, median
|beta - beta*|.  The card's name, power limit and max SM clock are read in the same run.
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
MODES = ('reference', 'exact')


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
    betas = torch.randn(B, 10, generator=gen).clamp(-2, 2).cuda()
    raw = (synth.mean_params()[:132] + 0.3 * torch.randn(B, 132, generator=gen)).cuda()
    rot = ops.decode_rot6d(raw)
    transl = torch.zeros(B, 3, device='cuda')
    v = ops.smplx_forward_shape(packed, betas)
    ops.face_incidence(faces)
    go = torch.randn(B, 5, generator=gen).cuda()
    meas, mjac, _ = ops.measure_jacobian_betas(packed, lm, v, faces)
    mt, mw = _measurement_terms({k: (meas[:, i] * 1.01).contiguous() for i, k in enumerate(NAMES)}, None, B, 'cuda')
    kp, kjac = ops.smplx_keypoint_jacobian(packed, betas, rot, transl)
    K = packed.K
    tg = (kp + 0.01 * torch.randn(B, K, 3, generator=gen).cuda()).contiguous()
    w = torch.ones(B, K, device='cuda')
    arms = {}
    for mode in MODES:
        ex = mode == 'exact'
        bs = {'betas': betas.clone(), 'meas': meas.clone(), 'jac': mjac.clone(), 'loss': torch.zeros(B, device='cuda'),
              'lambda': torch.ones(B, device='cuda'), 'accepted': torch.zeros(B, dtype=torch.int32, device='cuda')}
        btrial = betas.clone()
        ks = {'rot': rot.clone(), 'betas': betas.clone(), 'transl': transl.clone(), 'keypoints': kp.clone(),
              'jac': kjac.clone(), 'loss': torch.zeros(B, device='cuda'), 'lambda': torch.ones(B, device='cuda'),
              'accepted': torch.zeros(B, dtype=torch.int32, device='cuda'), 'meas': meas.clone(),
              'meas_jac': mjac.clone()}
        kt = {'rot': rot.clone(), 'betas': betas.clone(), 'transl': transl.clone()}

        def jacobian(ex=ex):
            ops.measure_jacobian_betas(packed, lm, v, faces, exact=ex)

        def backward(ex=ex):
            ops.measure_backward(lm, go, v_shaped=v, faces_i32=faces, exact=ex)

        def betas_iter(ex=ex, bs=bs, btrial=btrial):
            vt = ops.smplx_forward_shape(packed, btrial)
            m, j, _ = ops.measure_jacobian_betas(packed, lm, vt, faces, exact=ex)
            ops.fit_lm_step(bs, mt, mw, 0.0, LM_UP, LM_DOWN, False, btrial, m, j)

        def kpm_iter(ex=ex, ks=ks, kt=kt):
            k, j = ops.smplx_keypoint_jacobian(packed, kt['betas'], kt['rot'], kt['transl'])
            m, mj, _ = ops.measure_jacobian_betas(packed, lm, ops.smplx_forward_shape(packed, kt['betas']), faces,
                                                  exact=ex)
            ops.fit_lm_keypoints_measurements_step(ks, kt, tg, w, mt, mw, 0.0, LM_UP, LM_DOWN, False, k, j, m, mj)

        arms.update({f'jacobian_{mode}': jacobian, f'backward_{mode}': backward, f'betas_iter_{mode}': betas_iter,
                     f'kpm_iter_{mode}': kpm_iter})
    order = [f'{a}_{m}' for a in ('jacobian', 'backward', 'betas_iter', 'kpm_iter') for m in MODES]
    t = time_arms({k: arms[k] for k in order}, 20 if B <= 64 else 3, reps)
    return {'B': B, 'us': {k: [round(v[0] * 1e3, 1), round(v[1] * 1e3, 1)] for k, v in t.items()}}


def _row(res, meas, tgt, sec, kp=None, bstar=None):
    ok = torch.isfinite(tgt).all(1)
    rel = ((meas - tgt).abs() / tgt.abs())[ok]
    r = {'seconds': round(sec, 4), 'median_loss': float(res['loss'][ok].median()),
         'height_1mm': round(float(((meas[:, 1] - tgt[:, 1]).abs()[ok] < 1e-3).float().mean()), 4),
         'circ_0.5pct': round(float((rel[:, 2:] < 5e-3).all(1).float().mean()), 4),
         'mass_1pct': round(float((rel[:, 0] < 1e-2).float().mean()), 4)}
    if kp is not None:
        rms = (res['keypoints'] - kp).pow(2).sum(-1).mean(1).sqrt()
        r['frac_rms_1cm'] = round(float((rms < 1e-2).float().mean()), 4)
    if bstar is not None:
        r['median_beta_err'] = round(float((res['betas'] - bstar).norm(dim=1).median()), 4)
    return r


def _timed(fn):
    fn(warm=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = fn(warm=False)
    torch.cuda.synchronize()
    return res, time.perf_counter() - t0


def fit_quality(module, bm):
    from shapy_b200 import ops, synth
    from shapy_b200.fit import fit_betas_to_measurements, fit_body_to_keypoints

    def measure(betas):
        with torch.no_grad():
            m = bm.forward_vertices(module.forward_shape(betas=betas)['v_shaped'], module.faces_i32)['measurements']
        return torch.stack([m[k]['tensor'] for k in NAMES], 1)

    out = {}
    bstar = torch.randn(256, 10, generator=torch.Generator().manual_seed(21)).clamp(-2, 2).cuda()
    tgt = measure(bstar)
    tg = {k: tgt[:, i].clone() for i, k in enumerate(NAMES)}
    for mode in MODES:
        for method, its in (('lm', 50), ('adam', 400)):
            res, sec = _timed(lambda warm: fit_betas_to_measurements(
                module, bm, tg, method=method, iterations=2 if warm else its, circumference_derivative=mode))
            out[f'betas/{method}_{its}/{mode}'] = _row(res, res['measurements'], tgt, sec, bstar=bstar)
    gen = torch.Generator().manual_seed(31)
    bstar = torch.randn(256, 10, generator=gen).clamp(-2, 2).cuda()
    raw = synth.mean_params()[:132] + 0.3 * torch.randn(256, 132, generator=gen)
    with torch.no_grad():
        r = ops.decode_rot6d(raw.cuda())
        kp = module(global_rot=r[:, :1], body_pose=r[:, 1:], betas=bstar)['joints'][:].clone()
    tgt = measure(bstar)
    tg = {k: tgt[:, i].clone() for i, k in enumerate(NAMES)}
    mean = synth.mean_params().cuda()
    init = {'global_rot': mean[:6].expand(256, 6), 'body_pose': mean[6:132].expand(256, 126)}
    res, sec = _timed(lambda warm: fit_body_to_keypoints(module, kp, init=init, method='lm',
                                                         iterations=2 if warm else 50))
    out['kp/lm_50/keypoints_only'] = _row(res, measure(res['betas']), tgt, sec, kp, bstar)
    for mode in MODES:
        for method, its in (('lm', 50), ('adam', 600)):
            res, sec = _timed(lambda warm: fit_body_to_keypoints(
                module, kp, init=init, method=method, iterations=2 if warm else its, body_measurements=bm,
                measurements=tg, circumference_derivative=mode))
            out[f'kp_meas5/{method}_{its}/{mode}'] = _row(res, res['measurements'], tgt, sec, kp, bstar)
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--reps', type=int, default=5)
    p.add_argument('--out', default=None)
    a = p.parse_args()
    module, bm = _model()
    res = {'card': card(), 'kernels': [kernels(B, a.reps, module, bm) for B in (64, 4096)],
           'fit_quality': fit_quality(module, bm)}
    s = json.dumps(res)
    print(s)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(s + '\n')


if __name__ == '__main__':
    main()
