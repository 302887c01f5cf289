"""Times the keypoint Jacobian and the Levenberg-Marquardt keypoint fit on the seeded synthetic SMPL-X model.

    python tools/fit_kp_lm_bench.py [--reps 5] [--out fit_kp_lm_bench.json]

Per batch size (64 and 4096 bodies), n_rot = 22, with CUDA events, arms alternating within every rep, [min, max] over
the reps of the mean time per call (microseconds):
  forward     shapy_smplx_forward (vertices and joints)
  backward    shapy_smplx_backward with a joints cotangent (betas and rotation gradients)
  jacobian    shapy_smplx_keypoint_jacobian, one launch
  lm_step     shapy_fit_lm_keypoints_step
  lm_iter     one LM iteration: jacobian + step
  adam_iter   one Adam iteration of fit_body_to_keypoints: decoder + forward, backward, optimiser step
Then the time to quality of LM (50 iterations) against Adam (600) on the 256 bodies of
tests/test_gpu_fit_lm_keypoints.py (seed 31, mean-pose start): wall time, median loss, the fraction within 1 cm
keypoint RMS and the median RMS.  The Jacobian launch's bytes come from the shapes: the Jacobian and keypoints written
(HBM), and the model rows it reads at the touched vertices (template, shape rows and posedirs rows below Kp for v_posed,
9 posedirs rows per rotation block of a landmark or J14 entry), served from L2 (about 1.5 MB of distinct rows).  The
card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.fit_lm_bench import card, time_arms  # noqa: E402


def _us(t):
    return {k: [round(v[0] * 1e3, 1), round(v[1] * 1e3, 1)] for k, v in t.items()}


def kernels(B, reps):
    from shapy_b200 import ops, synth
    from shapy_b200.autograd import Rot6dFunction
    from shapy_b200.fit import LM_DOWN, LM_UP
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    d = synth.make_smplx()
    module = SMPLX(data_struct=d, use_face_contour=True).cuda()
    packed = module.packed()
    gen = torch.Generator().manual_seed(B)
    raw = (synth.mean_params()[:132] + 0.3 * torch.randn(B, 132, generator=gen)).cuda()
    rot = ops.decode_rot6d(raw)
    betas = torch.randn(B, 10, generator=gen).clamp(-2, 2).cuda()
    transl = torch.zeros(B, 3, device='cuda')
    K = packed.K
    cot = torch.randn(B, K, 3, generator=gen).cuda()
    kp, jac = ops.smplx_keypoint_jacobian(packed, betas, rot, transl)
    tg = (kp + 0.01 * torch.randn(B, K, 3, generator=gen).cuda()).contiguous()
    w = torch.ones(B, K, device='cuda')
    P = jac.shape[2]
    state = {'rot': rot.clone(), 'betas': betas.clone(), 'transl': transl.clone(), 'keypoints': kp.clone(),
             'jac': jac.clone(), 'loss': torch.zeros(B, device='cuda'), 'lambda': torch.ones(B, device='cuda'),
             'accepted': torch.zeros(B, dtype=torch.int32, device='cuda')}
    trial = {'rot': rot.clone(), 'betas': betas.clone(), 'transl': transl.clone()}

    def step():
        ops.fit_lm_keypoints_step(state, trial, tg, w, LM_UP, LM_DOWN, False, kp, jac)

    def iteration():
        k, j = ops.smplx_keypoint_jacobian(packed, trial['betas'], trial['rot'], trial['transl'])
        ops.fit_lm_keypoints_step(state, trial, tg, w, LM_UP, LM_DOWN, False, k, j)

    params = {'r': raw.clone().requires_grad_(True), 'b': betas.clone().requires_grad_(True),
              't': transl.clone().requires_grad_(True)}
    opt = torch.optim.Adam(list(params.values()), lr=0.05)

    def adam():                                    # the body of fit_body_to_keypoints' Adam loop
        opt.zero_grad(set_to_none=True)
        r = Rot6dFunction.apply(params['r'])
        out = module(global_rot=r[:, :1], body_pose=r[:, 1:], betas=params['b'], transl=params['t'],
                     return_shaped=False)
        ((out['joints'][:] - tg).pow(2).sum(-1) * w).sum().backward()
        opt.step()

    arms = {'forward': lambda: ops.smplx_forward(packed, betas, rot, want_v_shaped=False),
            'backward': lambda: ops.smplx_backward(packed, betas, rot, grad_joints=cot, want=('betas', 'rot')),
            'jacobian': lambda: ops.smplx_keypoint_jacobian(packed, betas, rot, transl),
            'lm_step': step, 'lm_iter': iteration, 'adam_iter': adam}
    t = time_arms(arms, 20 if B <= 64 else 3, reps)
    # bytes of the Jacobian launch, from the shapes
    L, D = d['lmk_faces_idx'].shape[0], d['dynamic_lmk_faces_idx'].shape[1]
    nnz = int((d['extra_joint_regressor'] != 0).sum())
    entries = 3 * (L + D) + nnz
    n_rot, NB, Kp = 22, 10, 21 * 9
    written = B * (3 * K * P + 3 * K) * 4
    l2_rows = B * (entries * (1 + NB + Kp) * 12 + entries * (n_rot - 1) * 9 * 12)
    tj = t['jacobian']
    return {'B': B, 'us': _us(t), 'entries_per_body': entries, 'jacobian_bytes_written': written,
            'jacobian_write_rate_GBps': [round(written / (tj[1] * 1e-3) / 1e9, 1),
                                         round(written / (tj[0] * 1e-3) / 1e9, 1)],
            'jacobian_row_bytes_from_l2': l2_rows,
            'jacobian_l2_row_rate_GBps': [round(l2_rows / (tj[1] * 1e-3) / 1e9, 1),
                                          round(l2_rows / (tj[0] * 1e-3) / 1e9, 1)]}


def time_to_quality():
    from shapy_b200 import ops, synth
    from shapy_b200.fit import fit_body_to_keypoints
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    module = SMPLX(data_struct=synth.make_smplx(), use_face_contour=True).cuda()
    gen = torch.Generator().manual_seed(31)
    bstar = torch.randn(256, 10, generator=gen).clamp(-2, 2)
    raw = synth.mean_params()[:132] + 0.3 * torch.randn(256, 132, generator=gen)
    with torch.no_grad():
        r = ops.decode_rot6d(raw.cuda())
        kp = module(global_rot=r[:, :1], body_pose=r[:, 1:], betas=bstar.cuda())['joints'][:].clone()
    mean = synth.mean_params().cuda()
    init = {'global_rot': mean[:6].expand(256, 6), 'body_pose': mean[6:132].expand(256, 126)}
    for m in ('lm', 'adam'):                                     # warm-up
        fit_body_to_keypoints(module, kp, init=init, method=m, iterations=2)
    out = {}
    for name, kw in (('lm_50', dict(method='lm')), ('adam_600', dict(method='adam'))):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = fit_body_to_keypoints(module, kp, init=init, **kw)
        torch.cuda.synchronize()
        rms = (res['keypoints'] - kp).pow(2).sum(-1).mean(1).sqrt()
        out[name] = {'seconds': round(time.perf_counter() - t0, 4), 'median_loss': float(res['loss'].median()),
                     'frac_rms_1cm': round(float((rms < 1e-2).float().mean()), 4),
                     'median_rms_m': float(rms.median())}
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--reps', type=int, default=5)
    p.add_argument('--out', default=None)
    a = p.parse_args()
    res = {'card': card(), 'kernels': [kernels(B, a.reps) for B in (64, 4096)], 'time_to_quality': time_to_quality()}
    s = json.dumps(res)
    print(s)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(s + '\n')


if __name__ == '__main__':
    main()
