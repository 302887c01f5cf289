"""Times the sequence 2D keypoint Levenberg-Marquardt step (one betas per video, smoothness between frames) against the
perspective step on the same frames, on the seeded synthetic SMPL-X.

    python tools/fit_kp2d_sequence_lm_bench.py [--reps 5] [--out fit_kp2d_sequence_lm_bench.json]

Per batch size (256 and 4096 frames) in sequences of T = 1, 8, 32 and 128 frames, plus 4 sequences of 1024 frames (a
few CTAs running the serial sweep), n_rot = 22, with CUDA events, arms alternating within every rep, [min, max] over
the reps of the mean time per call (microseconds), Geman-McClure loss, pose and betas priors and both smoothness terms
on, later steps:
  persp_step / persp_iter    shapy_fit_lm_keypoints_2d_perspective_step (one betas per frame), and one LM iteration:
                             keypoint Jacobian + step
  seq{T}_step / seq{T}_iter  shapy_fit_lm_keypoints_2d_sequence_step (three launches), and one LM iteration
  jacobian                   shapy_smplx_keypoint_jacobian alone
The fp64 operations of the sweep are printed from the shapes: per frame about n1^3 / 3 (the Cholesky of the n1 x n1
block) + 2 n1^3 (the two triangular solves against C_t^T) + n1^2 nb (against B_t), n1 = 3 n_rot + 3.  Then the quality
and wall time of the three fits of tests/test_gpu_fit_lm_kp2d_sequence.py's quality test.  The card's name, power limit
and SM clocks are read in the same run; nothing is set.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests'))
from tools.fit_kp2d_lm_bench import _us, clocks  # noqa: E402
from tools.fit_kp_meas_lm_bench import _model  # noqa: E402
from tools.fit_lm_bench import card, time_arms  # noqa: E402

LENGTHS = (1, 8, 32, 128)


def sweep_flops(n_rot=22, nb=10):
    n1 = 3 * n_rot + 3
    return n1 ** 3 / 3 + 2 * n1 ** 3 + n1 * n1 * nb


def kernels(B, lengths, reps, module):
    from shapy_b200 import ops, synth
    from shapy_b200.fit import LM_DOWN, LM_UP, _project
    packed = module.packed()
    gen = torch.Generator().manual_seed(B)
    raw = (synth.mean_params()[:132] + 0.3 * torch.randn(B, 132, generator=gen)).cuda()
    rot = ops.decode_rot6d(raw)
    betas = torch.randn(B, 10, generator=gen).clamp(-2, 2).cuda()
    tr = torch.tensor([0.0, 0.2, 3.0], device='cuda').repeat(B, 1)
    intr = torch.tensor([1000.0, 500.0, 500.0], device='cuda').repeat(B, 1)
    K = packed.K
    kp, jac = ops.smplx_keypoint_jacobian(packed, betas, rot)
    tg = (_project(kp + tr[:, None], intr) + 2.0 * torch.randn(B, K, 2, generator=gen).cuda()).contiguous()
    w = torch.ones(B, K, device='cuda')
    anchor = rot.clone()
    sigma, pw, bw, srw, stw = 10.0, 100.0, 10.0, 3e3, 1e4
    ps = {'rot': rot.clone(), 'betas': betas.clone(), 'transl': tr.clone(), 'keypoints': kp.clone(),
          'jac': jac.clone(), 'loss': torch.zeros(B, device='cuda'), 'lambda': torch.ones(B, device='cuda'),
          'accepted': torch.zeros(B, dtype=torch.int32, device='cuda')}
    pt = {'rot': rot.clone(), 'betas': betas.clone(), 'transl': tr.clone()}

    def pstep(k=kp, j=jac):
        ops.fit_lm_keypoints_2d_perspective_step(ps, pt, tg, w, intr, sigma, pw, bw, LM_UP, LM_DOWN, False, k, j,
                                                 pose_anchor=anchor)

    def piter():
        pstep(*ops.smplx_keypoint_jacobian(packed, pt['betas'], pt['rot']))

    def jacobian():
        ops.smplx_keypoint_jacobian(packed, pt['betas'], pt['rot'])

    arms = {'jacobian': jacobian, 'persp_step': pstep, 'persp_iter': piter}
    for T in lengths:
        S = B // T
        off = torch.arange(0, B + 1, T, dtype=torch.int32)
        sb = betas[::T].contiguous()
        ss = dict(ps, betas=sb.clone(), loss=torch.zeros(S, device='cuda'),
                  accepted=torch.zeros(S, dtype=torch.int32, device='cuda'), **{'lambda': torch.ones(S, device='cuda')})
        st = {'rot': rot.clone(), 'betas': sb.clone(), 'image_betas': sb.repeat_interleave(T, 0).contiguous(),
              'transl': tr.clone()}
        ws = ops.fit_lm_sequence_workspace(B, S, 22, 10, 'cuda')

        def sstep(k=kp, j=jac, ss=ss, st=st, off=off, ws=ws):
            ops.fit_lm_keypoints_2d_sequence_step(ss, st, tg, w, intr, sigma, pw, bw, srw, stw, LM_UP, LM_DOWN, False,
                                                  k, j, off, ws, pose_anchor=anchor)

        def siter(sstep=sstep, st=st):
            sstep(*ops.smplx_keypoint_jacobian(packed, st['image_betas'], st['rot']))

        arms[f'seq{T}_step'], arms[f'seq{T}_iter'] = sstep, siter
    t = time_arms(arms, 5 if B >= 4096 or max(lengths) > 128 else 20, reps)
    return {'B': B, 'us': _us(t)}


def quality(module):
    from test_gpu_fit_lm_kp2d_sequence import _video, quality_runs
    return quality_runs(module, _video(module, 32, 32))


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--reps', type=int, default=5)
    p.add_argument('--out', default=None)
    p.add_argument('--no-quality', dest='quality', action='store_false')
    a = p.parse_args()
    module, _ = _model()
    res = {'card': card(), 'clocks_before': clocks(),
           'sweep_fp64_flops_per_frame': round(sweep_flops()),
           'kernels': [kernels(256, LENGTHS, a.reps, module), kernels(4096, LENGTHS, a.reps, module),
                       kernels(4096, (1024,), a.reps, module)]}
    if a.quality:
        res['quality_32x32'] = quality(module)
    res['clocks_after'] = clocks()
    s = json.dumps(res)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(s + '\n')


if __name__ == '__main__':
    main()
