"""Times the shared-pose 2D keypoint Levenberg-Marquardt step (one body pose and betas per group of simultaneous views)
against the shape-sharing grouped step on the seeded synthetic SMPL-X.

    python tools/fit_kp2d_shared_pose_lm_bench.py [--reps 5] [--out fit_kp2d_shared_pose_lm_bench.json]

Per batch size (64 and 4096 images), n_rot = 22, with CUDA events, arms alternating within every rep, [min, max] over
the reps of the mean time per call (microseconds), Geman-McClure loss, pose and betas priors on, later steps:
  g{n}_step      shapy_fit_lm_keypoints_2d_groups_step with groups of n = 1, 4, 16 images (three launches)
  sp{n}_step     shapy_fit_lm_keypoints_2d_shared_pose_step with the same groups (three launches)
  g{n}_iter      one grouped LM iteration: keypoint Jacobian + the grouped step
  sp{n}_iter     one shared-pose LM iteration: keypoint Jacobian + the shared-pose step
Then `-Xptxas -v` of fit.cu compiled for sm_90a into a temporary directory: registers, spills and static shared memory
of the three shared-pose kernels.  The card's name, power limit and SM clocks are read in the same run; nothing is set.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
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
    w = torch.ones(B, K, device='cuda')
    sigma, pw, bw = 0.05, 1.0, 0.01
    arms = {}
    for n in GROUP_SIZES:
        G = B // n
        off = torch.arange(0, B + 1, n, dtype=torch.int32)
        gb = betas[::n].contiguous()
        gidx = torch.arange(B, device='cuda') // n
        srot = torch.cat([rot[:, :1], rot[::n, 1:][gidx]], 1).contiguous()    # one body pose per group
        kp, jac = ops.smplx_keypoint_jacobian(packed, gb[gidx].contiguous(), srot)
        tg = (torch.nn.functional.softplus(cam[:, :1, None]) * kp[..., :2] +
              0.01 * torch.randn(B, K, 2, generator=gen).cuda()).contiguous()
        for name, share in (('g', False), ('sp', True)):
            st = {'rot': srot.clone(), 'betas': gb.clone(), 'camera': cam.clone(), 'keypoints': kp.clone(),
                  'jac': jac.clone(), 'loss': torch.zeros(G, device='cuda'), 'lambda': torch.ones(G, device='cuda'),
                  'accepted': torch.zeros(G, dtype=torch.int32, device='cuda')}
            tr = {'rot': srot.clone(), 'betas': gb.clone(), 'image_betas': gb[gidx].contiguous(),
                  'camera': cam.clone()}
            if share:
                ws = ops.fit_lm_shared_pose_workspace(B, G, 22, 10, 'cuda')
                fn, anchor = ops.fit_lm_keypoints_2d_shared_pose_step, srot[::n].contiguous()
            else:
                ws = ops.fit_lm_groups_workspace(B, G, 22, 10, 'cuda')
                fn, anchor = ops.fit_lm_keypoints_2d_groups_step, srot.clone()

            def step(k=kp, j=jac, st=st, tr=tr, off=off, ws=ws, fn=fn, anchor=anchor, tg=tg):
                fn(st, tr, tg, w, sigma, pw, bw, LM_UP, LM_DOWN, False, k, j, off, ws, pose_anchor=anchor)

            def it(step=step, tr=tr):
                step(*ops.smplx_keypoint_jacobian(packed, tr['image_betas'], tr['rot']))

            arms[f'{name}{n}_step'], arms[f'{name}{n}_iter'] = step, it
    t = time_arms(arms, 20 if B <= 64 else 3, reps)
    return {'B': B, 'us': _us(t)}


def ptxas():
    """Registers, spill bytes and static shared memory of the shared-pose kernels, from nvcc -Xptxas -v."""
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    src = os.path.join(ROOT, 'shapy_b200', 'csrc', 'fit.cu')
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([nvcc, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17',
                            '--expt-relaxed-constexpr', '-fmad=false', '-Xptxas', '-v', '-c', src, '-o',
                            os.path.join(d, 'fit.o')], capture_output=True, text=True)
    if r.returncode:
        return {'error': r.stderr[-400:]}
    out, name = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            name = m.group(1)
            continue
        if name and 'lm_kp2dg' in name and 'ILb1' in name:
            kernel = re.search(r'lm_kp2dg_(\w+?)_kernel', name).group(1)
            e = out.setdefault(kernel, {})
            m = re.search(r'(\d+) bytes spill stores, (\d+) bytes spill loads', line)
            if m:
                e['spill_stores'], e['spill_loads'] = int(m.group(1)), int(m.group(2))
            m = re.search(r'Used (\d+) registers.*?(\d+) bytes smem', line)
            if m:
                e['registers'], e['static_smem'] = int(m.group(1)), int(m.group(2))
                name = None
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--reps', type=int, default=5)
    p.add_argument('--out', default=None)
    a = p.parse_args()
    module, _ = _model()
    res = {'card': card(), 'clocks_before': clocks(), 'kernels': [kernels(B, a.reps, module) for B in (64, 4096)],
           'clocks_after': clocks(), 'ptxas': ptxas()}
    s = json.dumps(res)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(s + '\n')


if __name__ == '__main__':
    main()
