"""Times the calibrated 2D keypoint Levenberg-Marquardt step (one body per group of calibrated views, one keypoint
Jacobian per body) against the weak-perspective shared-pose step of the same images on the seeded synthetic SMPL-X.

    python tools/fit_kp2d_calibrated_lm_bench.py [--reps 5] [--out fit_kp2d_calibrated_lm_bench.json]

Per number of views B = G V in (64, 256, 1024, 4096) and views per body V in (2, 4, 8), n_rot = 22, with CUDA events,
arms alternating within every rep, [min, max] over the reps of the mean time per call (microseconds), Geman-McClure
loss, pose and betas priors on, later steps:
  cal_step   shapy_fit_lm_keypoints_2d_calibrated_step over the G bodies (one launch)
  cal_iter   one calibrated LM iteration: the keypoint Jacobian of the G bodies + the step
  sp_step    shapy_fit_lm_keypoints_2d_shared_pose_step over the B images in groups of V (three launches)
  sp_iter    one shared-pose LM iteration: the keypoint Jacobian of the B images + the step
Then `-Xptxas -v` of fit.cu compiled for sm_90a into a temporary directory: registers, spills and static shared memory
of the two calibrated kernels.  The card's name, power limit and SM clocks are read in the same run; nothing is set.
"""
import argparse
import json
import math
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

VIEWS = (2, 4, 8)
SIZES = (64, 256, 1024, 4096)      # views B: small batches, the crossover, a full GPU


def _rig(G, V, centre):
    """(B, 3, 3) rotations and (B, 3) translations of V cameras per body on a 3 m circle about the vertical axis
    through `centre` (G, 3), at its height, looking at it."""
    R, T = [], []
    for g in range(G):
        for v in range(V):
            a = 2.0 * math.pi * v / V
            c = centre[g] + torch.tensor([3.0 * math.sin(a), 0.0, -3.0 * math.cos(a)])
            z = (centre[g] - c) / (centre[g] - c).norm()
            y = torch.tensor([0.0, 1.0, 0.0])
            x = torch.linalg.cross(y, z)
            Rv = torch.stack([x, y, z])
            R.append(Rv)
            T.append(-Rv @ c)
    return torch.stack(R).cuda().contiguous(), torch.stack(T).cuda().contiguous()


def kernels(B, V, reps, module):
    from shapy_b200 import ops, synth
    from shapy_b200.fit import LM_DOWN, LM_UP
    packed = module.packed()
    G = B // V
    gen = torch.Generator().manual_seed(B + V)
    raw = (synth.mean_params()[:132] + 0.3 * torch.randn(G, 132, generator=gen)).cuda()
    rot = ops.decode_rot6d(raw)
    betas = torch.randn(G, 10, generator=gen).clamp(-2, 2).cuda()
    transl = torch.zeros(G, 3, device='cuda')
    K = packed.K
    sigma, pw, bw = 5.0, 1.0, 0.01
    arms = {}
    # the calibrated step: G bodies, B views
    R, T = _rig(G, V, torch.zeros(G, 3))
    gidx = torch.arange(B, device='cuda') // V
    kp, jac = ops.smplx_keypoint_jacobian(packed, betas, rot)
    intr = torch.tensor([1000.0, 500.0, 500.0], device='cuda').repeat(B, 1)
    Y = torch.einsum('bij,bkj->bki', R, kp[gidx]) + T[:, None]
    tg = (1000.0 * Y[..., :2] / Y[..., 2:] + 500.0 + torch.randn(B, K, 2, generator=gen).cuda()).contiguous()
    w = torch.ones(B, K, device='cuda')
    ext = torch.cat([R.reshape(B, 9), T], 1).contiguous()
    off = torch.arange(0, B + 1, V, dtype=torch.int32)
    ws = ops.fit_lm_calibrated_workspace(B, G, 'cuda')
    st = {'rot': rot.clone(), 'betas': betas.clone(), 'transl': transl.clone(), 'keypoints': kp.clone(),
          'jac': jac.clone(), 'loss': torch.zeros(G, device='cuda'), 'lambda': torch.ones(G, device='cuda'),
          'accepted': torch.zeros(G, dtype=torch.int32, device='cuda')}
    tr = {'rot': rot.clone(), 'betas': betas.clone(), 'transl': transl.clone()}
    anchor = rot.clone()

    def cal_step(k=kp, j=jac):
        ops.fit_lm_keypoints_2d_calibrated_step(st, tr, tg, w, intr, ext, sigma, pw, bw, LM_UP, LM_DOWN, False, k, j,
                                                off, ws, pose_anchor=anchor)

    arms['cal_step'] = cal_step
    arms['cal_iter'] = lambda: cal_step(*ops.smplx_keypoint_jacobian(packed, tr['betas'], tr['rot']))
    # the shared-pose step: B images in groups of V
    srot = rot[gidx].contiguous()
    ib = betas[gidx].contiguous()
    cam = torch.tensor([1.0, 0.0, 0.0], device='cuda').repeat(B, 1)
    kpi, jaci = ops.smplx_keypoint_jacobian(packed, ib, srot)
    tgi = (torch.nn.functional.softplus(cam[:, :1, None]) * kpi[..., :2] +
           0.01 * torch.randn(B, K, 2, generator=gen).cuda()).contiguous()
    sst = {'rot': srot.clone(), 'betas': betas.clone(), 'camera': cam.clone(), 'keypoints': kpi.clone(),
           'jac': jaci.clone(), 'loss': torch.zeros(G, device='cuda'), 'lambda': torch.ones(G, device='cuda'),
           'accepted': torch.zeros(G, dtype=torch.int32, device='cuda')}
    stri = {'rot': srot.clone(), 'betas': betas.clone(), 'image_betas': ib.clone(), 'camera': cam.clone()}
    sws = ops.fit_lm_shared_pose_workspace(B, G, 22, 10, 'cuda')

    def sp_step(k=kpi, j=jaci):
        ops.fit_lm_keypoints_2d_shared_pose_step(sst, stri, tgi, w, 0.05, pw, bw, LM_UP, LM_DOWN, False, k, j, off, sws,
                                                 pose_anchor=anchor)

    arms['sp_step'] = sp_step
    arms['sp_iter'] = lambda: sp_step(*ops.smplx_keypoint_jacobian(packed, stri['image_betas'], stri['rot']))
    t = time_arms(arms, 20 if B <= 256 else 3, reps)
    return {'B': B, 'V': V, 'G': G, 'us': _us(t)}


def ptxas():
    """Registers, spill bytes and static shared memory of the calibrated kernels, from nvcc -Xptxas -v."""
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
        if name and 'lm_kp2dc_step' in name:
            e = out.setdefault('meas' if 'ILb1' in name else 'plain', {})
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
    res = {'card': card(), 'clocks_before': clocks(),
           'kernels': [kernels(B, V, a.reps, module) for B in SIZES for V in VIEWS],
           'clocks_after': clocks(), 'ptxas': ptxas()}
    s = json.dumps(res)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(s + '\n')


if __name__ == '__main__':
    main()
