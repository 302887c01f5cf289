"""Times one iteration of the LM scan fit launch by launch, the whole iteration, and one iteration of the Adam loop of
fit_body_to_scan (forward, closest and nearest points, backward, optimiser step), the arms alternating, at B = 64 and
1024 bodies of N = 8192 points on the synthetic model.  Prints one JSON line: [min, max] milliseconds over the reps,
the card's name and power limit read in the same run, and beside the times the vertex Jacobian's algorithmic bytes and
the row kernel's fp64 FLOPs from the shapes, with their fraction of the H100 SXM data sheet's 3.35 TB/s and 67 TFLOP/s
fp64 (tensor core) bounds.

    python tools/fit_scan_lm_bench.py [--batches 64 1024] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from shapy_b200 import ops, synth  # noqa: E402
from shapy_b200.autograd import ClosestPointsFunction, Rot6dFunction  # noqa: E402

HBM, FP64 = 3.35e12, 67e12


def _card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else 'unknown'


def _ms(fn, n=3):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    s.record()
    for _ in range(n):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / n


def bench(m, B, N, reps):
    g = torch.Generator().manual_seed(B)
    raw = synth.mean_params()[:132] + 0.3 * torch.randn(B, 132, generator=g)
    betas, transl = torch.randn(B, m.num_betas, generator=g).cuda(), (0.3 * torch.randn(B, 3, generator=g)).cuda()
    rot = ops.decode_rot6d(raw.cuda()).contiguous()
    with torch.no_grad():
        v0 = m(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=betas, transl=transl)['vertices']
    idx = torch.randint(0, v0.shape[1], (B, N), generator=g).cuda()
    pts = (torch.gather(v0, 1, idx[..., None].expand(-1, -1, 3)) + 0.002 * torch.randn(B, N, 3, device='cuda'))
    pts, w = pts.contiguous(), torch.ones(B, N, device='cuda')
    packed, faces = m.packed(), m.faces_i32
    P, V = 66 + m.num_betas + 3, packed.V
    trial = {'rot': rot, 'betas': betas.contiguous(), 'transl': transl.contiguous()}
    state = {'rot': rot.clone(), 'betas': betas.clone(), 'transl': transl.clone(),
             'A': torch.zeros(B, P, P, dtype=torch.float64, device='cuda'),
             'g': torch.zeros(B, P, dtype=torch.float64, device='cuda'), 'loss': torch.zeros(B, device='cuda'),
             'lambda': torch.zeros(B, device='cuda'), 'accepted': torch.zeros(B, dtype=torch.int32, device='cuda')}
    ws, tree = ops.fit_lm_scan_workspace(B, N, V, P, 'cuda'), ops.ScanTree()
    out = {}

    def vj():
        out['vj'] = ops.smplx_vertex_jacobian(packed, trial['betas'], trial['rot'], trial['transl'])

    def cp():
        out['cp'] = ops.closest_points(out['vj'][0], faces, pts, w, tree)

    def nn():
        out['nn'] = ops.nearest_points(out['vj'][0], pts, w)[0]

    def step():
        t = {k: v.clone() for k, v in trial.items()}
        ops.fit_lm_scan_step(state, t, pts, w, faces, None, 1.0, 1.0, 0.0, 0.0, 10.0, 3.0, True, *out['vj'],
                             out['cp'][0], out['cp'][1], out['nn'], ws)

    def iteration():
        vj(), cp(), nn(), step()
    iteration()
    # one iteration of fit_body_to_scan's Adam loop at both terms under least squares: its loss_fn (the forward, the
    # closest points with the tree refit, the nearest points), the backward and the optimiser step
    params = {'global_rot': raw[:, :6].cuda(), 'body_pose': raw[:, 6:].cuda(), 'betas': betas.clone(),
              'transl': transl.clone()}
    params = {k: v.contiguous().requires_grad_(True) for k, v in params.items()}
    opt, tree_a, wden = torch.optim.Adam(list(params.values()), lr=0.05), ops.ScanTree(), w.sum(1)

    def adam():
        opt.zero_grad(set_to_none=True)
        grot, bpose = Rot6dFunction.apply(params['global_rot']), Rot6dFunction.apply(params['body_pose'])
        v = m(global_rot=grot, body_pose=bpose, betas=params['betas'], transl=params['transl'],
              return_shaped=False)['vertices']
        per_body = (w * ClosestPointsFunction.apply(faces, v, pts, w, tree_a)).sum(1) / wden
        idx, _ = ops.nearest_points(v.detach(), pts, w)
        nn = torch.gather(pts, 1, idx.long()[..., None].expand(-1, -1, 3))
        per_body = per_body + (v - nn).pow(2).sum(-1).mean(1)
        per_body.sum().backward()
        opt.step()
    arms = {'vertex_jacobian': vj, 'closest_points': cp, 'nearest_points': nn, 'lm_scan_step': step,
            'lm_iteration': iteration, 'adam_iteration': adam}
    times = {k: [] for k in arms}
    for _ in range(reps):
        for k, fn in arms.items():
            times[k].append(_ms(fn))
    rows = 3 * N + 3 * V                      # at most: every point three rows, every vertex three
    res = {k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()}
    jb = 4.0 * B * V * 3 * P + 4.0 * B * V * 3
    fl = 2.0 * B * rows * (P * (P + 1) / 2 + P)
    res['vertex_jacobian_bytes'] = jb
    res['vertex_jacobian_frac_hbm'] = round(jb / HBM / (min(times['vertex_jacobian']) * 1e-3), 4)
    res['lm_scan_step_fp64_flop_max'] = fl
    res['lm_scan_step_frac_fp64'] = round(fl / FP64 / (min(times['lm_scan_step']) * 1e-3), 4)
    return res


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--batches', type=int, nargs='+', default=[64, 1024])
    p.add_argument('--points', type=int, default=8192)
    p.add_argument('--reps', type=int, default=5)
    a = p.parse_args()
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    m = SMPLX(data_struct=synth.make_smplx(), use_face_contour=True).cuda()
    out = {'card': _card()}
    for B in a.batches:
        out[f'B{B}'] = bench(m, B, a.points, a.reps)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
