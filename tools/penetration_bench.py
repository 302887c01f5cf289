#!/usr/bin/env python
"""Times the self-penetration term on posed synthetic bodies (real SMPL-X topology, 20 908 faces) and prints one JSON
line: the card, its power limit and max SM clock (read in the same run), and at B = 64 and 1 024

  pairs          intersecting face pairs per body (part-filtered by ops.face_parts / parent_child_part_pairs)
  detect_ms      ops.self_collisions with the tree refit, next to closest_ms, ops.closest_points (8 192 points) refit
  forward_ms     ops.penetration_forward at those pairs
  backward_ms    ops.penetration_backward
and one Adam and one LM iteration of fit_body_to_scan at B = 64 with and without the term (adam_iter_ms, lm_iter_ms).

    python tools/penetration_bench.py [--out penetration.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from shapy_b200 import ops, synth  # noqa: E402


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else 'unknown'


def timed(fn, reps=20):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def posed(m, B, seed):
    g = torch.Generator().manual_seed(seed)
    raw = synth.mean_params()[:132] + 0.3 * torch.randn(B, 132, generator=g)
    rot = ops.decode_rot6d(raw.cuda())
    bend = torch.rand(B, generator=g).cuda() * 1.2 + 1.6          # elbows flexed 90-160 degrees
    c, s = torch.cos(bend), torch.sin(bend)
    z, o = torch.zeros_like(c), torch.ones_like(c)
    ry = lambda sg: torch.stack([c, z, sg * s, z, o, z, -sg * s, z, c], 1).view(B, 3, 3)  # noqa: E731
    rot[:, 18], rot[:, 19] = ry(-1.0), ry(1.0)
    with torch.no_grad():
        v = m(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=torch.zeros(B, m.num_betas, device='cuda'),
              return_shaped=False)['vertices'].contiguous()
    return raw, v


def smooth_smplx():
    """The synthetic model without its random pose correctives, which crumple a posed mesh into hundreds of
    thousands of spurious intersections: linear blend skinning of the real SMPL-X template."""
    d = synth.make_smplx()
    d['posedirs'] = torch.zeros_like(d['posedirs'])
    return d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('penetration_bench: needs a CUDA device')
    from shapy_b200.fit import fit_body_to_scan
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    m = SMPLX(data_struct=smooth_smplx()).cuda()
    faces = m.faces_i32
    pen = dict(part_labels=ops.face_parts(m), ignored_part_pairs=ops.parent_child_part_pairs(m.parents))
    res = {'card': card(), 'faces': int(faces.shape[0])}
    for B in (64, 1024):
        _, v = posed(m, B, 7)
        pts = v[:, torch.randperm(v.shape[1], generator=torch.Generator().manual_seed(1))[:8192].cuda()].contiguous()
        tree = ops.ScanTree()
        ops.closest_points(v, faces, pts, tree=tree)
        pairs, count = ops.self_collisions(v, faces, 1024, tree=tree, **pen)
        gl = torch.ones(B, device='cuda')
        cnt = count.cpu().numpy()
        res[f'B{B}'] = dict(
            pairs=dict(mean=float(cnt.mean()), min=int(cnt.min()), max=int(cnt.max())),
            detect_ms=timed(lambda: ops.self_collisions(v, faces, 1024, tree=tree, **pen)),
            closest_ms=timed(lambda: ops.closest_points(v, faces, pts, tree=tree)),
            forward_ms=timed(lambda: ops.penetration_forward(v, faces, pairs, 0.02)),
            backward_ms=timed(lambda: ops.penetration_backward(v, faces, pairs, gl, 0.02)))
    B, iters = 64, 20
    raw, v = posed(m, B, 8)
    pts = v[:, ::4].contiguous()
    init = {'global_rot': raw[:, :6].cuda(), 'body_pose': raw[:, 6:].cuda()}
    for method in ('adam', 'lm'):
        for name, kw in (('without', {}), ('with', dict(penetration_weight=0.1, penetration_sigma=0.02, **pen))):
            fit_body_to_scan(m, pts, init=init, iterations=2, method=method, **kw)
            torch.cuda.synchronize()
            a0, a1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a0.record()
            fit_body_to_scan(m, pts, init=init, iterations=iters, method=method, **kw)
            a1.record()
            torch.cuda.synchronize()
            res.setdefault(f'{method}_iter_ms_B64', {})[name] = a0.elapsed_time(a1) / (iters + 1)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
