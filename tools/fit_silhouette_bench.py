#!/usr/bin/env python
"""Times the silhouette term on posed synthetic bodies (real SMPL-X topology, 20 908 faces) and prints one JSON line:
the card, its power limit and max SM clock (read in the same run), and at B = 64 with 1000 x 1000 masks and B = 1024
with 512 x 512 masks (SSP-3D's size, at f = 500 so that the bodies at 2-4 m fill a third of the frame), [min, max] over 5 reps of CUDA-event times, the arms alternating:

  prepare_ms     ops.silhouette_prepare, and its HBM fraction: the distance transform's 13 B H W bytes (the column pass
                 reads the masks and writes int32 g, the row pass reads g and writes dist) over 3.35 TB/s
  render_ms      ops.render_silhouette
  forward_ms     ops.silhouette_forward
  closest_ms     ops.closest_points on the projected mesh, tree refit and query, 4096 contour points per body
  backward_ms    ops.closest_points_backward + ops.silhouette_backward
  adam_iter_ms   one Adam iteration of fit_body_to_keypoints_2d (perspective) without and with the term (B = 64 only)

    python tools/fit_silhouette_bench.py [--out silhouette.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from shapy_b200 import ops, synth  # noqa: E402

HBM = 3.35e12          # bytes/s, the H100 SXM data sheet


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else 'unknown'


def event_ms(fn, reps=10):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def alternate(arms, rounds=5):
    """{name: [min, max]} over `rounds` of each arm, the arms alternating."""
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    t = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            t[k].append(event_ms(fn))
    return {k: [round(min(v), 4), round(max(v), 4)] for k, v in t.items()}


def bodies(m, B, seed, size, f):
    g = torch.Generator().manual_seed(seed)
    raw = synth.mean_params()[:132] + 0.3 * torch.randn(B, 132, generator=g)
    betas = torch.randn(B, m.num_betas, generator=g).clamp(-2, 2)
    t = torch.cat([0.2 * torch.randn(B, 2, generator=g), 2.0 + 2.0 * torch.rand(B, 1, generator=g)], 1)
    rot = ops.decode_rot6d(raw.cuda())
    with torch.no_grad():
        v = m(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=betas.cuda(), transl=t.cuda(),
              return_shaped=False)['vertices'].contiguous()
    intr = torch.tensor([f, size / 2, size / 2]).repeat(B, 1).cuda()
    return raw, betas, t, v, intr


def kernels(m, B, size, f):
    _, _, _, v, intr = bodies(m, B, 1, size, f)
    faces = m.faces_i32
    masks = ops.render_silhouette(v * 1.01, faces, intr, size, size)
    dist, contour, cw, count = ops.silhouette_prepare(masks, 4096)
    proj, _ = ops.silhouette_forward(v, intr, dist)
    tree = ops.ScanTree()
    face, bary, d2 = ops.closest_points(proj, faces, contour, cw, tree=tree)
    g = torch.ones(B, device='cuda')
    gd2 = torch.full_like(d2, 1e-3)

    def backward():
        gp = ops.closest_points_backward(proj, faces, contour, face, bary, gd2)
        ops.silhouette_backward(v, intr, dist, g, gp)

    t = alternate({'prepare_ms': lambda: ops.silhouette_prepare(masks, 4096),
                   'render_ms': lambda: ops.render_silhouette(v, faces, intr, size, size),
                   'forward_ms': lambda: ops.silhouette_forward(v, intr, dist),
                   'closest_ms': lambda: ops.closest_points(proj, faces, contour, cw, tree=tree),
                   'backward_ms': backward})
    nbytes = 13 * B * size * size      # column pass: the mask read, g written; row pass: g read, dist written
    t['prepare_hbm_fraction'] = round(nbytes / HBM / (t['prepare_ms'][0] * 1e-3), 4)
    t['contour_pixels_median'] = int(count.float().median())
    return t


def adam_iterations(m, B, size, f):
    from shapy_b200.fit import fit_body_to_keypoints_2d
    raw, betas, t, v, intr = bodies(m, B, 2, size, f)
    masks = ops.render_silhouette(v, m.faces_i32, intr, size, size)
    with torch.no_grad():
        x = m(global_rot=ops.decode_rot6d(raw[:, :6].cuda()), body_pose=ops.decode_rot6d(raw[:, 6:].cuda()),
              betas=betas.cuda(), transl=t.cuda(), return_shaped=False)['joints'][:]
        from shapy_b200.fit import _project
        x = _project(x, intr).contiguous()
    init = {'global_rot': raw[:, :6].cuda(), 'body_pose': raw[:, 6:].cuda(), 'betas': betas.cuda(),
            'transl': t.cuda()}
    kw = dict(focal_length=f, principal_point=(size / 2, size / 2))

    def per_iteration(extra):
        # the iteration's cost: the difference of a 21- and a 1-iteration fit over 20
        def run(n):
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fit_body_to_keypoints_2d(m, x, init=dict(init), iterations=n, **kw, **extra)
            b.record()
            torch.cuda.synchronize()
            return a.elapsed_time(b)
        return lambda: (run(21) - run(1)) / 20

    arms = {'without': per_iteration({}), 'with': per_iteration(dict(silhouettes=masks))}
    for fn in arms.values():
        fn()
    r = {k: [] for k in arms}
    for _ in range(5):
        for k, fn in arms.items():
            r[k].append(fn())
    return {k: [round(min(v), 3), round(max(v), 3)] for k, v in r.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    m = SMPLX(data_struct=synth.make_smplx()).cuda()
    res = {'card': card()}
    res['b64_1000'] = kernels(m, 64, 1000, 1000.0)
    res['b1024_512'] = kernels(m, 1024, 512, 500.0)
    res['adam_iter_ms_b64_1000'] = adam_iterations(m, 64, 1000, 1000.0)
    res['card_after'] = card()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, 'w') as fh:
            fh.write(line + '\n')


if __name__ == '__main__':
    main()
