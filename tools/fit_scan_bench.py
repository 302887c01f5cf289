"""Times the scan queries and the scan fit on the seeded synthetic SMPL-X model (20 908 faces, 10 475 vertices).

    python tools/fit_scan_bench.py [--reps 5] [--out fit_scan_bench.json]

Per batch size (64 and 4096 bodies), N = 8192 scan points per body (vertices of the posed body moved by 1 cm noise),
with CUDA events, arms alternating within every rep, [min, max] over the reps of the mean time per call (microseconds):
  closest_build   ops.closest_points: triangle soup, tree build (prepare, topology, refit) and the scan -> model query
  closest_refit   the same with the tree of an earlier call refit (the fit's path after its first iteration)
  nearest         ops.nearest_points: point soup, tree build and the model -> scan query of every vertex
  backward        ops.closest_points_backward
  adam_iter       one Adam iteration of fit_body_to_scan, and its parts: decoder + SMPLX.forward, the scan -> model
                  term, the model -> scan term, the backward through both and SMPL-X, the optimiser step
Kernel times (one call each under torch.profiler, microseconds) split the calls into their launches.  Bytes come from
the shapes.  Then the time to quality of the scan fit against the 3D keypoint LM fit on the 64 bodies of
tests/test_gpu_fit_scan.py.  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from tools.fit_lm_bench import card, time_arms  # noqa: E402

N = 8192


def _us(t):
    return {k: [round(v[0] * 1e3, 1), round(v[1] * 1e3, 1)] for k, v in t.items()}


def _bytes(B, V, F):
    f32 = 4
    return {'closest_points': B * (V * 3 + N * 3) * f32 + B * F * 9 * f32 * 2 + B * F * 76 + B * N * 5 * f32,
            'nearest_points': B * (V * 3 + N * 3 + N) * f32 + B * N * 9 * f32 * 2 + B * N * 76 + B * V * 2 * f32,
            'backward': B * (V * 3 * 2 + N * 8) * f32}


def _kernel_times(calls):
    """{call: {kernel: microseconds}} from one profiled call each."""
    from torch.profiler import ProfilerActivity, profile
    out = {}
    for name, fn in calls.items():
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        k = {}
        for e in prof.key_averages():
            if 'shapy' in e.key and e.device_type.name == 'CUDA':
                short = e.key.split('(')[0].replace('void ', '').replace('shapy::', '')
                k[short] = round(k.get(short, 0.0) + e.device_time_total, 1)
        out[name] = k
    return out


def kernels(B, reps):
    from shapy_b200 import ops, synth
    from shapy_b200.autograd import ClosestPointsFunction, Rot6dFunction
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    m = SMPLX(data_struct=synth.make_smplx()).cuda()
    faces = m.faces_i32
    gen = torch.Generator().manual_seed(B)
    raw = (synth.mean_params()[:132] + 0.3 * torch.randn(B, 132, generator=gen)).cuda()
    betas = torch.randn(B, 10, generator=gen).clamp(-2, 2).cuda()
    with torch.no_grad():
        rot = ops.decode_rot6d(raw)
        v = m(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=betas, return_shaped=False)['vertices'].contiguous()
    V, F = v.shape[1], faces.shape[0]
    pick = torch.randint(0, V, (B, N), generator=gen).cuda()
    pts = (torch.gather(v, 1, pick[..., None].expand(-1, -1, 3)) +
           0.01 * torch.randn(B, N, 3, generator=gen).cuda()).contiguous()
    w = torch.ones(B, N, device='cuda')
    face, bary, d2 = ops.closest_points(v, faces, pts)
    g = torch.randn(B, N, generator=gen).cuda()
    tree = ops.ScanTree()
    ops.closest_points(v, faces, pts, tree=tree)

    params = {'g': raw[:, :6].clone().requires_grad_(True), 'p': raw[:, 6:].clone().requires_grad_(True),
              'b': betas.clone().requires_grad_(True), 't': torch.zeros(B, 3, device='cuda', requires_grad=True)}
    opt = torch.optim.Adam(list(params.values()), lr=0.05)
    atree = ops.ScanTree()
    parts = {k: [] for k in ('forward', 'scan_to_model', 'model_to_scan', 'backward', 'step')}

    def adam(record=False):                # the body of fit_body_to_scan's Adam loop, both terms, least squares
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)] if record else None
        if record:
            ev[0].record()
        opt.zero_grad(set_to_none=True)
        vv = m(global_rot=Rot6dFunction.apply(params['g']), body_pose=Rot6dFunction.apply(params['p']),
               betas=params['b'], transl=params['t'], return_shaped=False)['vertices']
        if record:
            ev[1].record()
        loss = ClosestPointsFunction.apply(faces, vv, pts, w, atree).mean(1)
        if record:
            ev[2].record()
        idx, _ = ops.nearest_points(vv.detach(), pts, w)
        nn = torch.gather(pts, 1, idx.long()[..., None].expand(-1, -1, 3))
        loss = loss + (vv - nn).pow(2).sum(-1).mean(1)
        if record:
            ev[3].record()
        loss.sum().backward()
        if record:
            ev[4].record()
        opt.step()
        if record:
            ev[5].record()
            return ev

    arms = {'closest_build': lambda: ops.closest_points(v, faces, pts),
            'closest_refit': lambda: ops.closest_points(v, faces, pts, tree=tree),
            'nearest': lambda: ops.nearest_points(v, pts),
            'backward': lambda: ops.closest_points_backward(v, faces, pts, face, bary, g),
            'adam_iter': adam}
    t = time_arms(arms, 10 if B <= 64 else 2, reps)
    for _ in range(reps):
        ev = adam(record=True)
        ev[-1].synchronize()
        for i, k in enumerate(parts):
            parts[k].append(ev[i].elapsed_time(ev[i + 1]))
    t.update({f'adam_{k}': [round(min(x), 4), round(max(x), 4)] for k, x in parts.items()})
    kt = _kernel_times({k: arms[k] for k in ('closest_build', 'closest_refit', 'nearest', 'backward')})
    return {'B': B, 'N': N, 'V': V, 'F': F, 'us': _us(t), 'kernel_us': kt, 'bytes': _bytes(B, V, F)}


def time_to_quality():
    import test_gpu_fit_scan as t
    return t._rows()


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
