"""Times the measurement Jacobian and the Levenberg-Marquardt fit on the seeded synthetic SMPL-X model.

    python tools/fit_lm_bench.py [--reps 5] [--out fit_lm_bench.json]

Per batch size (64 and 4096 bodies), with CUDA events, arms alternating within every rep, [min, max] over the reps of
the mean time per call:
  forward     shapy_measure_forward (the reference point: phases 0-3 of every mode)
  jacobian    shapy_measure_jacobian_betas, one launch
  composite   the Jacobian composed from what existed before: 5 x (measure backward with a one-hot cotangent + shape
              backward)
  lm_step     shapy_fit_lm_step
  lm_iter     one LM iteration: forward_shape, jacobian, step
Then the time to quality of LM(50) against Adam(400) on the 256 bodies of tests/test_gpu_fit.py (seed 21, from
beta = 0): wall time, median loss and the three fractions of that test.  The card's name and power limit are read in
the same run.  The mass row's algorithmic traffic is one pass over the shape rows per body, NB 3V 4 bytes, served
from L2 (the 1.3 MB basis stays resident), reported as bytes and as the rate the Jacobian launch would need if it did
nothing else.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

NAMES = ('mass', 'height', 'chest', 'waist', 'hips')


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30)
        limit = r.stdout.strip().splitlines()[0] if r.returncode == 0 else 'unknown'
    except (OSError, subprocess.SubprocessError):
        limit = 'unknown'
    return {'name': name, 'power_limit_and_max_sm_clock': limit}


def time_arms(arms, n, reps):
    """{name: [min, max] ms per call}: every rep runs every arm n times between two events, arms alternating."""
    res = {k: [] for k in arms}
    for fn in arms.values():        # warm-up
        fn()
    torch.cuda.synchronize()
    for _ in range(reps):
        for k, fn in arms.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(n):
                fn()
            b.record()
            b.synchronize()
            res[k].append(a.elapsed_time(b) / n)
    return {k: [round(min(v), 4), round(max(v), 4)] for k, v in res.items()}


def kernels(B, reps):
    from shapy_b200 import ops, synth
    d = synth.make_smplx()
    packed = ops.SmplxModel(dict(d), 'cuda')
    faces = d['faces_tensor'].to(torch.int32).cuda()
    lm = ops.make_landmarks(synth.load_landmarks())
    betas = torch.randn(B, 10, generator=torch.Generator().manual_seed(B)).clamp(-2, 2).cuda()
    v = ops.smplx_forward_shape(packed, betas)
    onehot = [torch.zeros(B, 5, device='cuda').index_fill_(1, torch.tensor([k], device='cuda'), 1.0) for k in range(5)]

    def composite():
        return [ops.smplx_backward_shape(packed, ops.measure_backward(lm, g, v_shaped=v, faces_i32=faces))
                for g in onehot]

    meas, jac, _ = ops.measure_jacobian_betas(packed, lm, v, faces)
    tg = meas.clone().nan_to_num(1.0).contiguous()
    wt = torch.tensor([1.0, 100.0, 2000.0, 1000.0, 1000.0], device='cuda').expand(B, 5).contiguous()
    state = {'betas': betas.clone(), 'meas': meas.clone(), 'jac': jac.clone(), 'loss': torch.zeros(B, device='cuda'),
             'lambda': torch.ones(B, device='cuda'), 'accepted': torch.zeros(B, dtype=torch.int32, device='cuda')}
    trial = betas.clone()

    def step():
        ops.fit_lm_step(state, tg, wt, 0.0, 10.0, 3.0, False, trial, meas, jac)

    def iteration():
        vv = ops.smplx_forward_shape(packed, trial)
        m, j, _ = ops.measure_jacobian_betas(packed, lm, vv, faces)
        ops.fit_lm_step(state, tg, wt, 0.0, 10.0, 3.0, False, trial, m, j)

    arms = {'forward': lambda: ops.measure(lm, v_shaped=v, faces_i32=faces),
            'jacobian': lambda: ops.measure_jacobian_betas(packed, lm, v, faces),
            'composite': composite, 'lm_step': step, 'lm_iter': iteration}
    n = 20 if B <= 64 else 3
    t = time_arms(arms, n, reps)
    mass_bytes = 10 * 3 * packed.V * 4 * B
    return {'B': B, 'ms': t, 'composite_over_jacobian': [round(t['composite'][0] / t['jacobian'][1], 2),
                                                         round(t['composite'][1] / t['jacobian'][0], 2)],
            'lm_iterations_per_s': [round(1e3 / t['lm_iter'][1], 1), round(1e3 / t['lm_iter'][0], 1)],
            'mass_row_bytes_from_l2': mass_bytes,
            'mass_row_rate_at_jacobian_time_GBps': round(mass_bytes / (t['jacobian'][0] * 1e-3) / 1e9, 1)}


def fractions(res, tg):
    tgt = torch.stack([tg[k] for k in NAMES], 1)
    ok = torch.isfinite(tgt).all(1)
    meas = res['measurements']
    rel = ((meas - tgt).abs() / tgt.abs())[ok]
    return {'height_1mm': round(float(((meas[:, 1] - tgt[:, 1]).abs()[ok] < 1e-3).float().mean()), 4),
            'circ_0.5pct': round(float((rel[:, 2:] < 5e-3).all(1).float().mean()), 4),
            'mass_1pct': round(float((rel[:, 0] < 1e-2).float().mean()), 4),
            'median_loss': float(res['loss'][ok].median())}


def time_to_quality():
    from shapy_b200 import synth
    from shapy_b200.body_measurements import BodyMeasurements
    from shapy_b200.fit import fit_betas_to_measurements
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    smplx = SMPLX(data_struct=synth.make_smplx()).cuda()
    bm = BodyMeasurements({'landmarks': synth.load_landmarks()}).cuda()
    bstar = torch.randn(256, 10, generator=torch.Generator().manual_seed(21)).clamp(-2, 2).cuda()
    with torch.no_grad():
        m = bm.forward_vertices(smplx.forward_shape(betas=bstar)['v_shaped'], smplx.faces_i32)['measurements']
        tg = {k: m[k]['tensor'].clone() for k in NAMES}
    fit_betas_to_measurements(smplx, bm, tg, method='lm', iterations=2)     # warm-up
    fit_betas_to_measurements(smplx, bm, tg, iterations=2)
    out = {}
    for name, kw in (('lm_50', dict(method='lm', iterations=50)), ('adam_400', dict(iterations=400))):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = fit_betas_to_measurements(smplx, bm, tg, **kw)
        torch.cuda.synchronize()
        out[name] = dict(seconds=round(time.perf_counter() - t0, 4), **fractions(res, tg))
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
