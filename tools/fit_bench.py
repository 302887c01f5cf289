#!/usr/bin/env python
"""Device time of the kernels of a betas -> measurements fitting step, and fit iterations per second; one JSON line.

    python tools/fit_bench.py [--reps 5] [--iters 50]

Per batch size (64 and 4096 bodies of the seeded synthetic SMPL-X model): shape forward, measure forward, measure
backward (vertices entry) and shape backward, each timed with CUDA events over `--iters` launches; the arms are run
`--reps` times alternating and reported as [min, max].  HBM fractions are the algorithmic bytes over the time at the
H100 SXM's 3.35 TB/s: measure backward reads a body's vertices (125.7 KB) once per phase-0 stage and once per
gradient pass and writes its gradient (125.7 KB) = 251 KB per body; shape backward reads the (B, 3V) gradient once.
The CPU oracle's gradient of one body (oracle/measure_grad_oracle.measure_grad, a CPU port) is timed on the host for scale.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM = 3.35e12


def card():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f'unknown ({type(e).__name__})'


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--iters', type=int, default=50)
    a = ap.parse_args()
    from shapy_b200 import ops, synth
    from shapy_b200.body_measurements import BodyMeasurements
    from shapy_b200.fit import fit_betas_to_measurements
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    name = card()
    d = synth.make_smplx()
    packed = ops.SmplxModel(dict(d), 'cuda')
    faces = d['faces_tensor'].to(torch.int32).cuda()
    lm = ops.make_landmarks(synth.load_landmarks())
    res = {'card': name, 'bodies': {}}
    for B in (64, 4096):
        betas = torch.randn(B, 10, generator=torch.Generator().manual_seed(B)).clamp(-2, 2).cuda()
        vs = ops.smplx_forward_shape(packed, betas)
        go = torch.ones(B, 5, device='cuda')
        gv = torch.randn(B, packed.V, 3, device='cuda')
        arms = {'shape_forward': lambda: ops.smplx_forward_shape(packed, betas),
                'measure_forward': lambda: ops.measure(lm, v_shaped=vs, faces_i32=faces),
                'measure_backward_vertices': lambda: ops.measure_backward(lm, go, v_shaped=vs, faces_i32=faces),
                'shape_backward': lambda: ops.smplx_backward_shape(packed, gv)}
        t = {k: [] for k in arms}
        for _ in range(a.reps):
            for k, fn in arms.items():
                t[k].append(timed(fn, a.iters))
        r = {k: [round(min(v), 4), round(max(v), 4)] for k, v in t.items()}
        mb = B * 2 * packed.V * 12
        sb = B * packed.V * 12
        r['measure_backward_hbm_fraction'] = round(mb / HBM * 1e3 / min(t['measure_backward_vertices']), 3)
        r['shape_backward_hbm_fraction'] = round(sb / HBM * 1e3 / min(t['shape_backward']), 3)
        res['bodies'][str(B)] = r
    smplx = SMPLX(data_struct=d).cuda()
    bm = BodyMeasurements({'landmarks': synth.load_landmarks()}).cuda()
    for B in (64, 4096):
        tg = {'height': 1.75, 'mass': 70.0, 'chest': 0.95, 'waist': 0.85, 'hips': 1.0}
        fit_betas_to_measurements(smplx, bm, tg, iterations=2, batch_size=B)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fit_betas_to_measurements(smplx, bm, tg, iterations=20, batch_size=B)
        torch.cuda.synchronize()
        res['bodies'][str(B)]['fit_iterations_per_s'] = round(20 / (time.perf_counter() - t0), 2)
    from oracle import measure_grad_oracle
    v0 = vs[0].cpu().numpy()
    t0 = time.perf_counter()
    measure_grad_oracle.measure_grad(v0, d['faces_tensor'].numpy(), [1, 1, 1, 1, 1], synth.load_landmarks())
    res['cpu_port_oracle_grad_one_body_s'] = round(time.perf_counter() - t0, 3)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
