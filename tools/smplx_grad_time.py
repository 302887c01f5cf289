#!/usr/bin/env python
"""Device time of the posed SMPL-X forward + backward (shapy_smplx_forward, shapy_smplx_backward) at n_rot = 22, its
per-kernel split (torch.profiler, a separate run), and the iterations per second of fit_body_to_keypoints.

    python tools/smplx_grad_time.py [--batches 64 4096] [--json out.json]

Algorithmic bytes of the backward, from shapes (not measured): the posedirs rows below Kp = 9 (n_rot - 1) read once
(Kp x 3V fp32), plus per body four (V, 3) fp32 streams of 3V x 4 bytes (the vertex cotangent in, v_posed, its
cotangent and the cotangent of v_posed written once each).  The rate is those bytes over the measured backward time,
against the 3.35 TB/s HBM3 of the H100 SXM data sheet."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from shapy_b200 import ops, synth  # noqa: E402

PEAK = 3.35e12


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def inputs(B, n_rot=22, seed=0):
    g = torch.Generator().manual_seed(seed)
    raw = (torch.randn(B, 6 * n_rot, generator=g) * 0.3 + synth.mean_params()[:6 * n_rot]).cuda()
    return dict(betas=torch.randn(B, 10, generator=g).cuda(), rot=ops.decode_rot6d(raw),
                expr=torch.randn(B, 10, generator=g).cuda(), camera=torch.tensor([[0.9, 0.0, 0.0]]).repeat(B, 1).cuda())


def timed(fn, reps=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--batches', type=int, nargs='*', default=[64, 4096])
    p.add_argument('--fit-batches', type=int, nargs='*', default=[256, 4096])
    p.add_argument('--json', type=str, default=None)
    a = p.parse_args()
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    module = SMPLX(data_struct=synth.make_smplx(), use_face_contour=True).cuda()
    packed = module.packed()
    V3, K = packed.V * 3, packed.K
    res = {'card': card(), 'n_rot': 22, 'batches': {}}
    for B in a.batches:
        x = inputs(B)
        g = torch.Generator(device='cuda').manual_seed(1)
        cot = dict(grad_vertices=torch.randn(B, packed.V, 3, device='cuda', generator=g),
                   grad_v_shaped=torch.randn(B, packed.V, 3, device='cuda', generator=g),
                   grad_joints=torch.randn(B, K, 3, device='cuda', generator=g),
                   grad_proj_joints=torch.randn(B, K, 2, device='cuda', generator=g))
        fwd = lambda: ops.smplx_forward(packed, x['betas'], x['rot'], expr=x['expr'], camera=x['camera'])  # noqa: E731
        bwd = lambda: ops.smplx_backward(packed, x['betas'], x['rot'], x['expr'], x['camera'], **cot)  # noqa: E731
        t_f, t_f_min = timed(fwd)
        t_b, t_b_min = timed(bwd)
        Kp = 9 * 21
        nbytes = Kp * V3 * 4 + B * 4 * V3 * 4
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                bwd()
            torch.cuda.synchronize()
        kernels = {}
        for e in prof.key_averages():
            if e.device_time_total > 0:
                kernels[e.key[:80]] = round(e.device_time_total / max(e.count, 1) / 1.0, 1)
        r = {'forward_us': round(t_f, 1), 'forward_min_us': round(t_f_min, 1), 'backward_us': round(t_b, 1),
             'backward_min_us': round(t_b_min, 1), 'forward_plus_backward_us': round(t_f + t_b, 1),
             'algorithmic_bytes': nbytes, 'bytes_bound_us': round(nbytes / PEAK * 1e6, 1),
             'backward_fraction_of_hbm_peak': round(nbytes / PEAK / (t_b * 1e-6), 3),
             'kernels_us_per_call': dict(sorted(kernels.items(), key=lambda kv: -kv[1]))}
        res['batches'][B] = r
        print(f'B {B}: forward {t_f:.1f} us, backward {t_b:.1f} us (min {t_b_min:.1f}); algorithmic '
              f'{nbytes / 1e6:.1f} MB -> {r["backward_fraction_of_hbm_peak"]:.3f} of {PEAK / 1e12:.2f} TB/s', flush=True)
        for k, v in r['kernels_us_per_call'].items():
            print(f'    {v:9.1f} us  {k}')
    from shapy_b200.fit import fit_body_to_keypoints
    res['fit_iterations_per_s'] = {}
    for B in a.fit_batches:
        x = inputs(B, seed=2)
        with torch.no_grad():
            kp = module(global_rot=x['rot'][:, :1], body_pose=x['rot'][:, 1:], betas=x['betas'])['joints'][:].clone()
        fit_body_to_keypoints(module, kp, iterations=3)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n = 30
        e0.record()
        fit_body_to_keypoints(module, kp, iterations=n)
        e1.record()
        torch.cuda.synchronize()
        ips = n / (e0.elapsed_time(e1) * 1e-3)
        res['fit_iterations_per_s'][B] = round(ips, 1)
        print(f'fit_body_to_keypoints B {B}: {ips:.1f} iterations/s (incl. one final evaluation)', flush=True)
    print(json.dumps(res))
    if a.json:
        with open(a.json, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
