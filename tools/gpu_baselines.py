"""Same-box GPU baselines SURVEY.md 8d asks for (a tool, not part of bench.py: it executes oracle/ code on the GPU).

  1. The reference's HRNet graph on this GPU through stock PyTorch / cuDNN (oracle.net_oracle.hrnet_forward: the same
     conv2d / batch_norm / relu / interpolate call sequence as regressor/human_shape/models/backbone/hrnet.py), B = 64,
     224 x 224, three settings: fp32 (TF32 off), TF32 convolutions, fp16 autocast.
  2. The reference's own BVH kernel (oracle/_ref, mesh_mesh_intersect_cuda_op.cu patched for torch 2.11) on the
     measurement query of BASELINE configs[3] (2 plane triangles against the 20 908 body triangles, 3 planes per body),
     next to shapy_mmi_forward on the same inputs and to the fused measurement kernel that replaces all of it.
  3. The same operator in float64 and float32, reference and shapy_b200, on those planes and on the seeded triangle
     soup of tests/test_gpu_zz_reference_op.py (float32) / tests/test_mmi_f64_cpu.py (float64).

    python tools/gpu_baselines.py        # one JSON document on stdout
"""
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from oracle import net_oracle
from shapy_b200 import ops, synth


def timed(fn, n=5, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def time_reference(query, target, M, reps=3):
    """ms per call of the reference operator (oracle/time_ref_mmi.py, its own process), or the error text."""
    with tempfile.TemporaryDirectory() as td:
        inp, outp = os.path.join(td, 'in.npz'), os.path.join(td, 'out.json')
        np.savez(inp, query=query, target=target, max_collisions=np.int64(M))
        r = subprocess.run([sys.executable, os.path.join(ROOT, 'oracle', 'time_ref_mmi.py'), inp, outp, str(reps)],
                           capture_output=True, text=True, timeout=600)
        if r.returncode == 0 and os.path.exists(outp):
            return json.load(open(outp))['ms_per_call']
        return (r.stderr or r.stdout)[-300:]


def power_limit():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True)
    return r.stdout.strip() if r.returncode == 0 else 'unknown'


def main():
    out = {'gpu': torch.cuda.get_device_name(0), 'nvidia_smi_name_power_limit': power_limit()}
    model = synth.build_synthetic_regressor()
    sd = {k[9:]: v.cuda() for k, v in model.state_dict().items() if k.startswith('backbone.')}
    B = 64
    x = torch.randn(B, 3, 224, 224, device='cuda')
    res = {}
    with torch.no_grad():
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        res['pytorch_cudnn_fp32_ms'] = timed(lambda: net_oracle.hrnet_forward(sd, x))
        torch.backends.cudnn.allow_tf32 = True
        res['pytorch_cudnn_tf32_ms'] = timed(lambda: net_oracle.hrnet_forward(sd, x))
        torch.backends.cudnn.benchmark = True
        res['pytorch_cudnn_tf32_benchmark_ms'] = timed(lambda: net_oracle.hrnet_forward(sd, x))
        with torch.autocast('cuda', dtype=torch.float16):
            res['pytorch_cudnn_fp16_autocast_ms'] = timed(lambda: net_oracle.hrnet_forward(sd, x))
        torch.backends.cudnn.benchmark = False
    bb = model.backbone.cuda().eval()
    res['shapy_b200_split_fp16_ms'] = timed(lambda: bb(x)['concat'], n=10, warm=3)
    bb.precision_mode = 0
    bb.invalidate()
    res['shapy_b200_fp16_ms'] = timed(lambda: bb(x)['concat'], n=10, warm=3)
    out['hrnet_B64_224'] = {k: round(v, 3) for k, v in res.items()}
    out['hrnet_B64_224']['images_per_s'] = {k[:-3]: round(B / (v * 1e-3), 1) for k, v in res.items()}

    # ---- measurement path: reference BVH kernel vs shapy_mmi_forward vs the fused measurement kernel
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'img00_body.npz'))
    lm = synth.load_landmarks()
    nb = 64
    bodies = np.concatenate([g['v_shaped'][None], g['extra_v_shaped']], 0).astype(np.float32)
    bodies = bodies[np.arange(nb) % bodies.shape[0]] * (1.0 + 0.02 * np.sin(np.arange(nb)))[:, None, None].astype(np.float32)
    tris = np.ascontiguousarray(bodies[:, g['faces']])
    meas = {}
    per_plane_ref, per_plane_ours = [], []
    f64 = {'reference_f64': [], 'shapy_f64': [], 'reference_f32': [], 'shapy_f32': []}
    for name in ('chest', 'waist', 'hips'):
        qs = []
        for b in range(nb):
            h = float((tris[b, lm[name]['face_idx']] * np.float32(lm[name]['bc'])[:, None]).sum(0)[1])
            quad = np.float32([[-1, h, -1], [1, h, -1], [1, h, 1], [-1, h, 1]])
            qs.append(np.stack([quad[[0, 1, 2]], quad[[0, 2, 3]]]))
        query = np.stack(qs).astype(np.float32)
        with tempfile.TemporaryDirectory() as td:
            inp, outp = os.path.join(td, 'in.npz'), os.path.join(td, 'out.json')
            np.savez(inp, query=query, target=tris, max_collisions=np.int64(256))
            r = subprocess.run([sys.executable, os.path.join(ROOT, 'oracle', 'time_ref_mmi.py'), inp, outp, '3'],
                               capture_output=True, text=True, timeout=600)
            if r.returncode == 0 and os.path.exists(outp):
                per_plane_ref.append(json.load(open(outp))['ms_per_call'])
            else:
                meas['reference_kernel_error'] = (r.stderr or r.stdout)[-300:]
        q_d, t_d = torch.from_numpy(query).cuda(), torch.from_numpy(tris).cuda()
        per_plane_ours.append(timed(lambda: ops.mesh_to_mesh_forward(q_d, t_d, 256), n=10))
        f64['reference_f32'].append(per_plane_ref[-1] if len(per_plane_ref) == len(per_plane_ours) else float('nan'))
        f64['shapy_f32'].append(per_plane_ours[-1])
        q64, t64 = query.astype(np.float64), tris.astype(np.float64)
        r = time_reference(q64, t64, 256)
        f64['reference_f64'].append(r if isinstance(r, float) else float('nan'))
        q_d, t_d = torch.from_numpy(q64).cuda(), torch.from_numpy(t64).cuda()
        f64['shapy_f64'].append(timed(lambda: ops.mesh_to_mesh_forward(q_d, t_d, 256), n=10))
        del q_d, t_d
    if len(per_plane_ref) == 3:
        meas['reference_bvh_kernel_ms_3_planes_64_bodies'] = round(sum(per_plane_ref), 3)
        meas['reference_note'] = 'BVH build + traversal only; the reference then runs scipy ConvexHull per body and plane on the CPU'
    meas['shapy_mmi_forward_ms_3_planes_64_bodies'] = round(sum(per_plane_ours), 4)
    v_d = torch.from_numpy(bodies).cuda()
    f_d = torch.from_numpy(g['faces']).to(torch.int32).cuda()
    lmk = ops.make_landmarks(lm)
    meas['shapy_measure_kernel_ms_64_bodies_all_5_measurements'] = round(timed(lambda: ops.measure(lmk, v_shaped=v_d, faces_i32=f_d), n=20), 4)
    out['measurements_64_bodies'] = meas
    dtypes = {'3_planes_64_bodies_ms': {k: round(sum(v), 4) for k, v in f64.items()}}
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    import test_gpu_zz_reference_op as t32
    import test_mmi_f64_cpu as t64
    soup = {}
    for tag, (q, t, M) in (('f32', t32.soup_inputs()), ('f64', t64.soup_inputs_f64())):
        r = time_reference(q, t, M, reps=10)
        soup[f'reference_{tag}'] = round(r, 4) if isinstance(r, float) else r
        q_d, t_d = torch.from_numpy(q).cuda(), torch.from_numpy(t).cuda()
        soup[f'shapy_{tag}'] = round(timed(lambda: ops.mesh_to_mesh_forward(q_d, t_d, M), n=20), 4)
    dtypes['soup_B2_Q96_F400_ms'] = soup
    out['mesh_to_mesh_forward_by_dtype'] = dtypes
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
