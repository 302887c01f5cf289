"""Device time of the SMPL-X forward (pose kernel, wgmma pose-blend GEMM, vertex and joints kernels) at a few batch sizes.
usage: python tools/lbs_time.py [B ...]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from shapy_b200 import ops, synth
model = synth.build_synthetic_regressor().cuda().eval()
packed = model.model.packed(torch.device('cuda'))
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device='cuda')
flush2 = torch.zeros(64 * 1024 * 1024, dtype=torch.float32, device='cuda')
for B in [int(a) for a in sys.argv[1:]] or [64, 4096]:
    betas = torch.randn(B, 10, device='cuda')
    rot = ops.decode_rot6d(torch.randn(B, 132, device='cuda') * 0.3 + synth.mean_params()[:132].cuda())
    for _ in range(3):
        ops.smplx_forward(packed, betas, rot)
    torch.cuda.synchronize()
    if os.environ.get('LBS_PROF'):
        from torch.profiler import profile, ProfilerActivity
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                flush.zero_()
                ops.smplx_forward(packed, betas, rot)
            torch.cuda.synchronize()
        for e in prof.key_averages():
            if 'shapy' not in e.key: continue
            print(f'   {e.key[:60]:60s} n={e.count} avg {e.device_time_total / max(e.count, 1):.1f} us')
    ts = []
    clean = os.environ.get('LBS_CLEAN_FLUSH')
    for _ in range(20):
        flush.zero_()
        if clean:      # leave the L2 full of CLEAN lines of another buffer (a read pass) instead of dirty ones
            flush2.sum()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); ops.smplx_forward(packed, betas, rot); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ms = sum(ts) / len(ts)
    gbs = (68.93e6 + B * 254896) / (ms * 1e-3) / 1e9
    print(f'B {B}: {ms * 1e3:.1f} us (min {min(ts) * 1e3:.1f}), algorithmic {gbs:.0f} GB/s = {gbs / 3350.0:.3f} of the 3.35 TB/s H100 HBM3 data-sheet peak')
