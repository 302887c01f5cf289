"""Timeline of one HRNet forward on the lane executor (SHAPY_HRNET_TRACE): per-lane busy time, the span of every
HighResolutionModule / fuse stage and the gaps.  usage: python tools/hrnet_trace.py [batch] [out.txt]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
out = sys.argv[2] if len(sys.argv) > 2 else 'gpurun_out/hrnet_trace.txt'
os.environ['SHAPY_HRNET_TRACE'] = out
import torch
from shapy_b200 import synth
B = int(sys.argv[1]) if len(sys.argv) > 1 else 64
bb = synth.build_synthetic_regressor().backbone.cuda().eval()
x = torch.randn(B, 3, 224, 224, device='cuda')
for _ in range(3):
    bb(x)['concat']
torch.cuda.synchronize()
rows = [l.split() for l in open(out)]
ops = [dict(i=int(r[0]), lane=int(r[1]), kind=int(r[2]), cin=int(r[3]), cout=int(r[4]), k=int(r[5]), s=int(r[6]), div=int(r[7]),
            t0=float(r[8]), t1=float(r[9])) for r in rows]
end = max(o['t1'] for o in ops)
print(f'forward span {end:.1f} us, {len(ops)} ops')
for lane in range(4):
    lo = [o for o in ops if o['lane'] == lane]
    if lo:
        busy = sum(o['t1'] - o['t0'] for o in lo)
        print(f'lane {lane}: {len(lo)} ops, sum(end-start) {busy:.0f} us, first {min(o["t0"] for o in lo):.0f} last {max(o["t1"] for o in lo):.0f}')
# coarse timeline: 100-us buckets, number of lanes with an op in flight
import math
nb = int(math.ceil(end / 100.0))
occ = [[0.0] * 4 for _ in range(nb)]
for o in ops:
    b0, b1 = int(o['t0'] // 100), int(min(o['t1'], end - 1e-6) // 100)
    for b in range(b0, b1 + 1):
        lo_, hi_ = max(o['t0'], b * 100.0), min(o['t1'], (b + 1) * 100.0)
        occ[b][o['lane']] += max(0.0, hi_ - lo_)
print('bucket(100us): in-flight fraction per lane')
for b in range(nb):
    print(f'{b * 100:6d} ' + ' '.join(f'{v / 100:.2f}' for v in occ[b]))
# per-family share: sum of (end - start) of every op of the family over that of all ops (lanes overlap, so the sum
# exceeds the span; the share is of the summed op time)
fam = {}
for o in ops:
    key = f'conv {o["cin"]}->{o["cout"]} k{o["k"]} s{o["s"]} /{o["div"]}' if o['kind'] in (0, 1) else f'kind {o["kind"]} /{o["div"]}'
    n, t = fam.get(key, (0, 0.0))
    fam[key] = (n + 1, t + o['t1'] - o['t0'])
tot = sum(t for _, t in fam.values())
print(f'per family: count, sum(end-start) us, share of {tot:.0f} us')
for key, (n, t) in sorted(fam.items(), key=lambda kv: -kv[1][1]):
    print(f'{key:32s} {n:4d} {t:9.0f} {100 * t / tot:6.1f} %')
