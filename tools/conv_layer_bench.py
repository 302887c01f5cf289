"""Per-layer timing of the HRNet-W48 main convolutions at the bench batch (B=64, 224x224 input):
SHAPY_CONV_TEST_REPS launches of each plan; to stderr the average time per launch, the useful conv FLOP/s, and the
plan's TMA bytes and issued MMA FLOPs per launch with the rates they give at that time.  Layers named '+res' add a
residual of the output's shape in the epilogue (the Bottleneck / BasicBlock skip connection).  SHAPY_CONV_DEBUG=1 in the
environment prints each plan's path and tile configuration; SHAPY_CONV_HALO=0 times the per-tap path everywhere.
usage: python tools/conv_layer_bench.py [batch] [mode] [name,name,...]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ.setdefault('SHAPY_CONV_TEST_REPS', '20')
import torch
from shapy_b200 import ops

B = int(sys.argv[1]) if len(sys.argv) > 1 else 64
mode = int(sys.argv[2]) if len(sys.argv) > 2 else 1
which = sys.argv[3].split(',') if len(sys.argv) > 3 else None
LAYERS = {  # name: (cin, cout, k, stride, H[, residual])
    'c48': (48, 48, 3, 1, 56), 'c96': (96, 96, 3, 1, 28), 'c192': (192, 192, 3, 1, 14), 'c384': (384, 384, 3, 1, 7),
    'b64': (64, 64, 3, 1, 56), 'b1x1a': (256, 64, 1, 1, 56), 'b1x1b': (64, 256, 1, 1, 56),
    't48': (256, 48, 3, 1, 56), 'd96': (48, 96, 3, 2, 56), 'f1x1': (96, 48, 1, 1, 28),
    'd48': (48, 48, 3, 2, 56), 'd192': (48, 192, 3, 2, 28), 's2_96_192': (96, 192, 3, 2, 28),
    's2_64': (64, 64, 3, 2, 112), 's2_192_384': (192, 384, 3, 2, 14), 's2_256_96': (256, 96, 3, 2, 56),
    'c48+res': (48, 48, 3, 1, 56, True), 'c192+res': (192, 192, 3, 1, 14, True), 'b1x1b+res': (64, 256, 1, 1, 56, True),
    't2048': (2048, 2048, 1, 1, 7), 't512_2048+res': (512, 2048, 1, 1, 7, True), 't512': (512, 512, 3, 1, 7),
}
g = torch.Generator().manual_seed(0)
for name, (cin, cout, k, s, H, *res) in LAYERS.items():
    if which and name not in which:
        continue
    x = torch.randn(B, H, H, cin, generator=g).cuda()
    w = torch.randn(cout, cin, k, k, generator=g) * (1.0 / (cin * k * k) ** 0.5)
    sys.stderr.write(f'--- {name}\n')
    sys.stderr.flush()
    r = torch.randn(B, H // s, H // s, cout, generator=g).cuda() if res else None
    ops.conv_test(x, w, stride=s, res_nhwc=r, relu=True, mode=mode, engine=0)
