"""Where the time of a wgmma convolution tile goes: builds the cycle-stamp variant of the library (-DSHAPY_CONV_STAMPS,
which the default build leaves out) into OUT, then for each layer, precision mode and consumer schedule prints the
mean clock64 cycles per warpgroup-tile spent waiting for the first k-block, in the mainloop (first full-barrier pass
to the last commit; of that, the operand waits on the later k-blocks' full barriers), in the drain (last commit to the
return of wait<0>) and in the epilogue.  Cooperative tiles are
64-row halves issued by both consumers at once; ping-pong tiles are whole 128-row tiles of one consumer.
usage: python tools/conv_phase_stamps.py [--out DIR] [--layers c48,c96,...] [--reps N]"""
import argparse
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LAYERS = {'c48': (48, 48, 3, 1, 56), 'c96': (96, 96, 3, 1, 28), 'c192': (192, 192, 3, 1, 14),
          'c384': (384, 384, 3, 1, 7), 'b64': (64, 64, 3, 1, 56), 't48': (256, 48, 3, 1, 56)}
MODES = [(1, 64), (0, 32)]                                  # (mode, batch): split fp16 at B = 64, plain fp16 at B = 32
SCHEDULES = [('cooperative', 10), ('ping-pong', 20), ('planner', 0)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='build directory of the stamp variant (default: a temporary one)')
    ap.add_argument('--layers', default=','.join(LAYERS))
    ap.add_argument('--reps', type=int, default=20)
    a = ap.parse_args()
    out = a.out or tempfile.mkdtemp(prefix='shapy_stamps_')
    from shapy_b200 import build as b
    b.OBJ = os.path.join(out, 'obj')
    b.LIB = os.path.join(out, 'libshapy_b200_stamps.so')
    b.DEFS = b.DEFS + ['-DSHAPY_CONV_STAMPS']
    os.environ['SHAPY_B200_LIB'] = b.build()
    os.environ['SHAPY_CONV_TEST_REPS'] = str(a.reps)
    import torch
    from shapy_b200 import ops
    g = torch.Generator().manual_seed(0)
    for mode, B in MODES:
        for name in a.layers.split(','):
            cin, cout, k, s, H = LAYERS[name]
            x = torch.randn(B, H, H, cin, generator=g).cuda()
            w = torch.randn(cout, cin, k, k, generator=g) * (1.0 / (cin * k * k)) ** 0.5
            for sched, engine in SCHEDULES:
                sys.stderr.write(f'--- {name} mode {mode} B {B} {sched}\n')
                sys.stderr.flush()
                ops.conv_test(x, w, stride=s, relu=True, mode=mode, engine=engine)
                torch.cuda.synchronize()


if __name__ == '__main__':
    main()
