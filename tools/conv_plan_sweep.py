"""Checks the wgmma planner against the clock: for every distinct convolution HighResolutionNet.build_program() emits
(at the bench input, 224 x 224), in split fp16 at B = 64 and plain fp16 at B = 32, times every feasible (cout tile,
consumer schedule) pair on the data path the planner takes for that layer (the choice between the per-tap and the halo
path reorders fp32 sums, so it is not swept), with CUDA events over --reps back-to-back launches per candidate, the
candidates of a layer alternating over --rounds rounds (the fastest round counts).  Prints the card's name and power
limit, then per layer the planner's pick, the fastest candidate and the gap between them.  --stamps builds the
cycle-stamp variant of the library (-DSHAPY_CONV_STAMPS) into a temporary directory and also prints each candidate's
mean cycles per warpgroup-tile: wait before the first k-block / mainloop / drain / epilogue (tools/conv_phase_stamps.py).
--list prints the layers and their candidates and needs no device.
Outputs land in dense NHWC buffers; the few layers the network writes into a slice of the concatenated tensor are
timed with the same boxes.
usage: python tools/conv_plan_sweep.py [--modes 1,0] [--layers i,j,...] [--reps N] [--rounds R] [--stamps] [--list]"""
import argparse
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MODES = {1: 64, 0: 32}                     # precision mode -> bench batch: split fp16 at B = 64, plain fp16 at B = 32
NTS = (128, 96, 64, 48, 32, 16)            # cout tiles with a kernel instantiation (conv_wgmma.cu kNts)
COOP, PINGPONG = 10, 20                    # conv_test engine digits of the forced schedules
SIZE = 224


def layers():
    """Distinct (cin, cout, k, stride, H_in, residual) of the program's wgmma convolutions, with their launch counts."""
    from shapy_b200 import synth
    from shapy_b200._lib import OP_CONV
    convs, ops, slots, _, _ = synth.build_synthetic_regressor().backbone.build_program()
    count = {}
    for o in ops:
        if o['kind'] != OP_CONV:
            continue
        c = convs[o['conv']]
        key = (c['cin'], c['cout'], c['ksize'], c['stride'], SIZE // slots[o['in_slot']]['div'], o['res_slot'] >= 0)
        count[key] = count.get(key, 0) + 1
    # the engine's shape limits (wgmma_supported); the rest run on the SIMT engine
    return [(k, n) for k, n in count.items() if k[0] % 16 == 0 and k[1] % 16 == 0]


def candidates(cout, mode):
    out = []
    for nt in NTS:
        if cout % nt or (mode and nt > 96):
            continue
        out.append((nt, 'cooperative'))
        if nt <= (64 if mode else 128):          # pingpong_fits
            out.append((nt, 'ping-pong'))
    return out


def name(key):
    cin, cout, k, s, H, res = key
    return f'{cin}->{cout} {k}x{k} s{s} @{H // s}' + (' +res' if res else '')


class StderrCapture:
    """The library reports on the C stderr: route fd 2 into a file for the duration of one call."""
    def __enter__(self):
        sys.stderr.flush()
        self.f = tempfile.TemporaryFile(mode='w+')
        self.saved = os.dup(2)
        os.dup2(self.f.fileno(), 2)
        return self

    def __exit__(self, *a):
        sys.stderr.flush()
        os.dup2(self.saved, 2)
        os.close(self.saved)
        self.f.seek(0)
        self.text = self.f.read()
        self.f.close()


PATHS = {2: 'per-tap', 3: 'halo', 4: 'resident'}   # ops.ConvPlan digits
SCHEDULES = {1: 'cooperative', 2: 'ping-pong'}
TIME_RE = re.compile(r'\[conv_test\].*?: ([\d.]+) us/launch')
STAMP_RE = re.compile(r'wait (\d+) mainloop (\d+) \(operand waits \d+\) drain (\d+) epilogue (\d+)')


def run(ops, torch, x, w, r, s, mode, engine):
    with StderrCapture() as cap:
        _, plan = ops.conv_test(x, w, stride=s, res_nhwc=r, relu=True, mode=mode, engine=engine, report=True)
        torch.cuda.synchronize()
    t = TIME_RE.findall(cap.text)
    if not t:
        raise RuntimeError(f'conv_test engine {engine}: no timing line in\n{cap.text}')
    st = STAMP_RE.findall(cap.text)
    return (PATHS[plan.path], plan.nt, SCHEDULES[plan.schedule]), float(t[-1]), ('/'.join(st[-1]) if st else '')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--modes', default='1,0', help='precision modes: 1 = split fp16 (B = 64), 0 = plain fp16 (B = 32)')
    ap.add_argument('--layers', default=None, help='indices into the layer list (see --list)')
    ap.add_argument('--reps', type=int, default=50, help='launches timed per candidate and round (at least 20)')
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--stamps', action='store_true')
    ap.add_argument('--list', action='store_true')
    a = ap.parse_args()
    if a.reps < 20:
        ap.error('--reps must be at least 20')
    modes = [int(m) for m in a.modes.split(',')]
    if a.stamps and not a.list:              # before the first import of the library picks its path
        out = tempfile.mkdtemp(prefix='shapy_sweep_stamps_')
        from shapy_b200 import build as b
        b.OBJ = os.path.join(out, 'obj')
        b.LIB = os.path.join(out, 'libshapy_b200_stamps.so')
        b.DEFS = b.DEFS + ['-DSHAPY_CONV_STAMPS']
        os.environ['SHAPY_B200_LIB'] = b.build()
    ls = layers()
    pick = [int(i) for i in a.layers.split(',')] if a.layers else range(len(ls))
    if a.list:
        for i, (key, n) in enumerate(ls):
            print(f'{i:3d} {name(key):32s} x{n:<3d}',
                  ' | '.join(f'mode {m}: ' + ' '.join(f'{nt}{sc[0]}' for nt, sc in candidates(key[1], m)) for m in modes))
        return
    os.environ['SHAPY_CONV_TEST_REPS'] = str(a.reps)
    import torch
    from shapy_b200 import ops
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip()
    print(f'device: {torch.cuda.get_device_name()} | nvidia-smi: {q} | {a.reps} launches x {a.rounds} rounds'
          + (' | stamp build' if a.stamps else ''), flush=True)
    g = torch.Generator().manual_seed(0)
    for mode in modes:
        B = MODES[mode]
        for i in pick:
            (cin, cout, k, s, H, res), n = ls[i]
            x = torch.randn(B, H, H, cin, generator=g).cuda()
            w = torch.randn(cout, cin, k, k, generator=g) * (1.0 / (cin * k * k)) ** 0.5
            r = torch.randn(B, H // s, H // s, cout, generator=g).cuda() if res else None
            planned, _, _ = run(ops, torch, x, w, r, s, mode, 0)
            best = {}
            for _ in range(a.rounds):
                for nt, sc in candidates(cout, mode):
                    try:
                        got, us, st = run(ops, torch, x, w, r, s, mode, nt * 100 + (COOP if sc == 'cooperative' else PINGPONG))
                    except RuntimeError as e:   # no room for the staging boxes, or no kernel: not a candidate
                        best.setdefault((nt, sc), (None, str(e).splitlines()[0][:80], ''))
                        continue
                    if got[1] != nt or got[2] != sc:
                        raise RuntimeError(f'forced {nt} {sc}, planned {got}')
                    prev = best.get((nt, sc))
                    if prev is None or prev[0] is None or us < prev[0]:
                        best[(nt, sc)] = (us, got[0], st)
            timed = {c: v for c, v in best.items() if v[0] is not None}
            fast = min(timed, key=lambda c: timed[c][0])
            mine = (planned[1], planned[2])
            gap = timed[mine][0] / timed[fast][0] - 1 if mine in timed else float('nan')
            print(f'mode {mode} B {B} [{i}] {name(ls[i][0])} x{n} ({planned[0]}): planned NT {mine[0]} {mine[1]} '
                  f'{timed[mine][0] if mine in timed else float("nan"):.2f} us, fastest NT {fast[0]} {fast[1]} '
                  f'{timed[fast][0]:.2f} us, gap {100 * gap:+.1f} %', flush=True)
            for c in candidates(cout, mode):
                us, info, st = best[c]
                print(f'    NT {c[0]:3d} {c[1]:11s} ' + (f'{us:8.2f} us' + (f'  stamps {st}' if st else '')
                                                       if us is not None else f'   -      {info}'), flush=True)


if __name__ == '__main__':
    main()
