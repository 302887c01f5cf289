"""Times ops.closest_points, the triangle query of the scan fits, on posed synthetic SMPL-X bodies (20 908 faces).

    python tools/scan_query_bench.py [--reps 7] [--out scan_query_bench.json]

Two scenes: the 4 bodies x 512 points of tests/test_gpu_scan.py, and 64 bodies x 8192 points of the same recipe (half
on the surface, 3/8 up to 5 cm off it, 1/8 up to 1 m away).  Per scene, with CUDA events, [min, max] over the reps of
the mean time per call (milliseconds) of a call that builds the tree and of one that refits a tree built earlier.  To
compare two builds of the library, run it once per build (SHAPY_B200_LIB=<path>), alternating.  The card's name and
power limit are read in the same run.
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


def scene(B, N, seed):
    from test_gpu_scan import _bodies, _model, _points
    v = _bodies(B, seed)
    return v, _model().faces_i32, _points(v, N, seed + 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=7)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    from shapy_b200 import _lib, ops
    res = {'card': card(), 'lib': os.path.basename(_lib.LIB_PATH)}
    for B, N, n in ((4, 512, 200), (64, 8192, 20)):
        v, faces, p = scene(B, N, 1)
        tree = ops.ScanTree()
        ops.closest_points(v, faces, p, tree=tree)
        res[f'B{B}_N{N}'] = time_arms({'build': lambda: ops.closest_points(v, faces, p),
                                       'refit': lambda: ops.closest_points(v, faces, p, tree=tree)}, n, a.reps)
    print(json.dumps(res))
    if a.out:
        with open(a.out, 'w') as fh:
            json.dump(res, fh, indent=1)


if __name__ == '__main__':
    main()
