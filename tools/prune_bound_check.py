"""Checks the closest-point prune bound of shapy_b200/csrc/bvh.cu on its float32 restatement (tests/bvh_f32_oracle.py)
over ten times the adversarial cases of tests/test_bvh_f32_oracle_cpu.py.

    python tools/prune_bound_check.py [--cases 2000000] [--seed 7]

Prints how many leaves the bound would let an equally near primitive prune (it must be 0), the largest k that a case
needs against the k = 64 of the bound and the 46 of its proof, and how many cases the former relative bound
best + 1e-5 best + 1e-12 gets wrong.  CPU only.
"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests'))
import bvh_f32_oracle as bo  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--cases', type=int, default=2_000_000)
    ap.add_argument('--seed', type=int, default=7)
    a = ap.parse_args()
    rng = np.random.default_rng(a.seed)
    bad = old = 0
    need = 0.0
    for s in range(0, a.cases, 200_000):
        p, x, y, z = bo.adversarial_cases(rng, min(200_000, a.cases - s))
        bx, d2, M, k = bo.prune_margin(p, x, y, z)
        bad += int((bx > bo.prune_bound(d2, M)).sum())
        old += int((bx > bo.relative_prune_bound(d2)).sum())
        need = max(need, float(np.nanmax(k)))
    print(json.dumps({'cases': a.cases, 'prunable_by_an_equal': bad, 'largest_k_needed': round(need, 3),
                      'k': 64, 'proof_k': 46, 'relative_bound_wrong': old}))
    return 1 if bad else 0


if __name__ == '__main__':
    sys.exit(main())
