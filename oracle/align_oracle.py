"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference's scale / root alignments of PointError and of the J14
joint regression of the mpjpe14 metric, plus the build of oracle/align_host.cpp.

Only tests/ may import this file.

Reference: regressor/human_shape/utils/metrics.py
    ScaleAlignment   173-229   mu1, mu2 = means; var1, var2 = centred sums of squares; s = sqrt(var2 / var1);
                               t = mu2 - s mu1; est' = s est + t
    RootAlignment    279-303   both sides minus the mean of their points listed in `root` (default [0])
    point_error       31-53    sqrt(((est' - gt') ** 2).sum(-1))
regressor/human_shape/evaluation.py:161-190 (_compute_mpjpe14): np.einsum('jv,bvn->bjn', J14_regressor, vertices).

Pinned: tests/golden/align.npz holds outputs of the reference's own classes (loaded by path by tools/make_golden.py
align); tests/test_align_cpu.py checks this file against them.
"""
import os
import subprocess
import warnings

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))


def scale_error(est, gt):
    """PointError(ScaleAlignment()) for (B, P, 3) points with P != 3 -> (B, P), float64."""
    est, gt = np.asarray(est, np.float64), np.asarray(gt, np.float64)
    mu1, mu2 = est.mean(1, keepdims=True), gt.mean(1, keepdims=True)
    var1, var2 = ((est - mu1) ** 2).sum((1, 2)), ((gt - mu2) ** 2).sum((1, 2))
    s = np.sqrt(var2 / var1)[:, None, None]
    return np.sqrt(((s * est + (mu2 - s * mu1) - gt) ** 2).sum(-1))


def root_error(est, gt, root):
    """PointError(RootAlignment(root)) -> (B, P), float64.  numpy indexing: negative indices count from the end, an
    out-of-range index raises IndexError, an empty list gives NaN (the mean of an empty axis)."""
    est, gt = np.asarray(est, np.float64), np.asarray(gt, np.float64)
    root = np.asarray(root, np.int64).reshape(-1)
    with warnings.catch_warnings(), np.errstate(invalid='ignore'):
        warnings.simplefilter('ignore', RuntimeWarning)         # "Mean of empty slice"
        ra, rc = est[:, root].mean(1, keepdims=True), gt[:, root].mean(1, keepdims=True)
    return np.sqrt((((est - ra) - (gt - rc)) ** 2).sum(-1))


def regress_joints(regressor, vertices):
    """(J, V) regressor, (B, V, 3) vertices -> (B, J, 3) float64, the einsum of evaluation.py:183-184."""
    return np.einsum('jv,bvn->bjn', np.asarray(regressor, np.float64), np.asarray(vertices, np.float64))


def build_align_host(out_dir: str) -> str:
    """Compiles oracle/align_host.cpp (the per-point functions of shapy_b200/csrc/metrics.cuh for the host) into
    out_dir/libalign_host.so."""
    out = os.path.join(out_dir, 'libalign_host.so')
    subprocess.check_call(['g++', '-O2', '-ffp-contract=off', '-fno-fast-math', '-shared', '-fPIC', '-o', out,
                           os.path.join(_HERE, 'align_host.cpp')])
    return out
