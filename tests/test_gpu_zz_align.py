"""Scale / root alignments of PointError (shapy_point_error_aligned) and the J14 regression of mpjpe14
(shapy_regress_points) on the device, against the reference's outputs (tests/golden/align.npz) and the float64 oracle."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import align_oracle as ao

pytestmark = pytest.mark.gpu
G = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'align.npz'))
ROOT_TAGS = ('r23', 'r0', 'rm1', 'rempty')


def rel(x, ref):
    """max |x - ref| over the largest |ref|, NaN in exactly the same places"""
    x, ref = np.asarray(x, np.float64), np.asarray(ref, np.float64)
    assert x.shape == ref.shape
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(x), nan)
    if nan.all():
        return 0.0
    return np.abs(x[~nan] - ref[~nan]).max() / np.abs(ref[~nan]).max()


def run(pe, est, gt):
    err = pe(torch.as_tensor(est).cuda(), torch.as_tensor(gt).cuda())
    assert err.is_cuda and err.dtype == torch.float32
    return err.cpu().numpy(), pe.last_mean.cpu().numpy()


def test_scale_matches_reference():
    from shapy_b200 import metrics
    err, mean = run(metrics.PointError(metrics.build_alignment('scale')), G['est'], G['gt'])
    ref = G['error_scale']
    assert rel(err, ref) < 2e-5            # both sides fp32: eps * |coordinate| / error
    assert rel(mean, ref.mean(1)) < 2e-5


@pytest.mark.parametrize('tag', ROOT_TAGS)
def test_root_matches_reference(tag):
    from shapy_b200 import metrics
    pe = metrics.PointError(metrics.build_alignment('root'))
    pe.set_root([int(r) for r in G[f'root_{tag}']])        # as _compute_mpjpe does (evaluation.py:146-153)
    err, mean = run(pe, G['j_est'], G['j_gt'])
    ref = G[f'error_root_{tag}']
    assert rel(err, ref) < 2e-5
    assert rel(mean, ref.mean(1)) < 2e-5


def test_mpjpe14_through_joint_regressor_matches_reference():
    from shapy_b200 import metrics
    joints = metrics.JointRegressor(G['j14'])(torch.from_numpy(G['j14_verts']).cuda())
    assert joints.shape == (3, 14, 3) and joints.dtype == torch.float32
    assert rel(joints.cpu().numpy(), G['j14_joints']) < 1e-6
    gt = torch.from_numpy(G['j14_gt']).cuda()
    for tag in ('root', 'scale'):
        pe = metrics.PointError(metrics.build_alignment(tag, root=[2, 3]))     # evaluation.py:616-619
        err = pe(joints, gt).cpu().numpy()
        ref = G[f'error_mpjpe14_{tag}']
        assert rel(err, ref) < 2e-5
        assert rel(pe.last_mean.cpu().numpy(), ref.mean(1)) < 2e-5


def test_root_alignment_of_three_points_reads_points_first():
    """RootAlignment indexes points in the reference whatever P is, so (B, 3, 3) is served (only scale refuses it)."""
    from shapy_b200 import metrics
    rng = np.random.default_rng(3)
    est = (rng.normal(0, 0.3, (4, 3, 3)) + 2.5).astype(np.float32)
    gt = (est + rng.normal(0, 0.05, (4, 3, 3))).astype(np.float32)
    err, _ = run(metrics.PointError(metrics.build_alignment('root', root=[1])), est, gt)
    assert rel(err, ao.root_error(est, gt, [1])) < 2e-5


@pytest.fixture(scope='module')
def smplx_size():
    """B = 64 synthetic SMPL-X-sized meshes (V = 10 475) about 2.5 m from the origin, gt ~ 1.1 x est + noise"""
    g = torch.Generator().manual_seed(41)
    B, V = 64, 10475
    offset = torch.tensor([0.3, 0.4, 2.5])
    est = torch.randn(B, V, 3, generator=g) * 0.4 + offset
    gt = (est - offset) * 1.1 + torch.randn(B, V, 3, generator=g) * 0.01 + offset + torch.randn(B, 1, 3, generator=g) * 0.05
    return est.cuda(), gt.cuda()


@pytest.mark.parametrize('name', ['scale', 'root'])
def test_smplx_size_matches_float64_oracle_and_is_batch_independent(smplx_size, name):
    from shapy_b200 import metrics
    est, gt = smplx_size
    pe = metrics.PointError(metrics.build_alignment(name, root=[2, 3]))
    err = pe(est, gt)
    mean = pe.last_mean
    e64, g64 = est.double().cpu().numpy(), gt.double().cpu().numpy()
    ref = ao.scale_error(e64, g64) if name == 'scale' else ao.root_error(e64, g64, [2, 3])
    assert rel(err.cpu().numpy(), ref) < 2e-5
    assert rel(mean.cpu().numpy(), ref.mean(1)) < 2e-5
    err2 = pe(est, gt)                                                     # run to run: bit-identical
    assert torch.equal(err, err2) and torch.equal(mean, pe.last_mean)
    for b in (0, 17, 63):                                                  # row b does not depend on the rest of the batch
        e1 = pe(est[b:b + 1], gt[b:b + 1])
        assert torch.equal(e1[0], err[b]) and torch.equal(pe.last_mean[0], mean[b])


def test_entry_point_rejects_bad_arguments_on_the_host():
    from shapy_b200 import _lib
    L = _lib.lib()
    B, P = 2, 14
    est, gt = torch.randn(B, P, 3, device='cuda'), torch.randn(B, P, 3, device='cuda')
    err, mean = torch.empty(B, P, device='cuda'), torch.empty(B, device='cuda')
    nbytes = L.shapy_point_error_workspace_bytes(B)
    ws = torch.empty(nbytes, dtype=torch.uint8, device='cuda')
    p = _lib.ptr

    def call(a, mode, roots, work=ws, n=None):
        r = (C.c_int * max(len(roots), 1))(*roots)
        return L.shapy_point_error_aligned(p(a), p(gt), B, P, mode, r, len(roots) if n is None else n, p(err), p(mean), p(work),
                                           nbytes, _lib.stream_ptr())

    torch.cuda.synchronize()
    n0 = L.shapy_launch_count()
    for args, msg in (((None, _lib.ALIGN_SCALE, []), 'null argument'), ((est, _lib.ALIGN_ROOT, [0], None), 'null argument'),
                      ((est, 0, []), 'unknown alignment mode'), ((est, 3, [0]), 'unknown alignment mode'),
                      ((est, _lib.ALIGN_ROOT, list(range(_lib.MAX_ROOTS + 1))), 'root indices'),
                      ((est, _lib.ALIGN_ROOT, [0], ws, -1), 'root indices'),
                      ((est, _lib.ALIGN_ROOT, [2, P]), 'out of range'), ((est, _lib.ALIGN_ROOT, [-P - 1]), 'out of range')):
        assert call(*args) == -1, msg
        assert msg in L.shapy_last_error().decode()
    assert L.shapy_regress_points(None, None, None, p(est), B, P, P, p(err), _lib.stream_ptr()) == -1
    assert L.shapy_launch_count() == n0                                    # nothing was launched
    torch.cuda.synchronize()                                               # and no CUDA error is pending
    assert call(est, _lib.ALIGN_ROOT, [-P, P - 1]) == 0                    # the extreme valid indices
    torch.cuda.synchronize()
    ref = ao.root_error(est.double().cpu().numpy(), gt.double().cpu().numpy(), [0, P - 1])
    assert rel(err.cpu().numpy(), ref) < 2e-5
