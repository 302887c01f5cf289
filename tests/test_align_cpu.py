"""Scale / root alignments of PointError and the J14 regression of mpjpe14, CPU side: the numpy restatement, the
host-compiled copy of the kernels' per-point functions and the host logic of the mirror, against outputs of the
REFERENCE's own classes (tests/golden/align.npz, written by tools/make_golden.py align)."""
import ctypes as C
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from oracle import align_oracle as ao

G = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'align.npz'))
ROOT_TAGS = ('r23', 'r0', 'rm1', 'rempty')


def rel(x, ref):
    """max |x - ref| over the largest |ref|, NaN in exactly the same places"""
    assert x.shape == ref.shape
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(x), nan)
    if nan.all():
        return 0.0
    return np.abs(x[~nan] - ref[~nan]).max() / np.abs(ref[~nan]).max()


def cases():
    """(name, est, gt, fn) for every case of the fixture; fn(est, gt) is the oracle"""
    out = [('scale', G['est'], G['gt'], ao.scale_error, G['error_scale'])]
    for tag in ROOT_TAGS:
        out.append((f'root_{tag}', G['j_est'], G['j_gt'], lambda a, c, r=G[f'root_{tag}']: ao.root_error(a, c, r),
                    G[f'error_root_{tag}']))
    return out


@pytest.mark.parametrize('case', cases(), ids=lambda c: c[0])
def test_oracle_matches_reference(case):
    name, est, gt, fn, ref = case
    # the reference works in float32 here: eps * |coordinate| / error.  For scale its means are float32 sums along a
    # strided axis (the transposed view, metrics.py:197-205), which at 2.5 m from the origin are off by ~1e-6 m: that is
    # 1.2e-5 of the largest error of this fixture, whatever its noise level, so that case has the fp32-vs-fp32 bar.
    assert rel(fn(est, gt), ref) < (2e-5 if name == 'scale' else 5e-6)


def test_oracle_mpjpe14_matches_reference():
    joints = ao.regress_joints(G['j14'], G['j14_verts'])
    assert np.abs(joints - G['j14_joints']).max() < 1e-12
    assert rel(ao.root_error(joints, G['j14_gt'], [2, 3]), G['error_mpjpe14_root']) < 5e-6
    assert rel(ao.scale_error(joints, G['j14_gt']), G['error_mpjpe14_scale']) < 5e-6


@pytest.fixture(scope='module')
def host_lib(tmp_path_factory):
    lib = C.CDLL(ao.build_align_host(str(tmp_path_factory.mktemp('align_host'))))
    lib.align_host.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    lib.regress_host.argtypes = [C.c_void_p] * 4 + [C.c_int] * 3 + [C.c_void_p]
    return lib


def run_host(lib, est, gt, mode, roots=()):
    est, gt = np.ascontiguousarray(est, np.float32), np.ascontiguousarray(gt, np.float32)
    B, P = est.shape[:2]
    r = np.ascontiguousarray(roots, np.int32).reshape(-1)
    err, mean = np.empty((B, P), np.float32), np.empty(B, np.float32)
    lib.align_host(est.ctypes.data, gt.ctypes.data, B, P, mode, r.ctypes.data, len(r), err.ctypes.data, mean.ctypes.data)
    return err.astype(np.float64), mean.astype(np.float64)


@pytest.mark.parametrize('case', cases(), ids=lambda c: c[0])
def test_kernel_point_functions_compiled_for_host(host_lib, case):
    name, est, gt, _, ref = case
    roots = G[f'root_{name[5:]}'] if name.startswith('root') else ()
    err, mean = run_host(host_lib, est, gt, 1 if name == 'scale' else 2, roots)
    assert rel(err, ref) < 2e-5
    assert rel(mean, ref.mean(1)) < 2e-5


def test_kernel_regression_compiled_for_host(host_lib):
    from shapy_b200 import metrics
    reg = metrics.JointRegressor(G['j14'])
    rp, col, val = (t.numpy() for t in reg.csr)
    verts = np.ascontiguousarray(G['j14_verts'])
    B, V = verts.shape[:2]
    J = len(rp) - 1
    out = np.empty((B, J, 3), np.float32)
    host_lib.regress_host(rp.ctypes.data, col.ctypes.data, val.ctypes.data, verts.ctypes.data, B, J, V, out.ctypes.data)
    assert rel(out.astype(np.float64), G['j14_joints']) < 1e-6
    err, _ = run_host(host_lib, out, G['j14_gt'], 2, [2, 3])
    assert rel(err, G['error_mpjpe14_root']) < 2e-5
    err, _ = run_host(host_lib, out, G['j14_gt'], 1)
    assert rel(err, G['error_mpjpe14_scale']) < 2e-5


def test_alignment_names_and_reprs():
    from shapy_b200 import metrics
    s, r = metrics.build_alignment('scale'), metrics.build_alignment('root')
    assert isinstance(s, metrics.ScaleAlignment) and s.name == 'scale' and repr(s) == 'ScaleAlignment'
    assert isinstance(r, metrics.RootAlignment) and r.name == 'root' and r.root == [0]
    assert repr(r) == 'RootAlignment: root = [0]'
    r = metrics.build_alignment('root', root=[2, 3])                       # evaluation.py:616-619
    assert r.root == [2, 3] and repr(r) == 'RootAlignment: root = [2, 3]'
    assert metrics.build_alignment('scale', root=[2, 3]).name == 'scale'   # the evaluator passes root= to every alignment
    for name in ('procrustes', 'similarity'):
        with pytest.raises(NotImplementedError):
            metrics.build_alignment(name)


def test_set_root_forwards_through_point_error():
    from shapy_b200 import metrics
    pe = metrics.PointError(metrics.build_alignment('root', root=[0]))
    pe.set_root([2, 3])
    assert pe._alignment.root == [2, 3]
    assert repr(pe) == 'PointError: Alignment = RootAlignment: root = [2, 3]'
    metrics.PointError(metrics.build_alignment('scale')).set_root([1])    # no root: ignored, as in the reference
    metrics.PointError(metrics.build_alignment('translation')).set_root([1])


class FakeCuda(torch.Tensor):
    """A CPU tensor that claims to live on the GPU, so the host checks in front of the launch can be reached without one"""
    @property
    def is_cuda(self):
        return True


def fake(shape):
    return torch.zeros(shape).as_subclass(FakeCuda)


def test_host_checks_before_any_launch():
    from shapy_b200 import metrics
    pe = metrics.PointError(metrics.build_alignment('root', root=[14]))
    with pytest.raises(IndexError):
        pe(fake((2, 14, 3)), fake((2, 14, 3)))
    pe.set_root([-15])
    with pytest.raises(IndexError):
        pe(fake((2, 14, 3)), fake((2, 14, 3)))
    pe.set_root(list(range(17)))
    with pytest.raises(ValueError):
        pe(fake((2, 20, 3)), fake((2, 20, 3)))
    with pytest.raises(ValueError):                   # the reference would read (B, 3, 3) coordinates first
        metrics.PointError(metrics.build_alignment('scale'))(fake((2, 3, 3)), fake((2, 3, 3)))


def test_cpu_tensors_are_refused():
    from shapy_b200 import metrics
    for name in ('scale', 'root'):
        with pytest.raises(RuntimeError):
            metrics.PointError(metrics.build_alignment(name))(torch.from_numpy(G['j_est']), torch.from_numpy(G['j_gt']))
    with pytest.raises(RuntimeError):
        metrics.JointRegressor(G['j14'])(torch.from_numpy(G['j14_verts']))


@pytest.mark.parametrize('kind', ['dense', 'csr', 'coo'])
def test_joint_regressor_csr_equals_its_input(kind):
    from shapy_b200 import metrics
    dense = G['j14']
    m = {'dense': dense, 'csr': sp.csr_matrix(dense), 'coo': sp.coo_matrix(dense)}[kind]
    reg = metrics.JointRegressor(m)
    rp, col, val = (t.numpy() for t in reg.csr)
    assert rp.dtype == np.int32 and col.dtype == np.int32 and val.dtype == np.float32
    assert reg.shape == dense.shape and len(val) == np.count_nonzero(dense)       # exact zeros dropped
    back = sp.csr_matrix((val, col, rp), shape=dense.shape).toarray()
    assert np.array_equal(back.astype(np.float64), dense)                           # the fixture's weights are fp32 values
    with pytest.raises(ValueError):
        metrics.JointRegressor(dense[0])
