"""Point-to-point evaluation metric on the GPU (SURVEY.md 8f rank 3).

Host mirror of regressor/human_shape/utils/metrics.py:368-456 (`v2vhdError`): same constructor (two pickled scipy sparse
point regressors), same registered buffers (`input_point_regressor`, `target_point_regressor`, sparse COO) and the same
call `(input_points, target_points) -> (error.mean(1), error)`.  The reference evaluates it in float64 on the CPU after
copying every predicted mesh to the host (evaluation.py:227-265); here the meshes stay on the device and the result is
fp32 (`shapy_p2p_error`, csrc/metrics.cu).  There is no CPU fallback.

`PointError` with root / scale / translation / no alignment (metrics.py:85-98, 173-303, 335-366) and the J14 regression of
`mpjpe14` (`JointRegressor`) run on the device too; Procrustes is not built.
"""
import ctypes as C
import pickle

import numpy as np
import torch
import torch.nn as nn

from . import _lib


class v2vhdError(nn.Module):
    def __init__(self, input_point_regressor_path: str = '', target_point_regressor_path: str = '', align: bool = True) -> None:
        super().__init__()
        self.align = align
        self._csr = {}
        for name, path in (('input', input_point_regressor_path), ('target', target_point_regressor_path)):
            with open(path, 'rb') as f:
                m = pickle.load(f)
            self.register_buffer(f'{name}_point_regressor', self.to_pytorch(m))
            c = m.tocsr()
            c.sum_duplicates()
            self._csr[name] = (torch.from_numpy(c.indptr.astype(np.int32)), torch.from_numpy(c.indices.astype(np.int32)),
                               torch.from_numpy(c.data.astype(np.float32)), c.shape)
        if self._csr['input'][3][0] != self._csr['target'][3][0]:
            raise ValueError('v2vhdError: the two point regressors must produce the same number of points')
        self._dev = {}

    def to_pytorch(self, point_regressor):
        """metrics.py:398-414: scipy sparse -> torch sparse COO."""
        point_regressor = point_regressor.tocoo()
        indices = np.vstack((point_regressor.row, point_regressor.col))
        return torch.sparse_coo_tensor(indices, point_regressor.data, point_regressor.shape)

    def _arrays(self, device):
        key = str(device)
        if key not in self._dev:
            self._dev[key] = {n: tuple(t.to(device) for t in self._csr[n][:3]) for n in ('input', 'target')}
        return self._dev[key]

    def __call__(self, input_points, target_points):
        for name, t in (('input_points', input_points), ('target_points', target_points)):
            if not (torch.is_tensor(t) and t.is_cuda):
                raise RuntimeError(f'shapy_b200 v2vhdError: {name} must be a CUDA tensor (there is no CPU fallback)')
        P, V1 = self._csr['input'][3]
        _, V2 = self._csr['target'][3]
        if input_points.shape[1:] != (V1, 3) or target_points.shape[1:] != (V2, 3) or input_points.shape[0] != target_points.shape[0]:
            raise ValueError(f'v2vhdError: expected (B, {V1}, 3) and (B, {V2}, 3) vertices')
        dev = input_points.device
        a = self._arrays(dev)
        vi = input_points.contiguous().float()
        vt = target_points.to(dev).contiguous().float()
        B = vi.shape[0]
        error = torch.empty(B, P, dtype=torch.float32, device=dev)
        mean = torch.empty(B, dtype=torch.float32, device=dev)
        if B == 0:
            return mean, error
        with torch.cuda.device(dev):
            L = _lib.lib()
            nbytes = L.shapy_p2p_workspace_bytes(B, P)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            _lib.check(L.shapy_p2p_error(*[_lib.ptr(t) for t in a['input']], *[_lib.ptr(t) for t in a['target']], _lib.ptr(vi),
                                         _lib.ptr(vt), B, P, V1, V2, int(bool(self.align)), _lib.ptr(error), _lib.ptr(mean), _lib.ptr(ws),
                                         nbytes, _lib.stream_ptr()), 'p2p_error')
        return mean, error


class NoAlignment:
    """metrics.py:85-98."""
    name = 'none'

    def __repr__(self):
        return 'NoAlignment'


class TranslationAlignment:
    """metrics.py:232-277: est + (mean(gt) - mean(est))."""
    name = 'translation'

    def __repr__(self):
        return 'ScaleAlignment'       # sic: the reference's __repr__ (metrics.py:236-237)


class ScaleAlignment:
    """metrics.py:173-229: s est + (mu2 - s mu1) with s = sqrt(var2 / var1), per body (`shapy_point_error_aligned`).
    The reference reads a (B, 3, 3) input coordinates first (it transposes only when S1.shape[1] != 3); PointError refuses
    three points per body instead of reproducing that."""
    name = 'scale'

    def __repr__(self):
        return 'ScaleAlignment'


class RootAlignment:
    """metrics.py:279-303: both sides minus the mean of their points listed in `root` (default [0]; numpy indexing,
    negative indices count from the end, an empty list gives NaN)."""
    name = 'root'

    def __init__(self, root=None, **kwargs):
        self.root = [0] if root is None else root

    def set_root(self, new_root):
        self.root = new_root

    def __repr__(self):
        return f'RootAlignment: root = {self.root}'


def build_alignment(name: str, **kwargs):
    """metrics.py:14-29 for the alignments evaluated on the device; Procrustes is not built."""
    if name == 'root':
        return RootAlignment(**kwargs)
    if name == 'scale':
        return ScaleAlignment()
    if name == 'translation':
        return TranslationAlignment()
    if name in ('no', 'none'):
        return NoAlignment()
    raise NotImplementedError(f'shapy_b200.metrics: alignment `{name}` is not built (root / scale / translation / none are)')


def _root_indices(root, P):
    """The root list as numpy would index axis 1 of a (B, P, 3) array with it: IndexError out of range."""
    idx = [int(r) for r in np.asarray(root, dtype=np.int64).reshape(-1)]
    for r in idx:
        if not -P <= r < P:
            raise IndexError(f'index {r} is out of bounds for axis 1 with size {P}')
    if len(idx) > _lib.MAX_ROOTS:
        raise ValueError(f'shapy_b200 RootAlignment: at most {_lib.MAX_ROOTS} root indices, got {len(idx)}')
    return idx


class PointError:
    """metrics.py:335-366 for same-topology point sets on the device: `PointError(build_alignment(name))(est, gt)`
    returns the (B, P) per-point error as a CUDA fp32 tensor; `.last_mean` keeps the per-body mean of the same launch.
    translation / none: the `v2v_t` / `v2v` errors of `_compute_v2v` (evaluation.py:192-224, `shapy_v2v_error`).
    scale / root: the scale-corrected `v2v_t` and the root-aligned `mpjpe` / `mpjpe14` (evaluation.py:595-620,
    `shapy_point_error_aligned`).  The reference copies both sides to the host."""

    def __init__(self, alignment_object, name: str = ''):
        if not isinstance(alignment_object, (TranslationAlignment, NoAlignment, ScaleAlignment, RootAlignment)):
            raise NotImplementedError('shapy_b200 PointError: only root / scale / translation / no alignment run on the device')
        self._alignment, self._name, self.last_mean = alignment_object, name, None

    name = property(lambda self: self._name)

    def __repr__(self):
        return f'PointError: Alignment = {self._alignment}'

    def set_alignment(self, alignment_object):
        self.__init__(alignment_object, self._name)

    def set_root(self, new_root):
        """metrics.py:353-355: forwarded to alignments that have a root (RootAlignment), ignored by the others."""
        if hasattr(self._alignment, 'set_root'):
            self._alignment.set_root(new_root)

    def __call__(self, est_points, gt_points):
        for nm, t in (('est_points', est_points), ('gt_points', gt_points)):
            if not (torch.is_tensor(t) and t.is_cuda):
                raise RuntimeError(f'shapy_b200 PointError: {nm} must be a CUDA tensor (there is no CPU fallback)')
        if est_points.shape != gt_points.shape or est_points.dim() != 3 or est_points.shape[2] != 3:
            raise ValueError('PointError: expected two (B, P, 3) tensors of the same shape')
        B, V = est_points.shape[:2]
        scale, root = isinstance(self._alignment, ScaleAlignment), isinstance(self._alignment, RootAlignment)
        if scale and V == 3:
            raise ValueError('shapy_b200 PointError: ScaleAlignment of (B, 3, 3) points is refused (the reference would read '
                             'them coordinates first)')
        roots = _root_indices(self._alignment.root, V) if root else []
        dev = est_points.device
        a, b = est_points.contiguous().float(), gt_points.to(dev).contiguous().float()
        error = torch.empty(B, V, dtype=torch.float32, device=dev)
        mean = torch.empty(B, dtype=torch.float32, device=dev)
        if B == 0 or V == 0:
            self.last_mean = mean.fill_(float('nan')) if B else mean
            return error
        with torch.cuda.device(dev):
            L = _lib.lib()
            if scale or root:
                nbytes = L.shapy_point_error_workspace_bytes(B)
                ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
                _lib.check(L.shapy_point_error_aligned(_lib.ptr(a), _lib.ptr(b), B, V, _lib.ALIGN_SCALE if scale else _lib.ALIGN_ROOT,
                                                       (C.c_int * max(len(roots), 1))(*roots), len(roots), _lib.ptr(error),
                                                       _lib.ptr(mean), _lib.ptr(ws), nbytes, _lib.stream_ptr()), 'point_error_aligned')
            else:
                nbytes = L.shapy_p2p_workspace_bytes(B, V)
                ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
                _lib.check(L.shapy_v2v_error(_lib.ptr(a), _lib.ptr(b), B, V, int(isinstance(self._alignment, TranslationAlignment)),
                                             _lib.ptr(error), _lib.ptr(mean), _lib.ptr(ws), nbytes, _lib.stream_ptr()), 'v2v_error')
        self.last_mean = mean
        return error


class JointRegressor:
    """The J14 joint regression of `_compute_mpjpe14` (evaluation.py:161-190, `np.einsum('jv,bvn->bjn', J14_regressor,
    vertices)`) on the device.  `regressor` is the (J, V) matrix as the evaluator loads it (evaluation.py:620-635): a dense
    array or a scipy sparse matrix.  It is stored once as a CSR with exact zeros dropped and fp32 values;
    `__call__(vertices (B, V, 3) CUDA)` returns the (B, J, 3) CUDA fp32 joints (`shapy_regress_points`), which
    `PointError(build_alignment('root', root=[2, 3]))` and the others then compare with the ground-truth joints.  Only the
    summation order (and fp32 instead of the reference's float64) differs from the einsum."""

    def __init__(self, regressor):
        import scipy.sparse as sp
        if not sp.issparse(regressor) and np.ndim(regressor) != 2:
            raise ValueError('shapy_b200 JointRegressor: expected a 2-D (J, V) regressor')
        m = sp.csr_matrix(regressor, dtype=np.float64)
        m.sum_duplicates()
        m.eliminate_zeros()
        self.shape = m.shape
        self.csr = (torch.from_numpy(m.indptr.astype(np.int32)), torch.from_numpy(m.indices.astype(np.int32)),
                    torch.from_numpy(m.data.astype(np.float32)))
        self._dev = {}

    def __call__(self, vertices):
        if not (torch.is_tensor(vertices) and vertices.is_cuda):
            raise RuntimeError('shapy_b200 JointRegressor: vertices must be a CUDA tensor (there is no CPU fallback)')
        J, V = self.shape
        if vertices.dim() != 3 or vertices.shape[1:] != (V, 3):
            raise ValueError(f'shapy_b200 JointRegressor: expected (B, {V}, 3) vertices')
        dev = vertices.device
        B = vertices.shape[0]
        joints = torch.empty(B, J, 3, dtype=torch.float32, device=dev)
        if B == 0 or J == 0:
            return joints
        key = str(dev)
        if key not in self._dev:
            self._dev[key] = tuple(t.to(dev) for t in self.csr)
        v = vertices.contiguous().float()
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().shapy_regress_points(*[_lib.ptr(t) for t in self._dev[key]], _lib.ptr(v), B, J, V,
                                                       _lib.ptr(joints), _lib.stream_ptr()), 'regress_points')
        return joints
