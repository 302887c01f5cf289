"""Tensor-level wrappers over the C ABI (include/shapy_b200.h).

PyTorch is used for device memory and streams only: every function takes CUDA fp32 tensors, allocates
the outputs with torch, and launches the hand-written sm_90a kernels on the current stream.  Nothing
here computes with torch ops, and nothing falls back to the CPU: non-CUDA inputs raise.
"""
import collections
import ctypes as C
import weakref

import numpy as np
import torch

from . import _lib
from ._lib import check, lib, ptr, stream_ptr


def _cuda_f32(t, name):
    if not (torch.is_tensor(t) and t.is_cuda):
        raise RuntimeError(f'shapy_b200: `{name}` must be a CUDA tensor (there is no CPU path)')
    if t.dtype != torch.float32:
        raise RuntimeError(f'shapy_b200: `{name}` must be float32, got {t.dtype}')
    return t.contiguous()


class _Workspace:
    """Grow-only per-device scratch buffer (plumbing, not math)."""

    def __init__(self):
        self.bufs = {}

    def get(self, key, nbytes, device):
        k = (key, device.index)
        b = self.bufs.get(k)
        if b is None or b.numel() < nbytes:
            b = torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=device)
            self.bufs[k] = b
        return b


_WS = _Workspace()


# ------------------------------------------------------------------------------------------ SMPL-X
class SmplxModel:
    """Device-side packed SMPL-X constants (shapy_smplx_create).  `tensors` uses the reference's
    buffer names (body_models.py:112-166, 563-597)."""

    def __init__(self, tensors: dict, device):
        self.device = torch.device(device)
        h = {}

        def host(name, dtype, required=True):
            t = tensors.get(name)
            if t is None or (torch.is_tensor(t) and t.numel() == 0):
                if required:
                    raise RuntimeError(f'SMPL-X tensor `{name}` missing')
                return None
            a = np.ascontiguousarray(t.detach().cpu().numpy().astype(dtype))
            h[name] = a
            return a

        vt = host('v_template', np.float32)
        sd = host('shapedirs', np.float32)
        ed = host('expr_dirs', np.float32, False)
        pd = host('posedirs', np.float32)
        jr = host('J_regressor', np.float32)
        lw = host('lbs_weights', np.float32)
        par = host('parents', np.int64)
        fc = host('faces_tensor', np.int64)
        lf = host('lmk_faces_idx', np.int64, False)
        lb = host('lmk_bary_coords', np.float32, False)
        df = host('dynamic_lmk_faces_idx', np.int64, False)
        db = host('dynamic_lmk_bary_coords', np.float32, False)
        nk = host('neck_kin_chain', np.int64, False)
        ex = host('extra_joint_regressor', np.float32, False)
        si = host('source_idxs', np.int64, False)
        ti = host('target_idxs', np.int64, False)
        d = _lib.SmplxDesc()
        d.num_verts, d.num_joints = vt.shape[0], jr.shape[0]
        d.num_betas = sd.shape[-1]
        d.num_expr = 0 if ed is None else ed.shape[-1]
        d.num_faces = fc.shape[0]
        ap = lambda a: None if a is None else a.ctypes.data  # noqa: E731
        d.v_template, d.shapedirs, d.expr_dirs, d.posedirs = ap(vt), ap(sd), ap(ed), ap(pd)
        d.J_regressor, d.lbs_weights, d.parents, d.faces = ap(jr), ap(lw), ap(par), ap(fc)
        d.num_static_lmk = 0 if lf is None else lf.shape[0]
        d.lmk_faces_idx, d.lmk_bary_coords = ap(lf), ap(lb)
        use_dyn = df is not None and tensors.get('use_face_contour', True)
        d.num_dyn_lmk = df.shape[1] if use_dyn else 0
        d.num_dyn_rows = df.shape[0] if use_dyn else 0
        d.dynamic_lmk_faces_idx, d.dynamic_lmk_bary_coords = (ap(df), ap(db)) if use_dyn else (None, None)
        d.neck_chain_len = 0 if nk is None else nk.shape[0]
        d.neck_kin_chain = ap(nk)
        d.num_extra = 0 if ex is None else ex.shape[0]
        d.extra_joint_regressor = ap(ex)
        d.num_overwrite = 0 if si is None else si.shape[0]
        d.source_idxs, d.target_idxs = ap(si), ap(ti)
        self.V, self.J, self.NB, self.NE, self.F = d.num_verts, d.num_joints, d.num_betas, d.num_expr, d.num_faces
        handle = C.c_void_p()
        with torch.cuda.device(self.device):
            check(lib().shapy_smplx_create(C.byref(handle), C.byref(d)), 'smplx_create')
        self.handle = handle
        self.K = lib().shapy_smplx_num_keypoints(handle)
        self._fin = weakref.finalize(self, lib().shapy_smplx_destroy, handle)
        self._faces_ptr = lib().shapy_smplx_faces_i32(handle)

    @property
    def faces_ptr(self):
        return C.c_void_p(self._faces_ptr)


def decode_rot6d(raw: torch.Tensor) -> torch.Tensor:
    """(B, 6n) -> (B, n, 3, 3)  (ContinuousRotReprDecoder.forward, pose_utils.py:138-153)."""
    raw = _cuda_f32(raw, 'raw')
    B = raw.shape[0]
    n = raw.numel() // 6
    out = torch.empty(n, 3, 3, dtype=torch.float32, device=raw.device)
    if n == 0:            # empty batch: nothing to launch (torch semantics: empty in, empty out)
        return out.view(B, raw.shape[1] // 6 if raw.dim() > 1 else 0, 3, 3)
    with torch.cuda.device(raw.device):
        check(lib().shapy_decode_rot6d(ptr(raw), n, ptr(out), stream_ptr()), 'decode_rot6d')
    return out.view(B, -1, 3, 3)


def smplx_forward(model: SmplxModel, betas, rot, expr=None, camera=None, want_vertices=True, want_v_shaped=True,
                  want_joints=True):
    """rot (B, n_rot, 3, 3): rotations of the first n_rot joints of the full pose; the rest is identity."""
    betas = _cuda_f32(betas, 'betas')
    rot = _cuda_f32(rot, 'rot')
    B, n_rot = rot.shape[0], rot.shape[1]
    if betas.shape != (B, model.NB):
        raise RuntimeError(f'betas must be ({B}, {model.NB}), got {tuple(betas.shape)}')
    dev = betas.device
    expr = None if expr is None else _cuda_f32(expr, 'expression')
    camera = None if camera is None else _cuda_f32(camera, 'camera')
    mk = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)  # noqa: E731
    vertices = mk(B, model.V, 3) if want_vertices else None
    v_shaped = mk(B, model.V, 3) if want_v_shaped else None
    joints = mk(B, model.K, 3) if want_joints else None
    proj = mk(B, model.K, 2) if (want_joints and camera is not None) else None
    if B == 0:
        return dict(vertices=vertices, v_shaped=v_shaped, joints=joints, proj_joints=proj)
    with torch.cuda.device(dev):
        nbytes = lib().shapy_smplx_workspace_bytes(model.handle, B)
        ws = _WS.get('smplx', nbytes, dev)
        check(lib().shapy_smplx_forward(model.handle, ptr(betas), ptr(rot), n_rot, ptr(expr), ptr(camera), B,
                                        ptr(vertices), ptr(v_shaped), ptr(joints), ptr(proj), ptr(ws), ws.numel(),
                                        stream_ptr()), 'smplx_forward')
    return dict(vertices=vertices, v_shaped=v_shaped, joints=joints, proj_joints=proj)


def smplx_forward_shape(model: SmplxModel, betas) -> torch.Tensor:
    betas = _cuda_f32(betas, 'betas')
    B = betas.shape[0]
    out = torch.empty(B, model.V, 3, dtype=torch.float32, device=betas.device)
    if B == 0:
        return out
    with torch.cuda.device(betas.device):
        check(lib().shapy_smplx_forward_shape(model.handle, ptr(betas), B, ptr(out), stream_ptr()), 'forward_shape')
    return out


def decode_rot6d_backward(raw: torch.Tensor, grad_rot: torch.Tensor) -> torch.Tensor:
    """Gradient of decode_rot6d with respect to raw (B, 6n), from grad_rot (B, n, 3, 3)."""
    raw = _cuda_f32(raw, 'raw')
    g = _cuda_f32(grad_rot, 'grad_rot')
    n = raw.numel() // 6
    if g.numel() != 9 * n:
        raise RuntimeError(f'grad_rot has {g.numel()} values for {n} rotations')
    out = torch.empty_like(raw)
    if n == 0:
        return out
    with torch.cuda.device(raw.device):
        check(lib().shapy_decode_rot6d_backward(ptr(raw), n, ptr(g), ptr(out), stream_ptr()), 'decode_rot6d_backward')
    return out


def smplx_backward(model: SmplxModel, betas, rot, expr=None, camera=None, grad_vertices=None, grad_v_shaped=None,
                   grad_joints=None, grad_proj_joints=None, want=('betas', 'rot', 'expr', 'camera')):
    """Adjoint of smplx_forward (include/shapy_b200.h, shapy_smplx_backward).  A cotangent left None is zero; `want`
    names the gradients to compute.  Returns {'betas', 'rot', 'expr', 'camera'}, None where not wanted (and for expr /
    camera when the model has no expression basis / no camera was given)."""
    betas = _cuda_f32(betas, 'betas')
    rot = _cuda_f32(rot, 'rot')
    B, n_rot = rot.shape[0], rot.shape[1]
    if betas.shape != (B, model.NB):
        raise RuntimeError(f'betas must be ({B}, {model.NB}), got {tuple(betas.shape)}')
    dev = betas.device
    expr = None if expr is None else _cuda_f32(expr, 'expression')
    camera = None if camera is None else _cuda_f32(camera, 'camera')
    shapes = dict(grad_vertices=(B, model.V, 3), grad_v_shaped=(B, model.V, 3), grad_joints=(B, model.K, 3),
                  grad_proj_joints=(B, model.K, 2))
    gs = {}
    for name, g in (('grad_vertices', grad_vertices), ('grad_v_shaped', grad_v_shaped), ('grad_joints', grad_joints),
                    ('grad_proj_joints', grad_proj_joints)):
        if g is not None:
            g = _cuda_f32(g, name)
            if tuple(g.shape) != shapes[name]:
                raise RuntimeError(f'{name} must be {shapes[name]}, got {tuple(g.shape)}')
        gs[name] = g
    if camera is None:
        gs['grad_proj_joints'] = None
    mk = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)  # noqa: E731
    out = dict(betas=mk(B, model.NB) if 'betas' in want else None,
               rot=mk(B, n_rot, 3, 3) if 'rot' in want else None,
               expr=mk(B, model.NE) if ('expr' in want and model.NE) else None,
               camera=mk(B, 3) if ('camera' in want and camera is not None) else None)
    if B == 0:
        return out
    with torch.cuda.device(dev):
        nbytes = lib().shapy_smplx_backward_workspace_bytes(model.handle, B, n_rot)
        ws = _WS.get('smplx_bwd', nbytes, dev)
        check(lib().shapy_smplx_backward(model.handle, ptr(betas), ptr(rot), n_rot, ptr(expr), ptr(camera), B,
                                         ptr(gs['grad_vertices']), ptr(gs['grad_v_shaped']), ptr(gs['grad_joints']),
                                         ptr(gs['grad_proj_joints']), ptr(out['betas']), ptr(out['rot']),
                                         ptr(out['expr']), ptr(out['camera']), ptr(ws), ws.numel(), stream_ptr()),
              'smplx_backward')
    return out


# ------------------------------------------------------------------------------------ measurements
def make_landmarks(lm: dict) -> _lib.MeasureLandmarks:
    """lm: {'head_top','left_heel','chest','waist','hips'} -> {'face_idx', 'bc'}."""
    s = _lib.MeasureLandmarks()
    for i, k in enumerate(('head_top', 'left_heel', 'chest', 'waist', 'hips')):
        s.face_idx[i] = int(lm[k]['face_idx'])
        for c in range(3):
            s.bc[i][c] = float(lm[k]['bc'][c])
    return s


def _faces_i32(faces_i32):
    if not (torch.is_tensor(faces_i32) and faces_i32.is_cuda and faces_i32.dtype == torch.int32):
        raise RuntimeError('faces_i32 must be a CUDA int32 tensor')
    return faces_i32.contiguous()


def _measure_input(v_shaped, faces_i32, triangles):
    """(x, faces_i32, B, V, F) of a measurement call on either (v_shaped (B,V,3), faces_i32) or triangles (B,F,3,3)."""
    if triangles is not None:
        x = _cuda_f32(triangles, 'triangles')
        return x, None, x.shape[0], 0, x.shape[1]
    x = _cuda_f32(v_shaped, 'v_shaped')
    faces_i32 = _faces_i32(faces_i32)
    return x, faces_i32, x.shape[0], x.shape[1], faces_i32.shape[0]


def measure(landmarks: _lib.MeasureLandmarks, v_shaped=None, faces_i32=None, triangles=None, return_points=False,
            max_points=1024, strict=False):
    """Returns (B, 5) = mass, height, chest, waist, hips.  Either (v_shaped, faces_i32) or triangles (B,F,3,3).

    The kernel's point / candidate buffers have a fixed capacity, the same for every entry: 1024 points per plane and
    8192 AABB candidates per body (the reference's `max_collisions` has no equivalent).  A plane past 1024 points gets
    a NaN circumference, a body past 8192 candidates NaN on all three, never a truncated value, and the device status
    word is set; `max_points` below a plane's count truncates the returned points only, and also sets it.  A slice
    whose xz hull has zero area (fewer than 3 points, all collinear or all coincident) is NaN too, where the
    reference's qhull raises, but does not set the status.  The status word is returned as `out.status` (a 1-element
    int32 CUDA tensor, readable at the caller's next synchronisation point) and `strict=True` checks it here (one host
    synchronisation) and raises."""
    x, faces_i32, B, V, F = _measure_input(v_shaped, faces_i32, triangles)
    dev = x.device
    out = torch.empty(B, 5, dtype=torch.float32, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    pts = cnt = None
    if return_points:
        pts = torch.zeros(B, 3, max_points, 3, dtype=torch.float32, device=dev)
        cnt = torch.zeros(B, 3, dtype=torch.int32, device=dev)
    if B == 0:
        out.status = status
        return (out, pts, cnt, status) if return_points else out
    with torch.cuda.device(dev):
        if triangles is not None:
            check(lib().shapy_measure_forward_tris(ptr(x), B, F, C.byref(landmarks), ptr(out), ptr(pts), ptr(cnt),
                                                   max_points, ptr(status), stream_ptr()), 'measure')
        else:
            check(lib().shapy_measure_forward(ptr(x), ptr(faces_i32), B, V, F, C.byref(landmarks), ptr(out), ptr(pts),
                                              ptr(cnt), max_points, ptr(status), stream_ptr()), 'measure')
    out.status = status
    if strict and int(status.item()) != 0:
        raise RuntimeError('shapy_b200 measure: a slicing plane produced more intersection points than the kernel can '
                           'hold (the affected circumferences are NaN)')
    if return_points:
        return out, pts, cnt, status
    return out


_INCIDENCE = {}      # id(faces tensor) -> (weak reference, version, incidence); entries leave with their tensor


def face_incidence(faces_i32):
    """Vertex -> (face, corner) incidence of a CUDA int32 (F, 3) faces tensor in CSR form: (inc_ptr (V+1), inc (3F)),
    int32 on the same device, entries 3 f + k in ascending order per vertex (stable sort).  Built on the host once per
    faces tensor (one copy to the host) and cached for as long as that tensor lives."""
    key = id(faces_i32)
    hit = _INCIDENCE.get(key)
    if hit is not None and hit[0]() is faces_i32 and hit[1] == faces_i32._version:
        return hit[2]
    flat = faces_i32.detach().reshape(-1).cpu().numpy().astype(np.int64)
    V = int(flat.max()) + 1 if flat.size else 0
    order = np.argsort(flat, kind='stable').astype(np.int32)
    ptr_ = np.zeros(V + 1, np.int32)
    np.cumsum(np.bincount(flat, minlength=V), out=ptr_[1:])
    inc = (torch.from_numpy(ptr_).to(faces_i32.device), torch.from_numpy(order).to(faces_i32.device))
    if hit is None or hit[0]() is not faces_i32:
        weakref.finalize(faces_i32, _INCIDENCE.pop, key, None)
    _INCIDENCE[key] = (weakref.ref(faces_i32), faces_i32._version, inc)
    return inc


def measure_backward(landmarks: _lib.MeasureLandmarks, grad_out, v_shaped=None, faces_i32=None, triangles=None,
                     exact=False):
    """Gradient of `measure` (B, 5) with respect to v_shaped (B, V, 3) or triangles (B, F, 3, 3), with the reference's
    autograd semantics (include/shapy_b200.h, shapy_measure_backward): the intersection barycentrics are constants and
    the plane heights get no gradient.  exact=True gives the exact derivative of the circumferences instead
    (shapy_measure_backward_exact: the hull points move with their faces and with the plane heights); the mass and
    height terms are the same bits.  Deterministic, one launch."""
    g = _cuda_f32(grad_out, 'grad_out')
    x, faces_i32, B, V, F = _measure_input(v_shaped, faces_i32, triangles)
    if g.shape != (B, 5):
        raise RuntimeError(f'grad_out must be ({B}, 5), got {tuple(g.shape)}')
    grad = torch.empty_like(x)
    if B == 0:
        return grad
    with torch.cuda.device(x.device):
        if triangles is not None:
            fn = lib().shapy_measure_backward_tris_exact if exact else lib().shapy_measure_backward_tris
            check(fn(ptr(x), B, F, C.byref(landmarks), ptr(g), ptr(grad), stream_ptr()), 'measure_backward')
        else:
            inc_ptr, inc = _incidence_rows(faces_i32, V)
            fn = lib().shapy_measure_backward_exact if exact else lib().shapy_measure_backward
            check(fn(ptr(x), ptr(faces_i32), ptr(inc_ptr), ptr(inc), B, V, F, C.byref(landmarks), ptr(g), ptr(grad),
                     stream_ptr()), 'measure_backward')
    return grad


def _incidence_rows(faces_i32, V):
    inc_ptr, inc = face_incidence(faces_i32)
    if inc_ptr.numel() - 1 > V:
        raise RuntimeError(f'faces index vertex {inc_ptr.numel() - 2} of a mesh with {V} vertices')
    if inc_ptr.numel() - 1 < V:     # trailing vertices no face uses: empty rows
        inc_ptr = torch.cat([inc_ptr, inc_ptr[-1:].expand(V + 1 - inc_ptr.numel())])
    return inc_ptr, inc


MAX_JACOBIAN_BETAS = 16


def measure_jacobian_betas(model: SmplxModel, landmarks: _lib.MeasureLandmarks, v_shaped, faces_i32, exact=False):
    """The measurements (B, 5) of `measure` and their Jacobian (B, 5, NB) with respect to the model's betas at the
    vertices v_shaped (B, V, 3), one launch (include/shapy_b200.h, shapy_measure_jacobian_betas).  faces_i32: the
    model's faces as a CUDA int32 (F, 3) tensor (its incidence table is cached).  exact=True gives the exact
    circumference rows (shapy_measure_jacobian_betas_exact, see measure_backward); the measurements and the mass and
    height rows are the same bits.  Returns (out, jac, status), status the device status word of `measure`."""
    x = _cuda_f32(v_shaped, 'v_shaped')
    faces_i32 = _faces_i32(faces_i32)
    if x.dim() != 3 or x.shape[1:] != (model.V, 3):
        raise RuntimeError(f'v_shaped must be (B, {model.V}, 3), got {tuple(x.shape)}')
    if tuple(faces_i32.shape) != (model.F, 3):
        raise RuntimeError(f'faces_i32 must be ({model.F}, 3), got {tuple(faces_i32.shape)}')
    if model.NB > MAX_JACOBIAN_BETAS:
        raise RuntimeError(f'measure_jacobian_betas supports at most {MAX_JACOBIAN_BETAS} betas, the model has '
                           f'{model.NB}')
    B, dev = x.shape[0], x.device
    if x.data_ptr() % 16:           # the kernel stages the vertices with 16-byte loads from a 16-byte aligned base
        x = x.clone()
    out = torch.empty(B, 5, dtype=torch.float32, device=dev)
    jac = torch.empty(B, 5, model.NB, dtype=torch.float32, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    if B == 0:
        return out, jac, status
    with torch.cuda.device(dev):
        inc_ptr, inc = _incidence_rows(faces_i32, model.V)
        fn = lib().shapy_measure_jacobian_betas_exact if exact else lib().shapy_measure_jacobian_betas
        check(fn(model.handle, ptr(x), ptr(inc_ptr), ptr(inc), B, C.byref(landmarks), ptr(out), ptr(jac), ptr(status),
                 stream_ptr()), 'measure_jacobian_betas')
    return out, jac, status


def _check_step_tensors(what, f32, f32_names, accepted):
    """What every LM step wrapper requires of its tensors: `f32` (named by f32_names in the message) and the counter
    `accepted` contiguous on the device, float32 and int32."""
    for t in f32 + [accepted]:
        if not (torch.is_tensor(t) and t.is_cuda and t.is_contiguous()):
            raise RuntimeError(f'{what}: every tensor must be a contiguous CUDA tensor')
    for t in f32:
        if t.dtype != torch.float32:
            raise RuntimeError(f'{what}: {f32_names} must be float32')
    if accepted.dtype != torch.int32:
        raise RuntimeError(f'{what}: accepted must be int32')


def _kp_step_shapes_ok(state, trial_jac, weights, B, K, P):
    """Whether both Jacobians and the weights of a keypoint step have the shapes its sizes give."""
    return trial_jac.shape == (B, 3 * K, P) and state['jac'].shape == (B, 3 * K, P) and weights.shape == (B, K)


def _meas_step_shapes_ok(state, trial_meas, trial_meas_jac, meas_targets, meas_weights, B, nb):
    """Whether the measurement block of a stacked keypoint + measurement step has the shapes its sizes give."""
    return (trial_meas_jac.shape == (B, 5, nb) and state['meas_jac'].shape == (B, 5, nb) and
            all(t.shape == (B, 5) for t in (meas_targets, meas_weights, trial_meas, state['meas'])))


def _check_kp2d_scalars(what, robust_sigma, pose_prior_weight, betas_weight, lambda_up, lambda_down, pose_anchor):
    """The scalar checks of every 2D keypoint step; returns robust_sigma as the step takes it (inf for None)."""
    sigma = float('inf') if robust_sigma is None else float(robust_sigma)
    if not (sigma > 0 and pose_prior_weight >= 0 and betas_weight >= 0 and lambda_up >= 1 and lambda_down >= 1):
        raise ValueError(f'{what}: robust_sigma must be > 0, the prior weights >= 0 and the lambda factors >= 1')
    if pose_prior_weight > 0 and pose_anchor is None:
        raise ValueError(f'{what}: pose_prior_weight > 0 needs pose_anchor')
    return sigma


def _check_offsets(what, name, off, B, G=None):
    """The offsets `name` of a grouped step: a contiguous int32 CPU tensor rising strictly from 0 to B (no empty group),
    with G + 1 entries when G is given.  Returns the number of groups."""
    if not (torch.is_tensor(off) and off.device.type == 'cpu' and off.dtype == torch.int32 and off.dim() == 1 and
            off.is_contiguous()):
        raise RuntimeError(f'{what}: {name} must be a contiguous (G + 1,) int32 CPU tensor')
    n = off.numel() - 1
    if n < 0 or G not in (None, n) or int(off[0]) != 0 or int(off[-1]) != B or not bool((off[1:] > off[:-1]).all()):
        entries = '' if G is None else f' in {G + 1} entries'
        raise ValueError(f'{what}: {name} must rise strictly from 0 to {B}{entries}')
    return n


def _workspace(n, device):
    """The scratch of a grouped step, n bytes from its *_workspace_bytes entry: a uint8 CUDA tensor, allocated once
    before an LM loop."""
    return torch.empty(max(int(n), 1), dtype=torch.uint8, device=device)


def _check_workspace(what, workspace, need):
    if not (workspace.is_cuda and workspace.is_contiguous() and workspace.numel() * workspace.element_size() >= need):
        raise RuntimeError(f'{what}: the workspace must be a contiguous CUDA tensor of at least {need} bytes')


def fit_lm_step(state, targets, weights, betas_weight, lambda_up, lambda_down, first, trial, trial_meas, trial_jac):
    """One Levenberg-Marquardt step per body (include/shapy_b200.h, shapy_fit_lm_step), in place.  state: {'betas'
    (B, NB), 'meas' (B, 5), 'jac' (B, 5, NB), 'loss' (B,), 'lambda' (B,), 'accepted' (B,) int32}, CUDA tensors;
    trial (B, NB) is the evaluated trial on entry and the next trial on return."""
    B, nb = trial.shape
    ts = [state[k] for k in ('betas', 'meas', 'jac', 'loss', 'lambda')] + [targets, weights, trial, trial_meas,
                                                                           trial_jac]
    _check_step_tensors('fit_lm_step', ts, 'the state, targets, weights and trial', state['accepted'])
    if B == 0:
        return
    with torch.cuda.device(trial.device):
        check(lib().shapy_fit_lm_step(B, nb, ptr(targets), ptr(weights), float(betas_weight), float(lambda_up),
                                      float(lambda_down), int(bool(first)), ptr(state['betas']), ptr(state['meas']),
                                      ptr(state['jac']), ptr(state['loss']), ptr(state['lambda']),
                                      ptr(state['accepted']), ptr(trial), ptr(trial_meas), ptr(trial_jac),
                                      stream_ptr()), 'fit_lm_step')


def smplx_keypoint_jacobian(model: SmplxModel, betas, rot, transl=None, expr=None):
    """The keypoints (B, K, 3) of smplx_forward (its joints, expression zero) plus transl, and their Jacobian
    (B, 3K, P), P = 3 n_rot + NB + 3, with respect to [delta_j (right-multiplied tangents R_j Exp(delta_j)) | betas |
    transl], in one launch (include/shapy_b200.h, shapy_smplx_keypoint_jacobian).  Returns (keypoints, jac).
    expr (B, NE): the keypoints at that expression and NE more columns after betas, P = 3 n_rot + NB + NE + 3
    (shapy_smplx_keypoint_jacobian_expr); None is the launch above."""
    if expr is not None:
        return _smplx_keypoint_jacobian_expr(model, betas, rot, transl, expr)
    betas = _cuda_f32(betas, 'betas')
    rot = _cuda_f32(rot, 'rot')
    B, n_rot = rot.shape[0], rot.shape[1]
    if rot.shape[2:] != (3, 3) or betas.shape != (B, model.NB):
        raise RuntimeError(f'rot must be (B, n_rot, 3, 3) and betas ({B}, {model.NB}), got {tuple(rot.shape)} and '
                           f'{tuple(betas.shape)}')
    transl = None if transl is None else _cuda_f32(transl, 'transl')
    if transl is not None and transl.shape != (B, 3):
        raise RuntimeError(f'transl must be ({B}, 3), got {tuple(transl.shape)}')
    dev = betas.device
    kp = torch.empty(B, model.K, 3, dtype=torch.float32, device=dev)
    jac = torch.empty(B, 3 * model.K, 3 * n_rot + model.NB + 3, dtype=torch.float32, device=dev)
    if B == 0:
        return kp, jac
    with torch.cuda.device(dev):
        check(lib().shapy_smplx_keypoint_jacobian(model.handle, ptr(betas), ptr(rot), n_rot, ptr(transl), B, ptr(kp),
                                                  ptr(jac), stream_ptr()), 'smplx_keypoint_jacobian')
    return kp, jac


def smplx_vertex_jacobian(model: SmplxModel, betas, rot, transl=None):
    """Every posed vertex (B, V, 3) (+ transl) and its Jacobian (B, V, 3, P), P = 3 n_rot + NB + 3, with the columns of
    smplx_keypoint_jacobian, in one launch (include/shapy_b200.h, shapy_smplx_vertex_jacobian).  The Jacobian takes
    4 V 3 P bytes per body: 9.9 MB at V = 10475 and P = 79, 635 MB at B = 64.  Returns (vertices, jac)."""
    betas = _cuda_f32(betas, 'betas')
    rot = _cuda_f32(rot, 'rot')
    B, n_rot = rot.shape[0], rot.shape[1]
    if rot.dim() != 4 or rot.shape[2:] != (3, 3) or betas.shape != (B, model.NB):
        raise RuntimeError(f'rot must be (B, n_rot, 3, 3) and betas ({B}, {model.NB}), got {tuple(rot.shape)} and '
                           f'{tuple(betas.shape)}')
    transl = None if transl is None else _cuda_f32(transl, 'transl')
    if transl is not None and transl.shape != (B, 3):
        raise RuntimeError(f'transl must be ({B}, 3), got {tuple(transl.shape)}')
    dev = betas.device
    verts = torch.empty(B, model.V, 3, dtype=torch.float32, device=dev)
    jac = torch.empty(B, model.V, 3, 3 * n_rot + model.NB + 3, dtype=torch.float32, device=dev)
    if B == 0:
        return verts, jac
    with torch.cuda.device(dev):
        check(lib().shapy_smplx_vertex_jacobian(model.handle, ptr(betas), ptr(rot), n_rot, ptr(transl), B, ptr(verts),
                                                ptr(jac), stream_ptr()), 'smplx_vertex_jacobian')
    return verts, jac


def _smplx_keypoint_jacobian_expr(model, betas, rot, transl, expr):
    betas, rot, expr = _cuda_f32(betas, 'betas'), _cuda_f32(rot, 'rot'), _cuda_f32(expr, 'expression')
    B, n_rot = rot.shape[0], rot.shape[1]
    if rot.shape[2:] != (3, 3) or betas.shape != (B, model.NB) or expr.shape != (B, model.NE):
        raise RuntimeError(f'rot must be (B, n_rot, 3, 3), betas ({B}, {model.NB}) and expr ({B}, {model.NE}), got '
                           f'{tuple(rot.shape)}, {tuple(betas.shape)} and {tuple(expr.shape)}')
    transl = None if transl is None else _cuda_f32(transl, 'transl')
    if transl is not None and transl.shape != (B, 3):
        raise RuntimeError(f'transl must be ({B}, 3), got {tuple(transl.shape)}')
    dev = betas.device
    kp = torch.empty(B, model.K, 3, dtype=torch.float32, device=dev)
    jac = torch.empty(B, 3 * model.K, 3 * n_rot + model.NB + model.NE + 3, dtype=torch.float32, device=dev)
    if B == 0:
        return kp, jac
    with torch.cuda.device(dev):
        check(lib().shapy_smplx_keypoint_jacobian_expr(model.handle, ptr(betas), ptr(expr), ptr(rot), n_rot, ptr(transl),
                                                       B, ptr(kp), ptr(jac), stream_ptr()),
              'smplx_keypoint_jacobian')
    return kp, jac


def fit_lm_keypoints_step(state, trial, targets, weights, lambda_up, lambda_down, first, trial_keypoints, trial_jac):
    """One Levenberg-Marquardt step per body of the keypoint fit (include/shapy_b200.h, shapy_fit_lm_keypoints_step),
    in place.  state: {'rot' (B, n_rot, 3, 3), 'betas' (B, NB), 'transl' (B, 3), 'keypoints' (B, K, 3), 'jac'
    (B, 3K, P), 'loss' (B,), 'lambda' (B,), 'accepted' (B,) int32}; trial: {'rot', 'betas', 'transl'}, the evaluated
    trial on entry and the next trial on return; targets (B, K, 3), weights (B, K)."""
    B, n_rot = trial['rot'].shape[:2]
    nb, K = trial['betas'].shape[1], targets.shape[1]
    ts = [state[k] for k in ('rot', 'betas', 'transl', 'keypoints', 'jac', 'loss', 'lambda')] + \
        [trial[k] for k in ('rot', 'betas', 'transl')] + [targets, weights, trial_keypoints, trial_jac]
    _check_step_tensors('fit_lm_keypoints_step', ts, 'the state, trial, targets and weights', state['accepted'])
    P = 3 * n_rot + nb + 3
    if not _kp_step_shapes_ok(state, trial_jac, weights, B, K, P):
        raise RuntimeError(f'fit_lm_keypoints_step: jac must be ({B}, {3 * K}, {P}) and weights ({B}, {K})')
    if B == 0:
        return
    with torch.cuda.device(trial['rot'].device):
        check(lib().shapy_fit_lm_keypoints_step(
            B, K, n_rot, nb, ptr(targets), ptr(weights), float(lambda_up), float(lambda_down), int(bool(first)),
            *[ptr(state[k]) for k in ('rot', 'betas', 'transl', 'keypoints', 'jac', 'loss', 'lambda', 'accepted')],
            ptr(trial['rot']), ptr(trial['betas']), ptr(trial['transl']), ptr(trial_keypoints), ptr(trial_jac),
            stream_ptr()), 'fit_lm_keypoints_step')


def fit_lm_keypoints_measurements_step(state, trial, targets, weights, meas_targets, meas_weights, betas_weight,
                                       lambda_up, lambda_down, first, trial_keypoints, trial_jac, trial_meas,
                                       trial_meas_jac):
    """fit_lm_keypoints_step with the five measurements and a betas regulariser stacked under the keypoint rows
    (include/shapy_b200.h, shapy_fit_lm_keypoints_measurements_step), in place.  state: fit_lm_keypoints_step's plus
    'meas' (B, 5) and 'meas_jac' (B, 5, NB); meas_targets, meas_weights (B, 5) in the order mass, height, chest, waist,
    hips; trial_meas (B, 5) / trial_meas_jac (B, 5, NB) from measure_jacobian_betas at the trial betas."""
    B, n_rot = trial['rot'].shape[:2]
    nb, K = trial['betas'].shape[1], targets.shape[1]
    ts = [state[k] for k in ('rot', 'betas', 'transl', 'keypoints', 'jac', 'meas', 'meas_jac', 'loss', 'lambda')] + \
        [trial[k] for k in ('rot', 'betas', 'transl')] + [targets, weights, meas_targets, meas_weights,
                                                          trial_keypoints, trial_jac, trial_meas, trial_meas_jac]
    what = 'fit_lm_keypoints_measurements_step'
    _check_step_tensors(what, ts, 'the state, trial, targets and weights', state['accepted'])
    P = 3 * n_rot + nb + 3
    if not _kp_step_shapes_ok(state, trial_jac, weights, B, K, P):
        raise RuntimeError(f'{what}: jac must be ({B}, {3 * K}, {P}) and weights ({B}, {K})')
    if not _meas_step_shapes_ok(state, trial_meas, trial_meas_jac, meas_targets, meas_weights, B, nb):
        raise RuntimeError(f'{what}: meas_jac must be ({B}, 5, {nb}) and the measurements, their targets and weights '
                           f'({B}, 5)')
    if B == 0:
        return
    with torch.cuda.device(trial['rot'].device):
        check(lib().shapy_fit_lm_keypoints_measurements_step(
            B, K, n_rot, nb, ptr(targets), ptr(weights), ptr(meas_targets), ptr(meas_weights), float(betas_weight),
            float(lambda_up), float(lambda_down), int(bool(first)),
            *[ptr(state[k]) for k in ('rot', 'betas', 'transl', 'keypoints', 'jac', 'meas', 'meas_jac', 'loss',
                                      'lambda', 'accepted')],
            ptr(trial['rot']), ptr(trial['betas']), ptr(trial['transl']), ptr(trial_keypoints), ptr(trial_jac),
            ptr(trial_meas), ptr(trial_meas_jac), stream_ptr()), what)


def _fit_lm_kp2d(what, state, trial, targets, weights, robust_sigma, pose_prior_weight, betas_weight, lambda_up,
                 lambda_down, first, trial_keypoints, trial_jac, pose_anchor, meas=None, intrinsics=None,
                 expressive=None):
    """What the single-image 2D keypoint steps share: the checks and the call, `meas` None or the measurement block
    (meas_targets, meas_weights, trial_meas, trial_meas_jac) of the stacked step, `intrinsics` None (the
    weak-perspective camera 'camera') or (B, 3) (the perspective steps, translation 'transl'), `expressive` None (the
    22-joint steps) or (expression_weight, joint_weights) of the expressive steps, whose state and trial hold
    'expression'."""
    B, n_rot = trial['rot'].shape[:2]
    nb, K = trial['betas'].shape[1], targets.shape[1]
    ex = expressive is not None
    opt = lambda cond, *xs: list(xs) if cond else []  # noqa: E731
    ne = trial['expression'].shape[1] if ex else 0
    last = 'camera' if intrinsics is None else 'transl'
    sigma = _check_kp2d_scalars(what, robust_sigma, pose_prior_weight, betas_weight, lambda_up, lambda_down,
                                pose_anchor)
    expression_weight, joint_weights = expressive or (0.0, None)
    if not expression_weight >= 0:
        raise ValueError(f'{what}: expression_weight must be >= 0')
    if joint_weights is not None:
        jw = torch.as_tensor(joint_weights, dtype=torch.float32)
        if jw.shape != (n_rot,):
            raise RuntimeError(f'{what}: joint_weights must be ({n_rot},)')
        if jw.device.type == 'cpu':
            if not (float(jw[0]) == 0 and bool((jw >= 0).all())):
                raise ValueError(f'{what}: joint_weights must be >= 0 with joint 0 zero')
            jw = jw.to(trial['rot'].device)
        if pose_anchor is None:
            raise ValueError(f'{what}: joint_weights need pose_anchor')
        joint_weights = jw.contiguous()
    ekeys, mkeys = opt(ex, 'expression'), opt(meas is not None, 'meas', 'meas_jac')
    params = ['rot', 'betas'] + ekeys + [last]
    ts = [state[k] for k in params + ['keypoints', 'jac', 'loss', 'lambda'] + mkeys] + [trial[k] for k in params] + \
        [targets, weights, trial_keypoints, trial_jac] + \
        [t for t in (pose_anchor, joint_weights, intrinsics) if t is not None] + list(meas or ())
    names = 'anchor, joint weights and intrinsics' if ex else 'anchor and intrinsics'
    _check_step_tensors(what, ts, f'the state, trial, targets, weights, {names}', state['accepted'])
    P = 3 * n_rot + nb + ne + 3
    if not _kp_step_shapes_ok(state, trial_jac, weights, B, K, P) or targets.shape != (B, K, 2) or \
            (ex and state['expression'].shape != (B, ne)):
        shapes = f'jac must be ({B}, {3 * K}, {P}), weights ({B}, {K})'
        shapes += f', targets ({B}, {K}, 2) and expression ({B}, {ne})' if ex else f' and targets ({B}, {K}, 2)'
        raise RuntimeError(f'{what}: {shapes}')
    if pose_anchor is not None and pose_anchor.shape != (B, n_rot, 3, 3):
        raise RuntimeError(f'{what}: pose_anchor must be ({B}, {n_rot}, 3, 3)')
    if intrinsics is not None and intrinsics.shape != (B, 3):
        raise RuntimeError(f'{what}: intrinsics must be ({B}, 3)')
    if meas is not None and not _meas_step_shapes_ok(state, meas[2], meas[3], meas[0], meas[1], B, nb):
        raise RuntimeError(f'{what}: meas_jac must be ({B}, 5, {nb}) and the measurements, their targets and weights '
                           f'({B}, 5)')
    if B == 0:
        return
    # the arguments in the order of the entry's C signature; a zero-width expression is passed as null
    e = (lambda t: ptr(t) if ne else None)  # noqa: E731
    head = [B, K, n_rot, nb, *opt(ex, ne), ptr(targets), ptr(weights), *opt(intrinsics is not None, ptr(intrinsics)),
            ptr(pose_anchor), *opt(ex, ptr(joint_weights)), sigma, float(pose_prior_weight), float(betas_weight),
            *opt(ex, float(expression_weight)), *map(ptr, (meas or ())[:2]), float(lambda_up), float(lambda_down),
            int(bool(first))]
    st = [ptr(state['rot']), ptr(state['betas'])] + [e(state[k]) for k in ekeys] + \
        [ptr(state[k]) for k in (last, 'keypoints', 'jac', *mkeys, 'loss', 'lambda', 'accepted')]
    tr = [ptr(trial['rot']), ptr(trial['betas'])] + [e(trial[k]) for k in ekeys] + \
        [ptr(trial[last]), ptr(trial_keypoints), ptr(trial_jac), *map(ptr, (meas or ())[2:])]
    entry = 'shapy_fit_lm_keypoints_2d' + '_expressive' * ex + '_perspective' * (intrinsics is not None) + \
        '_measurements' * (meas is not None) + '_step'
    with torch.cuda.device(trial['rot'].device):
        check(getattr(lib(), entry)(*head, *st, *tr, stream_ptr()), what)


def fit_lm_keypoints_2d_step(state, trial, targets, weights, robust_sigma, pose_prior_weight, betas_weight, lambda_up,
                             lambda_down, first, trial_keypoints, trial_jac, pose_anchor=None):
    """One Levenberg-Marquardt step per body of the fit of pose, shape and weak-perspective camera to 2D keypoints
    (include/shapy_b200.h, shapy_fit_lm_keypoints_2d_step), in place.  state: {'rot' (B, n_rot, 3, 3), 'betas' (B, NB),
    'camera' (B, 3), 'keypoints' (B, K, 3), 'jac' (B, 3K, P), 'loss' (B,), 'lambda' (B,), 'accepted' (B,) int32};
    trial: {'rot', 'betas', 'camera'}, the evaluated trial on entry and the next trial on return; trial_keypoints /
    trial_jac from smplx_keypoint_jacobian without transl; targets (B, K, 2), weights (B, K); robust_sigma None or inf
    for least squares; pose_anchor (B, n_rot, 3, 3), needed when pose_prior_weight > 0."""
    _fit_lm_kp2d('fit_lm_keypoints_2d_step', state, trial, targets, weights, robust_sigma, pose_prior_weight,
                 betas_weight, lambda_up, lambda_down, first, trial_keypoints, trial_jac, pose_anchor)


def fit_lm_keypoints_2d_measurements_step(state, trial, targets, weights, robust_sigma, pose_prior_weight, betas_weight,
                                          meas_targets, meas_weights, lambda_up, lambda_down, first, trial_keypoints,
                                          trial_jac, trial_meas, trial_meas_jac, pose_anchor=None):
    """fit_lm_keypoints_2d_step with the five measurements stacked under its rows (include/shapy_b200.h,
    shapy_fit_lm_keypoints_2d_measurements_step), in place.  state: fit_lm_keypoints_2d_step's plus 'meas' (B, 5) and
    'meas_jac' (B, 5, NB); meas_targets, meas_weights (B, 5) in the order mass, height, chest, waist, hips; trial_meas
    (B, 5) / trial_meas_jac (B, 5, NB) from measure_jacobian_betas at the trial betas.  betas_weight is the one betas
    regulariser, the 2D step's."""
    _fit_lm_kp2d('fit_lm_keypoints_2d_measurements_step', state, trial, targets, weights, robust_sigma,
                 pose_prior_weight, betas_weight, lambda_up, lambda_down, first, trial_keypoints, trial_jac,
                 pose_anchor, (meas_targets, meas_weights, trial_meas, trial_meas_jac))


def fit_lm_keypoints_2d_perspective_step(state, trial, targets, weights, intrinsics, robust_sigma, pose_prior_weight,
                                         betas_weight, lambda_up, lambda_down, first, trial_keypoints, trial_jac,
                                         pose_anchor=None):
    """fit_lm_keypoints_2d_step under a perspective camera with known intrinsics (include/shapy_b200.h,
    shapy_fit_lm_keypoints_2d_perspective_step), in place: p_k = f (Y_x / Y_z, Y_y / Y_z) + (px, py), Y_k = kp_k + t,
    camera frame x right, y down, z forward.  state and trial hold 'transl' (B, 3) in the place of 'camera';
    intrinsics (B, 3) = (f, px, py) in the units of targets (B, K, 2).  A trial with a weighted keypoint at Y_z <= 0 is
    rejected; a start with one reports NaN and does not move."""
    _fit_lm_kp2d('fit_lm_keypoints_2d_perspective_step', state, trial, targets, weights, robust_sigma,
                 pose_prior_weight, betas_weight, lambda_up, lambda_down, first, trial_keypoints, trial_jac,
                 pose_anchor, intrinsics=intrinsics)


def fit_lm_keypoints_2d_perspective_measurements_step(state, trial, targets, weights, intrinsics, robust_sigma,
                                                      pose_prior_weight, betas_weight, meas_targets, meas_weights,
                                                      lambda_up, lambda_down, first, trial_keypoints, trial_jac,
                                                      trial_meas, trial_meas_jac, pose_anchor=None):
    """fit_lm_keypoints_2d_perspective_step with the five measurements stacked under its rows (include/shapy_b200.h,
    shapy_fit_lm_keypoints_2d_perspective_measurements_step), with fit_lm_keypoints_2d_measurements_step's
    measurement block."""
    _fit_lm_kp2d('fit_lm_keypoints_2d_perspective_measurements_step', state, trial, targets, weights, robust_sigma,
                 pose_prior_weight, betas_weight, lambda_up, lambda_down, first, trial_keypoints, trial_jac,
                 pose_anchor, (meas_targets, meas_weights, trial_meas, trial_meas_jac), intrinsics)


def fit_lm_keypoints_2d_expressive_step(state, trial, targets, weights, robust_sigma, pose_prior_weight, betas_weight,
                                        expression_weight, lambda_up, lambda_down, first, trial_keypoints, trial_jac,
                                        pose_anchor=None, joint_weights=None, intrinsics=None):
    """One Levenberg-Marquardt step per body of the 2D fit of the whole SMPL-X body (include/shapy_b200.h,
    shapy_fit_lm_keypoints_2d_expressive_step, or _perspective_ with intrinsics), in place: any pose width and the
    facial expression, P = 3 n_rot + NB + NE + 3 <= 200.  state: fit_lm_keypoints_2d_step's (or the perspective step's,
    with 'transl') plus 'expression' (B, NE), NE >= 0; trial: {'rot', 'betas', 'expression', 'camera' or 'transl'};
    trial_keypoints / trial_jac from smplx_keypoint_jacobian(..., expr=trial['expression']) without transl (without
    expr when NE = 0).  joint_weights: None (pose_prior_weight on every joint j >= 1) or (n_rot,) float32 per-joint
    pose-prior weights, joint 0 zero (a CPU tensor is checked, then copied; a CUDA tensor is used as it is, its joint 0
    not read).  expression_weight: the regulariser expression_weight |psi|^2.  With NE = 0 and joint_weights None the
    step is fit_lm_keypoints_2d_step's (or the perspective step's) bit for bit."""
    _fit_lm_kp2d('fit_lm_keypoints_2d_expressive_step', state, trial, targets, weights, robust_sigma,
                 pose_prior_weight, betas_weight, lambda_up, lambda_down, first, trial_keypoints, trial_jac,
                 pose_anchor, intrinsics=intrinsics, expressive=(expression_weight, joint_weights))


def smplx_backward_shape(model: SmplxModel, grad_v_shaped) -> torch.Tensor:
    """grad_betas (B, NB) = shapedirs^T . grad_v_shaped (B, V, 3): the adjoint of smplx_forward_shape."""
    g = _cuda_f32(grad_v_shaped, 'grad_v_shaped')
    B = g.shape[0]
    if g.shape != (B, model.V, 3):
        raise RuntimeError(f'grad_v_shaped must be ({B}, {model.V}, 3), got {tuple(g.shape)}')
    out = torch.empty(B, model.NB, dtype=torch.float32, device=g.device)
    if B == 0:
        return out
    with torch.cuda.device(g.device):
        nbytes = lib().shapy_smplx_backward_shape_workspace_bytes(model.handle, B)
        ws = _WS.get('shape_bwd', nbytes, g.device)
        check(lib().shapy_smplx_backward_shape(model.handle, ptr(g), B, ptr(out), ptr(ws), ws.numel(), stream_ptr()),
              'smplx_backward_shape')
    return out


def mesh_to_mesh_forward(query_triangles, target_triangles, max_collisions=16, print_timings=False):
    """Drop-in for mesh_mesh_intersect_cuda.mesh_to_mesh_forward (bind.cpp:59-64).

    Query and target triangles are both float32 or both float64, as the reference dispatches them; `collision_bcs`
    takes their dtype.  The float64 path keeps the reference's double-instantiation semantics, including the points
    where it rounds to float (see shapy_mmi_forward_f64 in include/shapy_b200.h).  Mixed, half and bfloat16 inputs
    raise RuntimeError before anything is launched."""
    for name, t in (('query_triangles', query_triangles), ('target_triangles', target_triangles)):
        if not (torch.is_tensor(t) and t.is_cuda):
            raise RuntimeError(f'{name} must be a CUDA tensor')
        if not t.is_contiguous():
            raise RuntimeError(f'{name} must be contiguous')
    dtype = query_triangles.dtype
    if target_triangles.dtype != dtype or dtype not in (torch.float32, torch.float64):
        raise RuntimeError(f'shapy_b200 mesh_to_mesh_forward: query and target triangles must both be float32 or both '
                           f'float64, got {dtype} and {target_triangles.dtype}')
    f64 = dtype == torch.float64
    B, Q = query_triangles.shape[:2]
    F = target_triangles.shape[1]
    dev = query_triangles.device
    M = int(max_collisions)
    faces = torch.empty(B, Q * M, dtype=torch.int64, device=dev)
    bcs = torch.empty(B, Q * M, 2, 3, dtype=dtype, device=dev)
    if B == 0 or Q == 0:
        return [faces, bcs]
    if F == 0:            # nothing to collide with: every slot is "no collision"
        return [faces.fill_(-1), bcs.zero_()]
    L = lib()
    ws_bytes, forward = ((L.shapy_mmi_workspace_bytes_f64, L.shapy_mmi_forward_f64) if f64 else
                         (L.shapy_mmi_workspace_bytes, L.shapy_mmi_forward))
    with torch.cuda.device(dev):
        ws = _WS.get('mmi', ws_bytes(B, Q, F), dev)
        check(forward(ptr(query_triangles), ptr(target_triangles), B, Q, F, M, ptr(faces), ptr(bcs),
                      ptr(ws), ws.numel(), stream_ptr()), 'mmi_forward_f64' if f64 else 'mmi_forward')
    return [faces, bcs]


# -------------------------------------------------------------------------------------------- scans
MAX_SCAN_FACES = 32768       # faces of a mesh the scan queries take (the tree's shared-memory sort)
MAX_SCAN_POINTS = 32768      # scan points per body (the point tree's and the backward's shared-memory sorts)


def _scan_points(points, weights, B=None):
    """points (B, N, 3) and weights (B, N) or None as the scan entries take them; ValueError past the limits."""
    p = _cuda_f32(points, 'points')
    if p.dim() != 3 or p.shape[2] != 3 or (B is not None and p.shape[0] != B):
        raise ValueError(f'points must be ({"B" if B is None else B}, N, 3), got {tuple(p.shape)}')
    if p.shape[1] > MAX_SCAN_POINTS:
        raise ValueError(f'{p.shape[1]} scan points per body exceed the {MAX_SCAN_POINTS} supported: subsample the scan')
    if weights is not None:
        weights = _cuda_f32(weights, 'weights')
        if weights.shape != p.shape[:2]:
            raise ValueError(f'weights must be {tuple(p.shape[:2])}, got {tuple(weights.shape)}')
    return p, weights


def _scan_mesh(vertices, faces_i32):
    v = _cuda_f32(vertices, 'vertices')
    faces_i32 = _faces_i32(faces_i32)
    if v.dim() != 3 or v.shape[2] != 3 or faces_i32.dim() != 2 or faces_i32.shape[1] != 3 or faces_i32.shape[0] == 0:
        raise ValueError(f'vertices must be (B, V, 3) and faces (F >= 1, 3), got {tuple(v.shape)} and '
                         f'{tuple(faces_i32.shape)}')
    if faces_i32.shape[0] > MAX_SCAN_FACES:
        raise ValueError(f'{faces_i32.shape[0]} faces exceed the {MAX_SCAN_FACES} the scan queries support')
    return v, faces_i32


class ScanTree:
    """The workspace of closest_points holding its LBVH, for a later call to refit instead of rebuilding."""

    def __init__(self):
        self.ws, self.key = None, None


def closest_points(vertices, faces_i32, points, weights=None, tree=None):
    """Exact closest point of each scan point on its body's mesh (include/shapy_b200.h, shapy_closest_points):
    vertices (B, V, 3), faces_i32 (F, 3) int32, points (B, N, 3), weights (B, N) or None.  Returns (face_idx (B, N)
    int32, bary (B, N, 3), sq_dist (B, N)); a point with weight <= 0 is never read and gets face -1, distance 0.
    tree: a ScanTree; the first call with it builds the tree in it, the next ones with the same batch size and faces
    refit it (the same bits as a fresh build)."""
    v, faces_i32 = _scan_mesh(vertices, faces_i32)
    B, V, F = v.shape[0], v.shape[1], faces_i32.shape[0]
    p, w = _scan_points(points, weights, B)
    N, dev = p.shape[1], v.device
    face = torch.empty(B, N, dtype=torch.int32, device=dev)
    bary = torch.empty(B, N, 3, dtype=torch.float32, device=dev)
    d2 = torch.empty(B, N, dtype=torch.float32, device=dev)
    if B == 0 or N == 0:
        return face, bary, d2
    _incidence_rows(faces_i32, V)          # checks that the faces index the vertices (cached for the backward)
    with torch.cuda.device(dev):
        nbytes = lib().shapy_closest_points_workspace_bytes(B, F)
        key = (B, F, faces_i32.data_ptr(), faces_i32._version, dev.index)
        if tree is None:
            ws, refit = _WS.get('scan', nbytes, dev), 0
        else:
            refit = int(tree.key == key)
            if not refit:
                tree.ws, tree.key = _workspace(nbytes, dev), key
            ws = tree.ws
        check(lib().shapy_closest_points(ptr(v), ptr(faces_i32), B, V, F, ptr(p), N, ptr(w), refit, ptr(face),
                                         ptr(bary), ptr(d2), ptr(ws), ws.numel(), stream_ptr()), 'closest_points')
    return face, bary, d2


def nearest_points(queries, points, weights=None):
    """Nearest kept scan point of each query (include/shapy_b200.h, shapy_nearest_points): queries (B, Q, 3), points
    (B, N, 3), weights (B, N) or None.  Returns (idx (B, Q) int32, sq_dist (B, Q)); idx -1 and distance 0 for a body
    without a point of weight > 0."""
    q = _cuda_f32(queries, 'queries')
    if q.dim() != 3 or q.shape[2] != 3:
        raise ValueError(f'queries must be (B, Q, 3), got {tuple(q.shape)}')
    B, Q = q.shape[:2]
    p, w = _scan_points(points, weights, B)
    N, dev = p.shape[1], q.device
    if N == 0:
        return (torch.full((B, Q), -1, dtype=torch.int32, device=dev),
                torch.zeros(B, Q, dtype=torch.float32, device=dev))
    idx = torch.empty(B, Q, dtype=torch.int32, device=dev)
    d2 = torch.empty(B, Q, dtype=torch.float32, device=dev)
    if B == 0 or Q == 0:
        return idx, d2
    with torch.cuda.device(dev):
        ws = _WS.get('scan_nn', lib().shapy_nearest_points_workspace_bytes(B, N), dev)
        check(lib().shapy_nearest_points(ptr(q), B, Q, ptr(p), N, ptr(w), ptr(idx), ptr(d2), ptr(ws), ws.numel(),
                                         stream_ptr()), 'nearest_points')
    return idx, d2


def closest_points_backward(vertices, faces_i32, points, face_idx, bary, grad_sq_dist):
    """Gradient (B, V, 3) of closest_points' sq_dist with respect to the vertices, face and barycentrics held at the
    forward's values (include/shapy_b200.h, shapy_closest_points_backward): deterministic, no atomics, one launch."""
    v, faces_i32 = _scan_mesh(vertices, faces_i32)
    B, V, F = v.shape[0], v.shape[1], faces_i32.shape[0]
    p, _ = _scan_points(points, None, B)
    N = p.shape[1]
    g = _cuda_f32(grad_sq_dist, 'grad_sq_dist')
    bary = _cuda_f32(bary, 'bary')
    if not (torch.is_tensor(face_idx) and face_idx.is_cuda and face_idx.dtype == torch.int32):
        raise RuntimeError('face_idx must be a CUDA int32 tensor')
    face_idx = face_idx.contiguous()
    if g.shape != (B, N) or face_idx.shape != (B, N) or bary.shape != (B, N, 3):
        raise ValueError(f'grad_sq_dist and face_idx must be ({B}, {N}) and bary ({B}, {N}, 3)')
    grad = torch.empty_like(v)
    if B == 0:
        return grad
    with torch.cuda.device(v.device):
        inc_ptr, inc = _incidence_rows(faces_i32, V)
        check(lib().shapy_closest_points_backward(ptr(v), ptr(faces_i32), ptr(inc_ptr), ptr(inc), B, V, F, ptr(p), N,
                                                  ptr(face_idx), ptr(bary), ptr(g), ptr(grad), stream_ptr()),
              'closest_points_backward')
    return grad


# ---------------------------------------------------------------------------------------------- self-penetration
MAX_PART_LABELS = 64          # part labels of the self-collision filter (one 64-bit mask per label)
MAX_PENETRATION_PAIRS = 4096  # rows per body the penetration loss takes (its backward's shared-memory sort)


def make_part_filter(part_labels, ignored_part_pairs, F, device):
    """The part filter of self_collisions on the device: (labels (F,) int32, masks (64,) uint64 as int64), or (None,
    None) without labels.  Built on the host (one copy to the device): a loop builds it once and passes it as
    self_collisions(part_filter=...)."""
    if part_labels is None:
        if ignored_part_pairs:
            raise ValueError('ignored_part_pairs needs part_labels')
        return None, None
    lab = torch.as_tensor(part_labels).reshape(-1)
    if lab.numel() != F:
        raise ValueError(f'part_labels must have one label per face ({F}), got {lab.numel()}')
    lab_h = lab.detach().cpu().numpy().astype(np.int64)
    if lab_h.size and (lab_h.min() < 0 or lab_h.max() >= MAX_PART_LABELS):
        raise ValueError(f'part labels must lie in [0, {MAX_PART_LABELS})')
    masks = np.zeros(MAX_PART_LABELS, np.uint64)
    for i, j in (ignored_part_pairs or ()):
        i, j = int(i), int(j)
        if not (0 <= i < MAX_PART_LABELS and 0 <= j < MAX_PART_LABELS):
            raise ValueError(f'ignored part pair {(i, j)} outside [0, {MAX_PART_LABELS})')
        masks[i] |= np.uint64(1) << np.uint64(j)
        masks[j] |= np.uint64(1) << np.uint64(i)
    return (torch.from_numpy(lab_h.astype(np.int32)).to(device),
            torch.from_numpy(masks.view(np.int64)).to(device))


def self_collisions(vertices, faces_i32, max_pairs, tree=None, part_labels=None, ignored_part_pairs=None,
                    part_filter=None):
    """Intersecting face pairs of each posed mesh (include/shapy_b200.h, shapy_self_collisions): vertices (B, V, 3),
    faces_i32 (F, 3) int32, F <= MAX_SCAN_FACES.  A pair (f, g), f < g, is kept when the faces share no vertex, their
    triangles' boxes overlap and the 11-axis SAT of mesh_to_mesh_forward finds them intersecting, and, with
    part_labels (F,) in [0, 64), the unordered label pair is not in ignored_part_pairs (pairs of labels).  Returns
    (pairs (B, max_pairs, 2) int32 in ascending (f, g) order padded with -1, count (B,) int32 the number found, which
    exceeds max_pairs when rows were cut).  The pairs are the same bits whatever the tree, the batch or the run.
    tree: the ops.ScanTree of closest_points; a call with the same batch size and faces refits it.  part_filter: the
    device tensors of ops.make_part_filter in place of part_labels / ignored_part_pairs (no host work)."""
    v, faces_i32 = _scan_mesh(vertices, faces_i32)
    B, V, F = v.shape[0], v.shape[1], faces_i32.shape[0]
    max_pairs, dev = int(max_pairs), v.device
    if max_pairs < 0:
        raise ValueError('max_pairs must be >= 0')
    if part_filter is None:
        labels, masks = make_part_filter(part_labels, ignored_part_pairs, F, dev)
    else:
        labels, masks = part_filter
        if labels is not None and not (labels.is_cuda and labels.dtype == torch.int32 and labels.shape == (F,) and
                                       masks.is_cuda and masks.shape == (MAX_PART_LABELS,)):
            raise ValueError(f'part_filter must be ops.make_part_filter(..., {F}, device)')
    pairs = torch.empty(B, max_pairs, 2, dtype=torch.int32, device=dev)
    count = torch.empty(B, dtype=torch.int32, device=dev)
    if B == 0:
        return pairs, count
    _incidence_rows(faces_i32, V)          # checks that the faces index the vertices
    with torch.cuda.device(dev):
        nbytes = lib().shapy_self_collisions_workspace_bytes(B, F)
        key = (B, F, faces_i32.data_ptr(), faces_i32._version, dev.index)
        if tree is None:
            ws, refit = _WS.get('self', nbytes, dev), 0
        else:
            refit = int(tree.key == key and tree.ws.numel() >= nbytes)
            if not refit:
                tree.ws, tree.key = _workspace(max(nbytes, lib().shapy_closest_points_workspace_bytes(B, F)), dev), key
            ws = tree.ws
        check(lib().shapy_self_collisions(ptr(v), ptr(faces_i32), B, V, F, ptr(labels), ptr(masks), refit, max_pairs,
                                          ptr(pairs), ptr(count), ptr(ws), ws.numel(), stream_ptr()), 'self_collisions')
    return pairs, count


def face_parts(body_model):
    """Each face's part: the joint with the largest lbs weight summed over the face's three vertices, the lower joint
    index on a tie.  body_model: a mapping or object with `lbs_weights` (V, J) and `faces_tensor` (F, 3) (the
    reference's buffer names).  Returns (F,) int64 on the CPU."""
    get = body_model.get if isinstance(body_model, dict) else lambda k: getattr(body_model, k)
    w = torch.as_tensor(get('lbs_weights')).detach().cpu().double()
    faces = torch.as_tensor(get('faces_tensor')).detach().cpu().long()
    return w[faces].sum(dim=1).argmax(dim=1)          # argmax returns the first maximum


def parent_child_part_pairs(parents):
    """The (joint, parent) label pairs of a kinematic tree (parents[0] < 0 is the root): the creases at every joint,
    for self_collisions' ignored_part_pairs."""
    p = torch.as_tensor(parents).reshape(-1).tolist()
    return [(j, int(q)) for j, q in enumerate(p) if int(q) >= 0]


def _penetration_args(vertices, faces_i32, pairs, sigma, linear_max):
    v = _cuda_f32(vertices, 'vertices')
    faces_i32 = _faces_i32(faces_i32)
    if v.dim() != 3 or v.shape[2] != 3 or faces_i32.dim() != 2 or faces_i32.shape[1] != 3 or faces_i32.shape[0] == 0:
        raise ValueError(f'vertices must be (B, V, 3) and faces (F >= 1, 3), got {tuple(v.shape)} and '
                         f'{tuple(faces_i32.shape)}')
    if not (torch.is_tensor(pairs) and pairs.is_cuda and pairs.dtype == torch.int32):
        raise RuntimeError('pairs must be a CUDA int32 tensor')
    pairs = pairs.contiguous()
    if pairs.dim() != 3 or pairs.shape[0] != v.shape[0] or pairs.shape[2] != 2:
        raise ValueError(f'pairs must be ({v.shape[0]}, C, 2), got {tuple(pairs.shape)}')
    if pairs.shape[1] > MAX_PENETRATION_PAIRS:
        raise ValueError(f'{pairs.shape[1]} pair rows per body exceed the {MAX_PENETRATION_PAIRS} supported')
    if not (float(sigma) > 0) or float(linear_max) != float(linear_max):
        raise ValueError('sigma must be > 0 and linear_max not NaN')
    _incidence_rows(faces_i32, v.shape[1])          # the faces index the vertices
    return v, faces_i32, pairs


def penetration_forward(vertices, faces_i32, pairs, sigma=0.5, penalize_outside=True, linear_max=1000.0):
    """The distance-field penetration loss (B,) of DistanceFieldPenetrationLoss at the (receiver, intruder) face rows
    pairs (B, C, 2) int32 (include/shapy_b200.h, shapy_penetration_forward): a row whose first index is < 0 is
    skipped.  One launch, deterministic."""
    v, faces_i32, pairs = _penetration_args(vertices, faces_i32, pairs, sigma, linear_max)
    B, V, F, Cn = v.shape[0], v.shape[1], faces_i32.shape[0], pairs.shape[1]
    loss = torch.empty(B, dtype=torch.float32, device=v.device)
    if B == 0:
        return loss
    with torch.cuda.device(v.device):
        check(lib().shapy_penetration_forward(ptr(v), ptr(faces_i32), B, V, F, ptr(pairs), Cn, float(sigma),
                                              int(bool(penalize_outside)), float(linear_max), ptr(loss), stream_ptr()),
              'penetration_forward')
    return loss


def penetration_backward(vertices, faces_i32, pairs, grad_loss, sigma=0.5, penalize_outside=True, linear_max=1000.0):
    """Gradient (B, V, 3) of grad_loss (B,) . penetration_forward with respect to the vertices, the pairs held
    constant (include/shapy_b200.h, shapy_penetration_backward): one launch, no atomics, bit-identical run to run."""
    v, faces_i32, pairs = _penetration_args(vertices, faces_i32, pairs, sigma, linear_max)
    B, V, F, Cn = v.shape[0], v.shape[1], faces_i32.shape[0], pairs.shape[1]
    g = _cuda_f32(grad_loss, 'grad_loss')
    if g.shape != (B,):
        raise ValueError(f'grad_loss must be ({B},), got {tuple(g.shape)}')
    grad = torch.empty_like(v)
    if B == 0:
        return grad
    with torch.cuda.device(v.device):
        ws = _WS.get('penetration', lib().shapy_penetration_workspace_bytes(B, Cn), v.device)
        check(lib().shapy_penetration_backward(ptr(v), ptr(faces_i32), B, V, F, ptr(pairs), Cn, float(sigma),
                                               int(bool(penalize_outside)), float(linear_max), ptr(g), ptr(grad),
                                               ptr(ws), ws.numel(), stream_ptr()), 'penetration_backward')
    return grad


# ---------------------------------------------------------------------------------------------- silhouettes
MAX_SILHOUETTE_SIDE = 4096    # mask height and width (the distance transform's row pass keeps a row in shared memory)


def _silhouette_size(what, height, width):
    if not (1 <= int(height) <= MAX_SILHOUETTE_SIDE and 1 <= int(width) <= MAX_SILHOUETTE_SIDE):
        raise ValueError(f'{what}: masks must be at least 1 x 1 and at most {MAX_SILHOUETTE_SIDE} x '
                         f'{MAX_SILHOUETTE_SIDE}, got {int(height)} x {int(width)}')
    return int(height), int(width)


def _silhouette_camera(what, vertices, intrinsics):
    v = _cuda_f32(vertices, 'vertices')
    if v.dim() != 3 or v.shape[2] != 3 or v.shape[1] == 0:
        raise ValueError(f'{what}: vertices must be (B, V >= 1, 3), got {tuple(v.shape)}')
    intr = _cuda_f32(intrinsics, 'intrinsics')
    if intr.shape != (v.shape[0], 3):
        raise ValueError(f'{what}: intrinsics must be ({v.shape[0]}, 3) (f, px, py), got {tuple(intr.shape)}')
    return v, intr


def _silhouette_dist(what, dist, B):
    d = _cuda_f32(dist, 'dist')
    if d.dim() != 3 or d.shape[0] != B:
        raise ValueError(f'{what}: dist must be ({B}, H, W), got {tuple(d.shape)}')
    _silhouette_size(what, d.shape[1], d.shape[2])
    return d


def silhouette_prepare(masks, max_points):
    """The distance transform and contour of person masks (include/shapy_b200.h, shapy_silhouette_prepare): masks (B, H,
    W) uint8 or bool on the device, nonzero a person pixel, H, W <= MAX_SILHOUETTE_SIDE; max_points in [1,
    MAX_SCAN_POINTS].  Returns (dist (B, H, W), contour (B, max_points, 3), contour_w (B, max_points), count (B,) int32):
    the exact Euclidean distance to the nearest person pixel (0 inside, 0 everywhere for an empty mask), the kept
    contour pixels (c, r, 0) in raster order then zero padding, their weights (1 kept, 0 padding) and the number of
    contour pixels found.  Five launches, deterministic."""
    if not (torch.is_tensor(masks) and masks.is_cuda and masks.dtype in (torch.uint8, torch.bool)):
        raise ValueError('silhouette_prepare: masks must be a CUDA uint8 or bool tensor')
    if masks.dim() != 3:
        raise ValueError(f'silhouette_prepare: masks must be (B, H, W), got {tuple(masks.shape)}')
    B = masks.shape[0]
    H, W = _silhouette_size('silhouette_prepare', masks.shape[1], masks.shape[2])
    max_points = int(max_points)
    if not 1 <= max_points <= MAX_SCAN_POINTS:
        raise ValueError(f'silhouette_prepare: max_points must be in [1, {MAX_SCAN_POINTS}], got {max_points}')
    m = masks.contiguous()
    if m.dtype == torch.bool:
        m = m.view(torch.uint8)
    dev = m.device
    dist = torch.empty(B, H, W, dtype=torch.float32, device=dev)
    contour = torch.empty(B, max_points, 3, dtype=torch.float32, device=dev)
    contour_w = torch.empty(B, max_points, dtype=torch.float32, device=dev)
    count = torch.empty(B, dtype=torch.int32, device=dev)
    if B == 0:
        return dist, contour, contour_w, count
    with torch.cuda.device(dev):
        ws = _WS.get('silhouette', lib().shapy_silhouette_workspace_bytes(B, H), dev)
        check(lib().shapy_silhouette_prepare(ptr(m), B, H, W, max_points, ptr(dist), ptr(contour), ptr(contour_w),
                                             ptr(count), ptr(ws), ws.numel(), stream_ptr()), 'silhouette_prepare')
    return dist, contour, contour_w, count


def silhouette_forward(vertices, intrinsics, dist):
    """The model -> mask half of the silhouette term (include/shapy_b200.h, shapy_silhouette_forward): vertices (B, V,
    3) in the camera frame, intrinsics (B, 3) (f, px, py), dist (B, H, W) of silhouette_prepare.  Returns (projected
    (B, V, 3) = (u, v, 0) at the depth max(Y_z, 1e-3), model_to_mask (B,) = the mean over the vertices of the squared
    bilinear distance at the projection clamped to the image).  One launch, deterministic."""
    v, intr = _silhouette_camera('silhouette_forward', vertices, intrinsics)
    B, V = v.shape[:2]
    d = _silhouette_dist('silhouette_forward', dist, B)
    proj = torch.empty_like(v)
    m2m = torch.empty(B, dtype=torch.float32, device=v.device)
    if B == 0:
        return proj, m2m
    with torch.cuda.device(v.device):
        check(lib().shapy_silhouette_forward(ptr(v), ptr(intr), ptr(d), B, V, d.shape[1], d.shape[2], ptr(proj),
                                             ptr(m2m), stream_ptr()), 'silhouette_forward')
    return proj, m2m


def silhouette_backward(vertices, intrinsics, dist, grad_model_to_mask, grad_projected=None):
    """Gradient (B, V, 3) of grad_model_to_mask (B,) . model_to_mask + <grad_projected, projected> of
    silhouette_forward with respect to the vertices (include/shapy_b200.h, shapy_silhouette_backward); grad_projected
    (B, V, 3) or None, its z unread.  One launch, no atomics."""
    v, intr = _silhouette_camera('silhouette_backward', vertices, intrinsics)
    B, V = v.shape[:2]
    d = _silhouette_dist('silhouette_backward', dist, B)
    g = _cuda_f32(grad_model_to_mask, 'grad_model_to_mask')
    if g.shape != (B,):
        raise ValueError(f'silhouette_backward: grad_model_to_mask must be ({B},), got {tuple(g.shape)}')
    if grad_projected is not None:
        grad_projected = _cuda_f32(grad_projected, 'grad_projected')
        if grad_projected.shape != v.shape:
            raise ValueError(f'silhouette_backward: grad_projected must be {tuple(v.shape)}, got '
                             f'{tuple(grad_projected.shape)}')
    grad = torch.empty_like(v)
    if B == 0:
        return grad
    with torch.cuda.device(v.device):
        check(lib().shapy_silhouette_backward(ptr(v), ptr(intr), ptr(d), B, V, d.shape[1], d.shape[2], ptr(g),
                                              ptr(grad_projected), ptr(grad), stream_ptr()), 'silhouette_backward')
    return grad


def render_silhouette(vertices, faces_i32, intrinsics, height, width):
    """The silhouette (B, height, width) bool of each posed mesh (include/shapy_b200.h, shapy_render_silhouette): a
    pixel is set when its centre lies inside a projected triangle whose three vertices have Y_z > 0.  vertices (B, V, 3)
    in the camera frame, faces_i32 (F, 3), intrinsics (B, 3) (f, px, py).  Bit-identical run to run and alone or in a
    batch."""
    v, intr = _silhouette_camera('render_silhouette', vertices, intrinsics)
    H, W = _silhouette_size('render_silhouette', height, width)
    faces_i32 = _faces_i32(faces_i32)
    if faces_i32.dim() != 2 or faces_i32.shape[1] != 3:
        raise ValueError(f'render_silhouette: faces must be (F, 3), got {tuple(faces_i32.shape)}')
    B, V = v.shape[:2]
    mask = torch.empty(B, H, W, dtype=torch.bool, device=v.device)
    if B == 0:
        return mask
    with torch.cuda.device(v.device):
        check(lib().shapy_render_silhouette(ptr(v), ptr(faces_i32), ptr(intr), B, V, faces_i32.shape[0], H, W,
                                            ptr(mask.view(torch.uint8)), stream_ptr()), 'render_silhouette')
    return mask


def fit_lm_scan_workspace(B, N, V, P, device):
    """The scratch of fit_lm_scan_step (include/shapy_b200.h, shapy_fit_lm_scan_workspace_bytes): a uint8 CUDA tensor,
    allocated once before an LM loop."""
    return _workspace(lib().shapy_fit_lm_scan_workspace_bytes(int(B), int(N), int(V), int(P)), device)


def fit_lm_scan_penetration_workspace(B, N, V, P, C, device):
    """The scratch of fit_lm_scan_step with `penetration` rows of C pairs per body
    (shapy_fit_lm_scan_penetration_workspace_bytes)."""
    return _workspace(lib().shapy_fit_lm_scan_penetration_workspace_bytes(int(B), int(N), int(V), int(P), int(C)),
                      device)


def fit_lm_scan_step(state, trial, points, weights, faces_i32, robust_sigma, scan_to_model_weight,
                     model_to_scan_weight, pose_prior_weight, betas_weight, lambda_up, lambda_down, first,
                     trial_vertices, trial_jac, trial_face_idx, trial_bary, trial_nearest, workspace, pose_anchor=None,
                     meas=None, penetration=None):
    """One Levenberg-Marquardt step per body of the scan fit (include/shapy_b200.h, shapy_fit_lm_scan_step), in place.
    state: {'rot' (B, n_rot, 3, 3), 'betas' (B, NB), 'transl' (B, 3), 'A' (B, P, P) and 'g' (B, P) float64, 'loss',
    'lambda' (B,), 'accepted' (B,) int32}, with meas also 'meas' (B, 5) and 'meas_jac' (B, 5, NB); trial: {'rot',
    'betas', 'transl'}, the evaluated trial on entry and the next trial on return.  points (B, N, 3), weights (B, N),
    faces_i32 (F, 3); the trial's vertices and Jacobian (smplx_vertex_jacobian, with transl), closest points
    (closest_points) and nearest points (nearest_points; None when model_to_scan_weight is 0).  robust_sigma None or
    inf: least squares.  meas: None or (meas_targets, meas_weights, trial_meas, trial_meas_jac).  workspace:
    fit_lm_scan_workspace(B, N, V, P).  penetration: None, or (pairs (B, C, 2) int32 of self_collisions on the trial's
    vertices, weight, sigma): the self-penetration rows (shapy_fit_lm_scan_penetration_step), with workspace
    fit_lm_scan_penetration_workspace(B, N, V, P, C)."""
    what = 'fit_lm_scan_step'
    B, n_rot = trial['rot'].shape[:2]
    nb, (N, V) = trial['betas'].shape[1], (points.shape[1], trial_vertices.shape[1])
    P = 3 * n_rot + nb + 3
    sigma = float('inf') if robust_sigma is None else float(robust_sigma)
    if not (sigma > 0 and pose_prior_weight >= 0 and betas_weight >= 0 and 0 <= scan_to_model_weight < float('inf')
            and 0 <= model_to_scan_weight < float('inf') and lambda_up >= 1 and lambda_down >= 1):
        raise ValueError(f'{what}: robust_sigma must be > 0, the term weights finite and >= 0, the prior weights >= 0 '
                         'and lambda_up and lambda_down >= 1')
    if pose_prior_weight > 0 and pose_anchor is None:
        raise ValueError(f'{what}: a pose prior needs pose_anchor')
    if model_to_scan_weight > 0 and trial_nearest is None:
        raise ValueError(f'{what}: the model -> scan term needs trial_nearest')
    mkeys = ['meas', 'meas_jac'] if meas is not None else []
    f32 = [state[k] for k in ['rot', 'betas', 'transl', 'loss', 'lambda'] + mkeys] + \
        [trial[k] for k in ('rot', 'betas', 'transl')] + [points, weights, trial_vertices, trial_jac, trial_bary] + \
        [t for t in (pose_anchor,) if t is not None] + list(meas or ())
    _check_step_tensors(what, f32, 'the state, trial, points, weights, vertices, Jacobian, barycentrics and anchor',
                        state['accepted'])
    for t in [state['A'], state['g']]:
        if not (t.is_cuda and t.is_contiguous() and t.dtype == torch.float64):
            raise RuntimeError(f"{what}: state['A'] and state['g'] must be contiguous float64 CUDA tensors")
    for t in [faces_i32, trial_face_idx] + ([] if trial_nearest is None else [trial_nearest]):
        if not (torch.is_tensor(t) and t.is_cuda and t.is_contiguous() and t.dtype == torch.int32):
            raise RuntimeError(f'{what}: faces, face_idx and nearest must be contiguous int32 CUDA tensors')
    shapes_ok = (points.shape == (B, N, 3) and weights.shape == (B, N) and trial_vertices.shape == (B, V, 3) and
                 trial_jac.shape == (B, V, 3, P) and trial_face_idx.shape == (B, N) and trial_bary.shape == (B, N, 3)
                 and (trial_nearest is None or trial_nearest.shape == (B, V)) and state['A'].shape == (B, P, P) and
                 state['g'].shape == (B, P) and (pose_anchor is None or pose_anchor.shape == (B, n_rot, 3, 3)))
    if not shapes_ok:
        raise RuntimeError(f'{what}: points must be ({B}, {N}, 3), weights, face_idx ({B}, {N}), bary ({B}, {N}, 3), '
                           f'vertices ({B}, {V}, 3), jac ({B}, {V}, 3, {P}), nearest ({B}, {V}), A ({B}, {P}, {P}), '
                           f'g ({B}, {P}) and pose_anchor ({B}, {n_rot}, 3, 3)')
    if meas is not None and not _meas_step_shapes_ok(state, meas[2], meas[3], meas[0], meas[1], B, nb):
        raise RuntimeError(f'{what}: meas_jac must be ({B}, 5, {nb}) and the measurements, their targets and weights '
                           f'({B}, 5)')
    if B == 0:
        return
    m = list(meas) if meas is not None else [None] * 4
    head = (B, N, V, n_rot, nb, ptr(points), ptr(weights), ptr(faces_i32))
    terms = (sigma, float(scan_to_model_weight), float(model_to_scan_weight), float(pose_prior_weight),
             float(betas_weight), ptr(m[0]), ptr(m[1]))
    if penetration is None:
        L, args = lib().shapy_fit_lm_scan_step, head + (ptr(pose_anchor),) + terms
    else:
        pairs, pw_, psig = penetration
        if not (torch.is_tensor(pairs) and pairs.is_cuda and pairs.is_contiguous() and pairs.dtype == torch.int32
                and pairs.dim() == 3 and pairs.shape[0] == B and pairs.shape[2] == 2):
            raise RuntimeError(f'{what}: the penetration pairs must be a contiguous int32 CUDA ({B}, C, 2) tensor')
        _incidence_rows(faces_i32, V)      # the faces index the vertices
        L = lib().shapy_fit_lm_scan_penetration_step
        args = head + (faces_i32.shape[0], ptr(pose_anchor)) + terms + (ptr(pairs), pairs.shape[1], float(pw_),
                                                                          float(psig))
    with torch.cuda.device(points.device):
        check(L(
            *args, float(lambda_up), float(lambda_down), int(bool(first)),
            *[ptr(state[k]) for k in ('rot', 'betas', 'transl', 'A', 'g')],
            *[ptr(state.get(k)) for k in ('meas', 'meas_jac')],
            *[ptr(state[k]) for k in ('loss', 'lambda', 'accepted')],
            *[ptr(trial[k]) for k in ('rot', 'betas', 'transl')], ptr(trial_vertices), ptr(trial_jac),
            ptr(trial_face_idx), ptr(trial_bary), ptr(trial_nearest), ptr(m[2]), ptr(m[3]), ptr(workspace),
            workspace.numel(), stream_ptr()), what)


# -------------------------------------------------------------------------------------------- head
def head_forward(feats, W0, b0, W1, b1, W2, b2, mean, num_stages=3):
    feats = _cuda_f32(feats, 'features')
    B, Fd = feats.shape
    P = mean.numel()
    h0, h1 = W0.shape[0], W1.shape[0]
    out = torch.empty(num_stages, B, P, dtype=torch.float32, device=feats.device)
    ts = [_cuda_f32(t, 'head weight') for t in (W0, b0, W1, b1, W2, b2, mean)]
    if B == 0:
        return out
    with torch.cuda.device(feats.device):
        nbytes = lib().shapy_head_workspace_bytes(B, Fd, P, h0, h1)
        ws = _WS.get('head', nbytes, feats.device)
        check(lib().shapy_head_forward(ptr(feats), B, Fd, P, h0, h1, *[ptr(t) for t in ts], num_stages, ptr(out),
                                       ptr(ws), ws.numel(), stream_ptr()), 'head_forward')
    return out


def collapse_head(W0, b0, W1, b1, W2, b2, feat_dim):
    """Contracts the activation-free 3-layer MLP into (MfT, MpT, c) in fp64 (host, once per weight load)."""
    d = lambda t: t.detach().double().cpu()  # noqa: E731
    W0, b0, W1, b1, W2, b2 = map(d, (W0, b0, W1, b1, W2, b2))
    W21 = W2 @ W1
    Mf = W21 @ W0[:, :feat_dim]
    Mp = W21 @ W0[:, feat_dim:]
    c = W2 @ (W1 @ b0 + b1) + b2
    return Mf.t().contiguous().float(), Mp.t().contiguous().float(), c.float()


def head_forward_collapsed(feats, MfT, Mp, c, mean, num_stages=3):
    feats = _cuda_f32(feats, 'features')
    B, Fd = feats.shape
    P = mean.numel()
    out = torch.empty(num_stages, B, P, dtype=torch.float32, device=feats.device)
    ts = [_cuda_f32(t, 'head matrix') for t in (MfT, Mp, c, mean)]
    if B == 0:
        return out
    with torch.cuda.device(feats.device):
        ws = _WS.get('headc', B * P * 4, feats.device)
        check(lib().shapy_head_forward_collapsed(ptr(feats), B, Fd, P, *[ptr(t) for t in ts], num_stages, ptr(out),
                                                 ptr(ws), ws.numel(), stream_ptr()), 'head_forward_collapsed')
    return out


# ------------------------------------------------------------------------------------------- HRNet
class HrnetPlan:
    """Owns a shapy_hrnet_t built from a conv table + op program (see human_shape/models/backbone/hrnet.py)."""

    def __init__(self, convs, ops, slots, feat_slot, feat_dim, mode, engine, device):
        self.device = torch.device(device)
        self._keep = []
        cd = (_lib.ConvDesc * len(convs))()
        for i, c in enumerate(convs):
            def hp(t):
                if t is None:
                    return None
                a = np.ascontiguousarray(t.detach().float().cpu().numpy())
                self._keep.append(a)
                return a.ctypes.data
            cd[i].cin, cd[i].cout, cd[i].ksize, cd[i].stride = c['cin'], c['cout'], c['ksize'], c['stride']
            cd[i].weight, cd[i].bias = hp(c['weight']), hp(c.get('bias'))
            bn = c.get('bn')
            if bn is not None:
                cd[i].bn_weight, cd[i].bn_bias = hp(bn['weight']), hp(bn['bias'])
                cd[i].bn_mean, cd[i].bn_var = hp(bn['mean']), hp(bn['var'])
                cd[i].bn_eps = float(bn['eps'])
        od = (_lib.Op * len(ops))()
        for i, o in enumerate(ops):
            od[i].kind, od[i].conv = o['kind'], o.get('conv', -1)
            od[i].in_slot, od[i].out_slot, od[i].out_coff = o.get('in_slot', -1), o.get('out_slot', -1), o.get('out_coff', 0)
            od[i].res_slot, od[i].relu = o.get('res_slot', -1), int(o.get('relu', 0))
            od[i].lane = int(o.get('lane', 0))
            ins = o.get('fuse_in', [])
            od[i].n_in = len(ins)
            for k, (s, sh) in enumerate(zip(ins, o.get('fuse_shift', []))):
                od[i].fuse_in[k], od[i].fuse_shift[k] = s, sh
        sd = (_lib.Slot * len(slots))()
        for i, s in enumerate(slots):
            sd[i].channels, sd[i].div = s['channels'], s['div']
        self.slots, self.feat_dim, self.mode, self.engine = slots, feat_dim, mode, engine
        handle = C.c_void_p()
        with torch.cuda.device(self.device):
            check(lib().shapy_hrnet_create(C.byref(handle), cd, len(convs), od, len(ops), sd, len(slots), feat_slot,
                                           mode, engine), 'hrnet_create')
        self._keep = []
        self.handle = handle
        self._fin = weakref.finalize(self, lib().shapy_hrnet_destroy, handle)
        self._ws = None
        self._shape = None

    def forward(self, images: torch.Tensor) -> torch.Tensor:
        images = _cuda_f32(images, 'images')
        B, Cc, H, W = images.shape
        if Cc != 3:
            raise RuntimeError('images must be (B, 3, H, W)')
        feats = torch.empty(B, self.feat_dim, dtype=torch.float32, device=images.device)
        if H % 32 or W % 32 or H == 0 or W == 0:
            raise RuntimeError(f'image size {H}x{W} must be a multiple of 32')
        if B == 0:
            return feats
        with torch.cuda.device(images.device):
            nbytes = lib().shapy_hrnet_workspace_bytes(self.handle, B, H, W)
            if nbytes == 0:
                raise RuntimeError(f'image size {H}x{W} must be a multiple of 32')
            if self._ws is None or self._ws.numel() < nbytes or self._shape != (B, H, W):
                self._ws = torch.empty(nbytes, dtype=torch.uint8, device=images.device)
                self._shape = (B, H, W)
            check(lib().shapy_hrnet_forward(self.handle, ptr(images), B, H, W, ptr(feats), ptr(self._ws),
                                            self._ws.numel(), stream_ptr()), 'hrnet_forward')
        return feats

    def read_slot(self, slot: int) -> torch.Tensor:
        B, H, W = self._shape
        s = self.slots[slot]
        out = torch.empty(B, s['channels'], H // s['div'], W // s['div'], dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            check(lib().shapy_hrnet_read_slot(self.handle, slot, ptr(out), stream_ptr()), 'hrnet_read_slot')
        return out

    def flops(self, B, H, W) -> float:
        return lib().shapy_hrnet_flops(self.handle, B, H, W)


class ConvPlan(collections.namedtuple('ConvPlan', 'path schedule nt')):
    """A wgmma plan in conv_test's engine digits: path 2 per-tap, 3 halo, 4 weight-resident; schedule 1 cooperative,
    2 ping-pong; nt the cout tile."""
    @property
    def engine(self):
        """the conv_test engine number that forces this plan"""
        return self.path + 10 * self.schedule + 100 * self.nt


def conv_test(x_nhwc, weight, bias=None, bn=None, stride=1, res_nhwc=None, relu=False, mode=1, engine=0,
              in_view=None, out_view=None, report=False):
    """Single convolution through either engine on fp32 NHWC tensors (unit tests).  engine: 0 = wgmma with the path
    the network would take, 1 = SIMT, 2 = wgmma per-tap path, 3 = wgmma halo-resident path, 4 = wgmma halo path with
    the weights resident in shared memory; + 10 forces the
    cooperative consumer schedule of the wgmma engine, + 20 the ping-pong one; + 100 * NT forces its cout tile NT.
    in_view=(ctot, coff): x has ctot channels and the convolution reads coff .. coff + cin of them.
    out_view=(ctot, coff): the convolution writes channels coff .. coff + cout of (B + 1, Ho, Wo, ctot) planes filled
    with NaN beforehand, and all of them are returned, the guard image B included.
    report=True: returns (y, ConvPlan(path, schedule, nt)), the plan built in the engine digits above (-1 for SIMT)."""
    x = _cuda_f32(x_nhwc, 'x')
    B, H, W, Cx = x.shape
    Cout, Cin, k, _ = weight.shape
    if Cx != (in_view[0] if in_view else Cin):
        raise RuntimeError(f'x has {Cx} channels: expected {in_view[0] if in_view else Cin}')
    keep = []

    def hp(t):
        if t is None:
            return None
        a = np.ascontiguousarray(t.detach().float().cpu().numpy())
        keep.append(a)
        return a.ctypes.data
    d = _lib.ConvDesc()
    d.cin, d.cout, d.ksize, d.stride = Cin, Cout, k, stride
    d.weight, d.bias = hp(weight), hp(bias)
    if bn is not None:
        d.bn_weight, d.bn_bias, d.bn_mean, d.bn_var = hp(bn['weight']), hp(bn['bias']), hp(bn['mean']), hp(bn['var'])
        d.bn_eps = float(bn['eps'])
    Ho, Wo = (H // 2, W // 2) if stride == 2 else (H, W)
    y = torch.empty((B + 1, Ho, Wo, out_view[0]) if out_view else (B, Ho, Wo, Cout), dtype=torch.float32,
                    device=x.device)
    res = None if res_nhwc is None else _cuda_f32(res_nhwc, 'res')
    plan = (C.c_int * 3)()
    with torch.cuda.device(x.device):
        check(lib().shapy_conv_test(C.byref(d), ptr(x), ptr(res), B, H, W, int(relu), mode, engine,
                                    *(in_view or (0, 0)), *(out_view or (0, 0)), plan, ptr(y), stream_ptr()),
              'conv_test')
    return (y, ConvPlan(*plan)) if report else y


def fit_lm_groups_workspace(B, G, n_rot, nb, device):
    """The scratch of the grouped 2D step (include/shapy_b200.h, shapy_fit_lm_groups_workspace_bytes): a uint8 CUDA
    tensor, allocated once before an LM loop."""
    return _workspace(lib().shapy_fit_lm_groups_workspace_bytes(int(B), int(G), int(n_rot), int(nb)), device)


def _check_group_state(what, state, trial, G, B, nb):
    """The per-group state of the grouped and sequence 2D steps: betas, trial betas, loss, lambda and accepted per
    group (G rows), and image_betas per image (B rows)."""
    if (state['betas'].shape != (G, nb) or trial['betas'].shape != (G, nb) or trial['image_betas'].shape != (B, nb) or
            any(state[k].shape != (G,) for k in ('loss', 'lambda', 'accepted'))):
        raise RuntimeError(f'{what}: betas and trial betas must be ({G}, {nb}), image_betas ({B}, {nb}) and loss, '
                           f'lambda and accepted ({G},)')


def _fit_lm_kp2d_groups(what, state, trial, targets, weights, robust_sigma, pose_prior_weight, betas_weight, lambda_up,
                        lambda_down, first, trial_keypoints, trial_jac, group_offsets, workspace, pose_anchor,
                        meas=None, share_pose=False):
    """What the four grouped 2D steps share: the checks and the call, `meas` None or (meas_targets, meas_weights,
    trial_meas, trial_meas_jac), all (G, ...); share_pose: the shared-pose steps, with a per-group pose_anchor."""
    B, n_rot = trial['rot'].shape[:2]
    nb, K = trial['betas'].shape[1], targets.shape[1]
    sigma = _check_kp2d_scalars(what, robust_sigma, pose_prior_weight, betas_weight, lambda_up, lambda_down,
                                pose_anchor)
    G = _check_offsets(what, 'group_offsets', group_offsets, B)
    anchor = [] if pose_anchor is None else [pose_anchor]
    mstate = [] if meas is None else [state['meas'], state['meas_jac']]
    ts = [state[k] for k in ('rot', 'betas', 'camera', 'keypoints', 'jac', 'loss', 'lambda')] + mstate + \
        [trial[k] for k in ('rot', 'betas', 'image_betas', 'camera')] + [targets, weights, trial_keypoints,
                                                                         trial_jac] + anchor + list(meas or ())
    _check_step_tensors(what, ts, 'the state, trial, targets, weights and anchor', state['accepted'])
    P = 3 * n_rot + nb + 3
    if not _kp_step_shapes_ok(state, trial_jac, weights, B, K, P) or targets.shape != (B, K, 2):
        raise RuntimeError(f'{what}: jac must be ({B}, {3 * K}, {P}), weights ({B}, {K}) and targets ({B}, {K}, 2)')
    na = G if share_pose else B
    if pose_anchor is not None and pose_anchor.shape != (na, n_rot, 3, 3):
        raise RuntimeError(f'{what}: pose_anchor must be ({na}, {n_rot}, 3, 3)')
    _check_group_state(what, state, trial, G, B, nb)
    if meas is not None and not _meas_step_shapes_ok(state, meas[2], meas[3], meas[0], meas[1], G, nb):
        raise RuntimeError(f'{what}: meas_jac must be ({G}, 5, {nb}) and the measurements, their targets and weights '
                           f'({G}, 5)')
    L = lib()
    _check_workspace(what, workspace, (L.shapy_fit_lm_shared_pose_workspace_bytes if share_pose else
                                       L.shapy_fit_lm_groups_workspace_bytes)(B, G, n_rot, nb))
    if B == 0:
        return
    head = [B, G, group_offsets.data_ptr(), K, n_rot, nb, ptr(targets), ptr(weights), ptr(pose_anchor), sigma,
            float(pose_prior_weight), float(betas_weight)]
    lam = [float(lambda_up), float(lambda_down), int(bool(first))]
    tr = [ptr(trial['rot']), ptr(trial['betas']), ptr(trial['image_betas']), ptr(trial['camera']),
          ptr(trial_keypoints), ptr(trial_jac)]
    with torch.cuda.device(trial['rot'].device):
        if meas is None:
            step = L.shapy_fit_lm_keypoints_2d_shared_pose_step if share_pose else \
                L.shapy_fit_lm_keypoints_2d_groups_step
            check(step(
                *head, *lam,
                *[ptr(state[k]) for k in ('rot', 'betas', 'camera', 'keypoints', 'jac', 'loss', 'lambda', 'accepted')],
                *tr, ptr(workspace), stream_ptr()), what)
        else:
            step = L.shapy_fit_lm_keypoints_2d_shared_pose_measurements_step if share_pose else \
                L.shapy_fit_lm_keypoints_2d_groups_measurements_step
            check(step(
                *head, ptr(meas[0]), ptr(meas[1]), *lam,
                *[ptr(state[k]) for k in ('rot', 'betas', 'camera', 'keypoints', 'jac', 'meas', 'meas_jac', 'loss',
                                          'lambda', 'accepted')],
                *tr, ptr(meas[2]), ptr(meas[3]), ptr(workspace), stream_ptr()), what)


def fit_lm_keypoints_2d_groups_step(state, trial, targets, weights, robust_sigma, pose_prior_weight, betas_weight,
                                    lambda_up, lambda_down, first, trial_keypoints, trial_jac, group_offsets,
                                    workspace, pose_anchor=None):
    """One Levenberg-Marquardt step of the 2D fit over groups of images sharing their betas (include/shapy_b200.h,
    shapy_fit_lm_keypoints_2d_groups_step), in place.  group_offsets: (G + 1,) int32 CPU tensor, group g the images
    [off[g], off[g + 1]).  state: fit_lm_keypoints_2d_step's, with 'betas' (G, NB), 'loss', 'lambda', 'accepted' (G,);
    trial: {'rot' (B, n_rot, 3, 3), 'betas' (G, NB), 'image_betas' (B, NB) (each image's group betas, what
    smplx_keypoint_jacobian evaluated), 'camera' (B, 3)}, the evaluated trial on entry and the next on return;
    workspace from fit_lm_groups_workspace.  Three launches, no host synchronisation."""
    _fit_lm_kp2d_groups('fit_lm_keypoints_2d_groups_step', state, trial, targets, weights, robust_sigma,
                        pose_prior_weight, betas_weight, lambda_up, lambda_down, first, trial_keypoints, trial_jac,
                        group_offsets, workspace, pose_anchor)


def fit_lm_keypoints_2d_groups_measurements_step(state, trial, targets, weights, robust_sigma, pose_prior_weight,
                                                 betas_weight, meas_targets, meas_weights, lambda_up, lambda_down,
                                                 first, trial_keypoints, trial_jac, trial_meas, trial_meas_jac,
                                                 group_offsets, workspace, pose_anchor=None):
    """fit_lm_keypoints_2d_groups_step with the five measurements of each group (include/shapy_b200.h,
    shapy_fit_lm_keypoints_2d_groups_measurements_step), in place.  state adds 'meas' (G, 5) and 'meas_jac'
    (G, 5, NB); meas_targets, meas_weights (G, 5); trial_meas (G, 5) / trial_meas_jac (G, 5, NB) from
    measure_jacobian_betas at the G trial betas."""
    _fit_lm_kp2d_groups('fit_lm_keypoints_2d_groups_measurements_step', state, trial, targets, weights, robust_sigma,
                        pose_prior_weight, betas_weight, lambda_up, lambda_down, first, trial_keypoints, trial_jac,
                        group_offsets, workspace, pose_anchor, (meas_targets, meas_weights, trial_meas, trial_meas_jac))


def fit_lm_shared_pose_workspace(B, G, n_rot, nb, device):
    """The scratch of the shared-pose 2D step (include/shapy_b200.h, shapy_fit_lm_shared_pose_workspace_bytes): a uint8
    CUDA tensor, allocated once before an LM loop."""
    return _workspace(lib().shapy_fit_lm_shared_pose_workspace_bytes(int(B), int(G), int(n_rot), int(nb)), device)


def fit_lm_keypoints_2d_shared_pose_step(state, trial, targets, weights, robust_sigma, pose_prior_weight, betas_weight,
                                         lambda_up, lambda_down, first, trial_keypoints, trial_jac, group_offsets,
                                         workspace, pose_anchor=None):
    """fit_lm_keypoints_2d_groups_step for simultaneous views of one posed body (include/shapy_b200.h,
    shapy_fit_lm_keypoints_2d_shared_pose_step), in place: the images of a group also share the body rotations of
    joints 1 .., each keeps its global rotation and camera.  state and trial as fit_lm_keypoints_2d_groups_step's;
    'rot' stays per image, and every image of a group holds the group's body rotations in rows 1 .. (the step reads
    the first image's and writes all).  pose_anchor (G, n_rot, 3, 3), joint 0 unread; the pose prior counts once per
    group.  workspace from fit_lm_shared_pose_workspace.  Three launches, no host synchronisation."""
    _fit_lm_kp2d_groups('fit_lm_keypoints_2d_shared_pose_step', state, trial, targets, weights, robust_sigma,
                        pose_prior_weight, betas_weight, lambda_up, lambda_down, first, trial_keypoints, trial_jac,
                        group_offsets, workspace, pose_anchor, share_pose=True)


def fit_lm_keypoints_2d_shared_pose_measurements_step(state, trial, targets, weights, robust_sigma, pose_prior_weight,
                                                      betas_weight, meas_targets, meas_weights, lambda_up,
                                                      lambda_down, first, trial_keypoints, trial_jac, trial_meas,
                                                      trial_meas_jac, group_offsets, workspace, pose_anchor=None):
    """fit_lm_keypoints_2d_shared_pose_step with the five measurements of each group (include/shapy_b200.h,
    shapy_fit_lm_keypoints_2d_shared_pose_measurements_step), in place; the measurement arguments as
    fit_lm_keypoints_2d_groups_measurements_step's."""
    _fit_lm_kp2d_groups('fit_lm_keypoints_2d_shared_pose_measurements_step', state, trial, targets, weights,
                        robust_sigma, pose_prior_weight, betas_weight, lambda_up, lambda_down, first, trial_keypoints,
                        trial_jac, group_offsets, workspace, pose_anchor,
                        (meas_targets, meas_weights, trial_meas, trial_meas_jac), share_pose=True)


def fit_lm_sequence_workspace(B, S, n_rot, nb, device):
    """The scratch of the sequence 2D step (include/shapy_b200.h, shapy_fit_lm_sequence_workspace_bytes): a uint8 CUDA
    tensor, allocated once before an LM loop."""
    return _workspace(lib().shapy_fit_lm_sequence_workspace_bytes(int(B), int(S), int(n_rot), int(nb)), device)


def fit_lm_keypoints_2d_sequence_step(state, trial, targets, weights, intrinsics, robust_sigma, pose_prior_weight,
                                      betas_weight, smooth_rot_weight, smooth_transl_weight, lambda_up, lambda_down,
                                      first, trial_keypoints, trial_jac, sequence_offsets, workspace, pose_anchor=None):
    """One Levenberg-Marquardt step of the perspective 2D fit over video sequences (include/shapy_b200.h,
    shapy_fit_lm_keypoints_2d_sequence_step), in place.  sequence_offsets: (S + 1,) int32 CPU tensor, sequence s the
    frames [off[s], off[s + 1]) in time order.  Per frame (B rows): targets (B, K, 2), weights (B, K), intrinsics (B, 3)
    = (f, px, py), pose_anchor (B, n_rot, 3, 3), state 'rot', 'transl', 'keypoints', 'jac' and trial 'rot', 'transl',
    'image_betas' (each frame's sequence betas, what smplx_keypoint_jacobian evaluated).  Per sequence (S rows): state
    'betas', 'loss', 'lambda', 'accepted' and trial 'betas'.  smooth_rot_weight / 2 |R_{t+1} - R_t|_F^2 over every
    rotation and smooth_transl_weight |t_{t+1} - t_t|^2 tie consecutive frames.  workspace from
    fit_lm_sequence_workspace.  Three launches, no host synchronisation."""
    what = 'fit_lm_keypoints_2d_sequence_step'
    B, n_rot = trial['rot'].shape[:2]
    nb, K = trial['betas'].shape[1], targets.shape[1]
    sigma = _check_kp2d_scalars(what, robust_sigma, pose_prior_weight, betas_weight, lambda_up, lambda_down,
                                pose_anchor)
    srw, stw = float(smooth_rot_weight), float(smooth_transl_weight)
    if not (0 <= srw < float('inf') and 0 <= stw < float('inf')):
        raise ValueError(f'{what}: the smoothness weights must be finite and >= 0')
    S = _check_offsets(what, 'sequence_offsets', sequence_offsets, B)
    anchor = [] if pose_anchor is None else [pose_anchor]
    ts = [state[k] for k in ('rot', 'betas', 'transl', 'keypoints', 'jac', 'loss', 'lambda')] + \
        [trial[k] for k in ('rot', 'betas', 'image_betas', 'transl')] + [targets, weights, intrinsics, trial_keypoints,
                                                                         trial_jac] + anchor
    _check_step_tensors(what, ts, 'the state, trial, targets, weights, intrinsics and anchor', state['accepted'])
    P = 3 * n_rot + nb + 3
    if not _kp_step_shapes_ok(state, trial_jac, weights, B, K, P) or targets.shape != (B, K, 2):
        raise RuntimeError(f'{what}: jac must be ({B}, {3 * K}, {P}), weights ({B}, {K}) and targets ({B}, {K}, 2)')
    if intrinsics.shape != (B, 3) or state['transl'].shape != (B, 3) or trial['transl'].shape != (B, 3):
        raise RuntimeError(f'{what}: intrinsics and transl must be ({B}, 3)')
    if pose_anchor is not None and pose_anchor.shape != (B, n_rot, 3, 3):
        raise RuntimeError(f'{what}: pose_anchor must be ({B}, {n_rot}, 3, 3)')
    _check_group_state(what, state, trial, S, B, nb)
    L = lib()
    _check_workspace(what, workspace, L.shapy_fit_lm_sequence_workspace_bytes(B, S, n_rot, nb))
    if B == 0:
        return
    with torch.cuda.device(trial['rot'].device):
        check(L.shapy_fit_lm_keypoints_2d_sequence_step(
            B, S, sequence_offsets.data_ptr(), K, n_rot, nb, ptr(targets), ptr(weights), ptr(intrinsics), ptr(pose_anchor), sigma,
            float(pose_prior_weight), float(betas_weight), srw, stw, float(lambda_up), float(lambda_down),
            int(bool(first)),
            *[ptr(state[k]) for k in ('rot', 'betas', 'transl', 'keypoints', 'jac', 'loss', 'lambda', 'accepted')],
            ptr(trial['rot']), ptr(trial['betas']), ptr(trial['image_betas']), ptr(trial['transl']),
            ptr(trial_keypoints), ptr(trial_jac), ptr(workspace), stream_ptr()), what)


def fit_lm_calibrated_workspace(B, G, device):
    """The scratch of the calibrated 2D step (include/shapy_b200.h, shapy_fit_lm_calibrated_workspace_bytes): a uint8
    CUDA tensor, allocated once before an LM loop."""
    return _workspace(lib().shapy_fit_lm_calibrated_workspace_bytes(int(B), int(G)), device)


def _fit_lm_kp2d_calibrated(what, state, trial, targets, weights, intrinsics, extrinsics, robust_sigma,
                            pose_prior_weight, betas_weight, lambda_up, lambda_down, first, trial_keypoints, trial_jac,
                            view_offsets, workspace, pose_anchor, meas=None):
    """What the two calibrated 2D steps share: the checks and the call, `meas` None or (meas_targets, meas_weights,
    trial_meas, trial_meas_jac), all (G, ...)."""
    G, n_rot = trial['rot'].shape[:2]
    nb, B, K = trial['betas'].shape[1], targets.shape[0], targets.shape[1]
    sigma = _check_kp2d_scalars(what, robust_sigma, pose_prior_weight, betas_weight, lambda_up, lambda_down,
                                pose_anchor)
    _check_offsets(what, 'view_offsets', view_offsets, B, G)
    anchor = [] if pose_anchor is None else [pose_anchor]
    mstate = [] if meas is None else [state['meas'], state['meas_jac']]
    ts = [state[k] for k in ('rot', 'betas', 'transl', 'keypoints', 'jac', 'loss', 'lambda')] + mstate + \
        [trial[k] for k in ('rot', 'betas', 'transl')] + [targets, weights, intrinsics, extrinsics, trial_keypoints,
                                                          trial_jac] + anchor + list(meas or ())
    _check_step_tensors(what, ts, 'the state, trial, targets, weights, cameras and anchor', state['accepted'])
    P = 3 * n_rot + nb + 3
    if trial_jac.shape != (G, 3 * K, P) or state['jac'].shape != (G, 3 * K, P) or \
            any(state[k].shape != (G,) for k in ('loss', 'lambda', 'accepted')):
        raise RuntimeError(f'{what}: per body, jac must be ({G}, {3 * K}, {P}) and loss, lambda and accepted ({G},)')
    if targets.shape != (B, K, 2) or weights.shape != (B, K) or intrinsics.shape != (B, 3) or \
            extrinsics.shape != (B, 12):
        raise RuntimeError(f'{what}: per view, targets must be ({B}, {K}, 2), weights ({B}, {K}), intrinsics ({B}, 3) '
                           f'and extrinsics ({B}, 12)')
    if pose_anchor is not None and pose_anchor.shape != (G, n_rot, 3, 3):
        raise RuntimeError(f'{what}: pose_anchor must be ({G}, {n_rot}, 3, 3)')
    if meas is not None and not _meas_step_shapes_ok(state, meas[2], meas[3], meas[0], meas[1], G, nb):
        raise RuntimeError(f'{what}: meas_jac must be ({G}, 5, {nb}) and the measurements, their targets and weights '
                           f'({G}, 5)')
    L = lib()
    _check_workspace(what, workspace, L.shapy_fit_lm_calibrated_workspace_bytes(B, G))
    if G == 0:
        return
    head = [B, G, view_offsets.data_ptr(), K, n_rot, nb, ptr(targets), ptr(weights), ptr(intrinsics), ptr(extrinsics),
            ptr(pose_anchor), sigma, float(pose_prior_weight), float(betas_weight)]
    lam = [float(lambda_up), float(lambda_down), int(bool(first))]
    tr = [ptr(trial['rot']), ptr(trial['betas']), ptr(trial['transl']), ptr(trial_keypoints), ptr(trial_jac)]
    with torch.cuda.device(trial['rot'].device):
        if meas is None:
            check(L.shapy_fit_lm_keypoints_2d_calibrated_step(
                *head, *lam,
                *[ptr(state[k]) for k in ('rot', 'betas', 'transl', 'keypoints', 'jac', 'loss', 'lambda', 'accepted')],
                *tr, ptr(workspace), stream_ptr()), what)
        else:
            check(L.shapy_fit_lm_keypoints_2d_calibrated_measurements_step(
                *head, ptr(meas[0]), ptr(meas[1]), *lam,
                *[ptr(state[k]) for k in ('rot', 'betas', 'transl', 'keypoints', 'jac', 'meas', 'meas_jac', 'loss',
                                          'lambda', 'accepted')],
                *tr, ptr(meas[2]), ptr(meas[3]), ptr(workspace), stream_ptr()), what)


def fit_lm_keypoints_2d_calibrated_step(state, trial, targets, weights, intrinsics, extrinsics, robust_sigma,
                                        pose_prior_weight, betas_weight, lambda_up, lambda_down, first,
                                        trial_keypoints, trial_jac, view_offsets, workspace, pose_anchor=None):
    """One Levenberg-Marquardt step per body of the fit to the 2D keypoints of a calibrated rig (include/shapy_b200.h,
    shapy_fit_lm_keypoints_2d_calibrated_step), in place.  view_offsets: (G + 1,) int32 CPU tensor, body g seen by the
    views [off[g], off[g + 1]).  Per view (B rows): targets (B, K, 2), weights (B, K), intrinsics (B, 3) = (f, px, py)
    and extrinsics (B, 12) = world-to-camera R (row-major) then T.  Per body (G rows): state {'rot' (G, n_rot, 3, 3),
    'betas', 'transl' (the world translation), 'keypoints', 'jac', 'loss', 'lambda', 'accepted'}, trial {'rot',
    'betas', 'transl'} (the evaluated trial on entry and the next on return), trial_keypoints / trial_jac from
    smplx_keypoint_jacobian without transl and pose_anchor (G, n_rot, 3, 3).  workspace from
    fit_lm_calibrated_workspace.  One launch, no host synchronisation."""
    _fit_lm_kp2d_calibrated('fit_lm_keypoints_2d_calibrated_step', state, trial, targets, weights, intrinsics,
                            extrinsics, robust_sigma, pose_prior_weight, betas_weight, lambda_up, lambda_down, first,
                            trial_keypoints, trial_jac, view_offsets, workspace, pose_anchor)


def fit_lm_keypoints_2d_calibrated_measurements_step(state, trial, targets, weights, intrinsics, extrinsics,
                                                     robust_sigma, pose_prior_weight, betas_weight, meas_targets,
                                                     meas_weights, lambda_up, lambda_down, first, trial_keypoints,
                                                     trial_jac, trial_meas, trial_meas_jac, view_offsets, workspace,
                                                     pose_anchor=None):
    """fit_lm_keypoints_2d_calibrated_step with the five measurements of each body (include/shapy_b200.h,
    shapy_fit_lm_keypoints_2d_calibrated_measurements_step), in place: state adds 'meas' (G, 5) and 'meas_jac'
    (G, 5, NB); meas_targets, meas_weights, trial_meas (G, 5) and trial_meas_jac (G, 5, NB) as
    fit_lm_keypoints_2d_measurements_step's."""
    _fit_lm_kp2d_calibrated('fit_lm_keypoints_2d_calibrated_measurements_step', state, trial, targets, weights,
                            intrinsics, extrinsics, robust_sigma, pose_prior_weight, betas_weight, lambda_up,
                            lambda_down, first, trial_keypoints, trial_jac, view_offsets, workspace, pose_anchor,
                            (meas_targets, meas_weights, trial_meas, trial_meas_jac))
