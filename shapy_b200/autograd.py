"""Autograd for the SMPL-X forward, the 6D decoder, the T-pose shape blend and the virtual measurements (first order
only).

    measure(landmarks, v_shaped=, faces_i32=)   (B,V,3) vertices + (F,3) int32 faces -> (B,5)
    measure(landmarks, triangles=)              (B,F,3,3) triangles -> (B,5)
    ShapeFunction.apply(packed_model, betas)    betas (B,NB) -> v_shaped (B,V,3)
    SmplxFunction.apply(packed_model, betas, rot, expression, camera, want_v_shaped)
                                                -> vertices, v_shaped, joints, proj_joints (None where not computed)
    Rot6dFunction.apply(raw)                    raw (B,6n) -> (B,n,3,3)
    ClosestPointsFunction.apply(faces_i32, vertices, points, weights)
                                                scan points (B,N,3) on posed meshes (B,V,3) -> sq_dist (B,N)
    PenetrationFunction.apply(vertices, faces_i32, pairs, sigma, penalize_outside, linear_max)
                                                self-penetration loss at fixed face pairs (B,C,2) -> (B,)
    SilhouetteFunction.apply(vertices, intrinsics, faces_i32, dist, contour, contour_w, inv_count, tree)
                                                the silhouette term of perspective posed meshes against masks -> (B,)

The forward of each is the same launches as the no-grad path; the backward is the matching CUDA adjoint
(measure_smem_kernel in gradient mode, the shape-blend adjoint, shapy_smplx_backward which recomputes the posed
forward, or the decoder's elementwise adjoint).  SmplxFunction's semantics are those of the reference's lbs() and
SMPLX.forward under autograd: see include/shapy_b200.h and DESIGN.md §6b.  For the measurements they are the
reference's autograd ones (mesh-mesh-intersection/body_measurements/body_measurements.py:137-215): the intersection points' barycentrics are
constants and the slicing planes' heights get no gradient, so a circumference's gradient is the derivative of the
perimeter with the hull's points sliding on fixed faces at fixed barycentrics, not the finite difference of the mesh.
measure(..., exact=True) backpropagates the exact derivative of the circumferences instead (ops.measure_backward
with exact=True; the forward is the same launch).
Every function is `once_differentiable`: a double backward (`create_graph=True`, e.g. the TrustRegion optimiser of
the reference's examples/fit_measurements.py) raises.
"""
import torch
from torch.autograd.function import once_differentiable

from . import ops as _ops


class MeasureFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, landmarks, x, faces_i32, status, exact):
        if faces_i32 is None:
            out = _ops.measure(landmarks, triangles=x)
        else:
            out = _ops.measure(landmarks, v_shaped=x, faces_i32=faces_i32)
        ctx.landmarks = landmarks
        ctx.exact = exact
        ctx.save_for_backward(x, faces_i32)
        status.append(out.status)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        x, faces_i32 = ctx.saved_tensors
        grad_out = grad_out.contiguous()
        if faces_i32 is None:
            g = _ops.measure_backward(ctx.landmarks, grad_out, triangles=x, exact=ctx.exact)
        else:
            g = _ops.measure_backward(ctx.landmarks, grad_out, v_shaped=x, faces_i32=faces_i32, exact=ctx.exact)
        return None, g, None, None, None


class ShapeFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, packed, betas):
        ctx.packed = packed
        return _ops.smplx_forward_shape(packed, betas)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_v):
        return None, _ops.smplx_backward_shape(ctx.packed, grad_v.contiguous())


class SmplxFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, packed, betas, rot, expression, camera, want_v_shaped):
        out = _ops.smplx_forward(packed, betas, rot, expr=expression, camera=camera, want_vertices=True,
                                 want_v_shaped=want_v_shaped, want_joints=True)
        ctx.packed = packed
        ctx.save_for_backward(betas, rot, expression, camera)
        ctx.set_materialize_grads(False)      # an unused output passes None, read as a zero cotangent
        return out['vertices'], out['v_shaped'], out['joints'], out['proj_joints']

    @staticmethod
    @once_differentiable
    def backward(ctx, g_vertices, g_v_shaped, g_joints, g_proj):
        betas, rot, expression, camera = ctx.saved_tensors
        names = ('betas', 'rot', 'expr', 'camera')
        want = tuple(n for n, need in zip(names, ctx.needs_input_grad[1:5]) if need)
        c = lambda g: None if g is None else g.contiguous()  # noqa: E731
        r = _ops.smplx_backward(ctx.packed, betas, rot, expression, camera, grad_vertices=c(g_vertices),
                                grad_v_shaped=c(g_v_shaped), grad_joints=c(g_joints), grad_proj_joints=c(g_proj),
                                want=want)
        return (None,) + tuple(r[n] for n in names) + (None,)


class Rot6dFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, raw):
        ctx.save_for_backward(raw)
        return _ops.decode_rot6d(raw)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_rot):
        raw, = ctx.saved_tensors
        return _ops.decode_rot6d_backward(raw, grad_rot.contiguous()).view_as(raw)


class ClosestPointsFunction(torch.autograd.Function):
    """ClosestPointsFunction.apply(faces_i32, vertices, points, weights, tree=None) -> sq_dist (B, N): the squared
    distance of each scan point to its body's posed mesh (ops.closest_points), differentiable in the vertices only.
    The backward is ops.closest_points_backward: the closest face and barycentrics held at the forward's values, which
    at the exact closest point is the distance's derivative away from region switches.  tree: an ops.ScanTree the
    forward refits (same bits as a fresh build)."""

    @staticmethod
    def forward(ctx, faces_i32, vertices, points, weights, tree=None):
        face, bary, d2 = _ops.closest_points(vertices, faces_i32, points, weights, tree=tree)
        ctx.save_for_backward(faces_i32, vertices, points, face, bary)
        return d2

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_d2):
        faces_i32, vertices, points, face, bary = ctx.saved_tensors
        g = _ops.closest_points_backward(vertices, faces_i32, points, face, bary, grad_d2.contiguous())
        return None, g, None, None, None


class PenetrationFunction(torch.autograd.Function):
    """PenetrationFunction.apply(vertices, faces_i32, pairs, sigma, penalize_outside, linear_max) -> (B,): the
    distance-field penetration loss of each body at the (receiver, intruder) face rows pairs (B, C, 2)
    (ops.penetration_forward), differentiable in the vertices; the pairs are constants of the call."""

    @staticmethod
    def forward(ctx, vertices, faces_i32, pairs, sigma, penalize_outside, linear_max):
        ctx.args = (float(sigma), bool(penalize_outside), float(linear_max))
        ctx.save_for_backward(vertices, faces_i32, pairs)
        return _ops.penetration_forward(vertices, faces_i32, pairs, *ctx.args)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_loss):
        vertices, faces_i32, pairs = ctx.saved_tensors
        g = _ops.penetration_backward(vertices, faces_i32, pairs, grad_loss.contiguous(), *ctx.args)
        return g, None, None, None, None, None


class SilhouetteFunction(torch.autograd.Function):
    """SilhouetteFunction.apply(vertices, intrinsics, faces_i32, dist, contour, contour_w, inv_count, tree=None) -> (B,):
    the silhouette term of each body without its weight, (1/V) sum_v D(pi(v))^2 + inv_count sum_i d_i^2, from
    ops.silhouette_prepare's dist, contour and contour_w; inv_count (B,) is 1 / (kept contour pixels), 0 for none.  D
    is ops.silhouette_forward's; d_i the distance of contour pixel i to the projected mesh (u, v, 0), by
    ops.closest_points on `tree` (an ops.ScanTree, refit after the first call).  Differentiable in the vertices: the
    backward holds the closest face and barycentrics (ops.closest_points_backward on the projected mesh) and chains both
    halves through the projection in ops.silhouette_backward."""

    @staticmethod
    def forward(ctx, vertices, intrinsics, faces_i32, dist, contour, contour_w, inv_count, tree=None):
        proj, m2m = _ops.silhouette_forward(vertices, intrinsics, dist)
        face, bary, d2 = _ops.closest_points(proj, faces_i32, contour, contour_w, tree=tree)
        ctx.save_for_backward(vertices, intrinsics, faces_i32, dist, contour, inv_count, proj, face, bary)
        return m2m + (d2 * inv_count[:, None]).sum(1)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        vertices, intrinsics, faces_i32, dist, contour, inv_count, proj, face, bary = ctx.saved_tensors
        grad = grad.contiguous()
        g_d2 = (grad * inv_count)[:, None].expand(face.shape).contiguous()
        g_proj = _ops.closest_points_backward(proj, faces_i32, contour, face, bary, g_d2)
        g = _ops.silhouette_backward(vertices, intrinsics, dist, grad, g_proj)
        return g, None, None, None, None, None, None, None


def wants_grad(t) -> bool:
    """True when a differentiable launch is needed for `t` (grad mode on and `t` requires grad)."""
    return torch.is_grad_enabled() and torch.is_tensor(t) and t.requires_grad


def measure(landmarks, v_shaped=None, faces_i32=None, triangles=None, exact=False):
    """ops.measure, differentiable in v_shaped / triangles; `out.status` is the forward's device status word.
    exact: the backward gives the exact circumference derivative (ops.measure_backward)."""
    status = []
    if triangles is not None:
        out = MeasureFunction.apply(landmarks, triangles, None, status, bool(exact))
    else:
        out = MeasureFunction.apply(landmarks, v_shaped, faces_i32, status, bool(exact))
    out.status = status[0]
    return out
