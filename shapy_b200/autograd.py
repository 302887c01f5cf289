"""Autograd for the T-pose shape blend and the virtual measurements (first order only).

    measure(landmarks, v_shaped=, faces_i32=)   (B,V,3) vertices + (F,3) int32 faces -> (B,5)
    measure(landmarks, triangles=)              (B,F,3,3) triangles -> (B,5)
    ShapeFunction.apply(packed_model, betas)    betas (B,NB) -> v_shaped (B,V,3)

The forward of each is the same launch as the no-grad path; the backward is one CUDA launch (measure_smem_kernel in
gradient mode, or the shape-blend adjoint).  The semantics are the reference's autograd ones
(mesh-mesh-intersection/body_measurements/body_measurements.py:137-215): the intersection points' barycentrics are
constants and the slicing planes' heights get no gradient, so a circumference's gradient is the derivative of the
perimeter with the hull's points sliding on fixed faces at fixed barycentrics, not the finite difference of the mesh.
Both functions are `once_differentiable`: a double backward (`create_graph=True`, e.g. the TrustRegion optimiser of
the reference's examples/fit_measurements.py) raises.
"""
import torch
from torch.autograd.function import once_differentiable

from . import ops as _ops


class MeasureFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, landmarks, x, faces_i32, status):
        if faces_i32 is None:
            out = _ops.measure(landmarks, triangles=x)
        else:
            out = _ops.measure(landmarks, v_shaped=x, faces_i32=faces_i32)
        ctx.landmarks = landmarks
        ctx.save_for_backward(x, faces_i32)
        status.append(out.status)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        x, faces_i32 = ctx.saved_tensors
        grad_out = grad_out.contiguous()
        if faces_i32 is None:
            g = _ops.measure_backward(ctx.landmarks, grad_out, triangles=x)
        else:
            g = _ops.measure_backward(ctx.landmarks, grad_out, v_shaped=x, faces_i32=faces_i32)
        return None, g, None, None


class ShapeFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, packed, betas):
        ctx.packed = packed
        return _ops.smplx_forward_shape(packed, betas)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_v):
        return None, _ops.smplx_backward_shape(ctx.packed, grad_v.contiguous())


def wants_grad(t) -> bool:
    """True when a differentiable launch is needed for `t` (grad mode on and `t` requires grad)."""
    return torch.is_grad_enabled() and torch.is_tensor(t) and t.requires_grad


def measure(landmarks, v_shaped=None, faces_i32=None, triangles=None):
    """ops.measure, differentiable in v_shaped / triangles; `out.status` is the forward's device status word."""
    status = []
    if triangles is not None:
        out = MeasureFunction.apply(landmarks, triangles, None, status)
    else:
        out = MeasureFunction.apply(landmarks, v_shaped, faces_i32, status)
    out.status = status[0]
    return out
