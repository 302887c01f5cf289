"""DistanceFieldPenetrationLoss, mirror of mesh-mesh-intersection/mesh_mesh_intersection/loss.py:201-317, on the
penetration kernels of include/shapy_b200.h (shapy_penetration_forward / _backward).

The triangles (B, F, 3, 3) are read as the vertices (B, 3F, 3) of the faces arange(3F).view(F, 3), so the loss runs on
the same kernels as the fits' self-penetration term.  The semantics are those of the reference's default
vectorized=True path; point2plane only changes the reference's rounding (the axis is a unit vector) and is accepted
for its signature.  float32 CUDA triangles only.
"""
import torch
import torch.nn as nn

from . import autograd as _ag

_FACES = {}


def _soup_faces(F, device):
    key = (F, device)
    f = _FACES.get(key)
    if f is None:
        f = _FACES[key] = torch.arange(3 * F, dtype=torch.int32, device=device).view(F, 3)
    return f


class DistanceFieldPenetrationLoss(nn.Module):
    def __init__(self, sigma=0.5, point2plane=False, vectorized=True, penalize_outside=True, linear_max=1000):
        super().__init__()
        self.sigma = sigma
        self.point2plane = point2plane
        self.vectorized = vectorized
        self.penalize_outside = penalize_outside
        self.linear_max = linear_max

    def forward(self, triangles, collision_idxs):
        """triangles (B, F, 3, 3) float32 CUDA, collision_idxs (B, C, 2) (receiver, intruder) face indices, rows whose
        first index is < 0 skipped.  Returns the loss (B,), differentiable with respect to the triangles."""
        if not self.vectorized:
            raise NotImplementedError('vectorized=False is not a working mode of the reference loss (its forward '
                                      'raises IndexError); only the vectorized path is mirrored')
        if not (torch.is_tensor(triangles) and triangles.dtype == torch.float32):
            raise TypeError(f'triangles must be a float32 tensor, got {getattr(triangles, "dtype", type(triangles))}')
        if triangles.dim() != 4 or triangles.shape[2:] != (3, 3):
            raise ValueError(f'triangles must be (B, F, 3, 3), got {tuple(triangles.shape)}')
        B, F = triangles.shape[:2]
        pairs = collision_idxs.to(device=triangles.device, dtype=torch.int32).contiguous()
        vertices = triangles.reshape(B, 3 * F, 3)
        return _ag.PenetrationFunction.apply(vertices, _soup_faces(F, triangles.device), pairs, float(self.sigma),
                                             bool(self.penalize_outside), float(self.linear_max))
