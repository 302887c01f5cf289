"""Cameras, host mirror of regressor/human_shape/models/camera/camera_projection.py (build_cam_proj 44-89,
PerspectiveCamera 92-165, WeakPerspectiveCamera 168-213).  The weak-perspective projection of the 123 model joints is
fused into the SMPL-X joints kernel (csrc/smplx.cu: smplx_joints_kernel); this module carries the config and exposes
the same objects to callers.  PerspectiveCamera is the projection of the perspective keypoint fit
(shapy_b200.fit.fit_body_to_keypoints_2d with a focal length): the regressor itself has only the weak-perspective
head, and build_cam_proj rejects 'persp'."""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F


class CameraParams(object):
    attributes = ['translation', 'rotation', 'scale', 'focal_length']
    KEYS = ['translation', 'rotation', 'scale', 'focal_length']

    def __init__(self, translation=None, rotation=None, scale=None, focal_length=None, scale_first=False):
        self.translation, self.rotation, self.scale = translation, rotation, scale
        self.focal_length, self.scale_first = focal_length, scale_first

    def keys(self):
        return [k for k in self.KEYS if getattr(self, k) is not None]

    def get(self, key, default=None):
        return getattr(self, key, default)

    def __getitem__(self, key):
        return getattr(self, key)


DEFAULT_FOCAL_LENGTH = 5000


class PerspectiveCamera(nn.Module):
    """Pinhole camera, camera frame x right, y down, z forward: p = f (Y_x / Y_z, Y_y / Y_z) + camera_center with
    Y = rotation X + translation.  The focal length is a constant of the projection (no gradient flows into it)."""

    FOCAL_LENGTH = DEFAULT_FOCAL_LENGTH

    def __init__(self, dtype=torch.float32, focal_length=None, **kwargs):
        super().__init__()
        self.dtype = dtype
        self.register_buffer('focal_length', torch.tensor(self.FOCAL_LENGTH if focal_length is None else focal_length,
                                                          dtype=dtype))

    def forward(self, points, focal_length=None, translation=None, rotation=None, camera_center=None, **kwargs):
        """points (B, N, 3); focal_length a scalar or (B,) (default the module's); translation (B, 3), rotation
        (B, 3, 3) and camera_center (B, 2), by default zero, identity and zero.  Returns (B, N, 2)."""
        B = points.shape[0]
        y = points if rotation is None else torch.einsum('bji,bmi->bmj', rotation, points)
        if translation is not None:
            y = y + translation.unsqueeze(1)
        f = self.focal_length if focal_length is None else focal_length
        f = torch.as_tensor(f, dtype=self.dtype, device=points.device).detach().reshape(-1).expand(B)
        img = f.view(B, 1, 1) * (y[..., :2] / y[..., 2:])
        if camera_center is not None:
            img = img + camera_center.reshape(-1, 1, 2)
        return img


class WeakPerspectiveCamera(nn.Module):
    def __init__(self, scale_first=False, **kwargs):
        super().__init__()
        self.scale_first = scale_first


def build_cam_proj(camera_cfg, dtype=torch.float32):
    get = (lambda k, d=None: camera_cfg.get(k, d)) if camera_cfg is not None else (lambda k, d=None: d)
    camera_type = get('type', 'weak-persp') or 'weak-persp'
    pos = get('pos_func', 'softplus')
    if camera_type.lower() != 'weak-persp' or pos != 'softplus':
        raise ValueError('shapy_b200 implements the weak-persp camera with pos_func=softplus only')
    wp = get('weak_persp', {}) or {}
    if wp.get('scale_first', False):
        raise ValueError('shapy_b200: weak_persp.scale_first=True is not implemented')
    mean_scale = wp.get('mean_scale', 0.9)
    mean_scale = math.log(math.exp(mean_scale) - 1)
    return {'camera': WeakPerspectiveCamera(scale_first=False), 'mean': torch.tensor([mean_scale, 0.0, 0.0]),
            'scale_func': F.softplus, 'dim': 3}
