"""Pose parameterisation, host mirror of regressor/human_shape/models/common/pose_utils.py
(ContinuousRotReprDecoder 73-153, build_pose_parameterization).  Only `cont_rot_repr` is on the
SHAPY_A path (configs/b2a_expose_hrnet_demo.yaml:226-229)."""
from dataclasses import dataclass

import torch
import torch.nn as nn

from .... import autograd as _ag
from .... import ops as _ops


@dataclass
class PoseParameterization:
    dim: int
    ind_dim: int
    decoder: nn.Module
    mean: torch.Tensor
    regressor: nn.Module = None


class ContinuousRotReprDecoder(nn.Module):
    """6D -> rotation matrix (Gram-Schmidt).  The 6 numbers are a row-major 3x2 matrix."""

    def __init__(self, num_angles, dtype=torch.float32, mean=None, **kwargs):
        super().__init__()
        self.num_angles = num_angles
        self.dtype = dtype
        if isinstance(mean, dict):
            mean = mean.get('cont_rot_repr', None)
        if mean is None:
            mean = torch.tensor([1.0, 0.0, 0.0, 1.0, 0.0, 0.0], dtype=dtype).unsqueeze(0).expand(
                num_angles, -1).contiguous().view(-1)
        if not torch.is_tensor(mean):
            mean = torch.tensor(mean)
        mean = mean.reshape(-1, 6)
        if mean.shape[0] < num_angles:
            mean = mean.repeat(num_angles // mean.shape[0] + 1, 1).contiguous()
            mean = mean[:num_angles]
        elif mean.shape[0] > num_angles:
            mean = mean[:num_angles]
        self.register_buffer('mean', mean.reshape(-1).to(dtype))

    def get_type(self):
        return 'cont_rot_repr'

    def get_param_dim(self):
        return 6

    def get_dim_size(self):
        return self.num_angles * 6

    def get_mean(self):
        return self.mean.clone()

    def forward(self, module_input):
        """Differentiable (shapy_b200.autograd.Rot6dFunction) when grad mode is on and the input requires grad."""
        if _ag.wants_grad(module_input):
            return _ag.Rot6dFunction.apply(module_input)
        return _ops.decode_rot6d(module_input)


def build_pose_parameterization(num_angles, type='cont_rot_repr', mean=None, **kwargs):
    if type != 'cont_rot_repr':
        raise ValueError(f'shapy_b200 implements the cont_rot_repr pose parameterisation only, got: {type}')
    decoder = ContinuousRotReprDecoder(num_angles, mean=mean)
    return PoseParameterization(dim=decoder.get_dim_size(), ind_dim=6, decoder=decoder, mean=decoder.get_mean())
