"""`lbs()` with the reference signature (regressor/human_shape/models/body_models/lbs.py:99-108),
evaluated by the fused sm_90a kernels (csrc/smplx.cu).  The reference's own TODO reads "Create merged
c++ and CUDA kernel" (lbs.py:97-98)."""
from collections import defaultdict

import torch

from .... import ops as _ops

_CACHE = {}


def lbs(betas, pose, v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights, pose2rot=True,
        return_shaped=True):
    """pose: (B, J, 3, 3) / (B, J*9) rotation matrices (pose2rot=False).  Axis-angle input
    (pose2rot=True) is not on the SHAPY_A path and raises."""
    if pose2rot:
        raise NotImplementedError('shapy_b200 lbs(): pass rotation matrices (pose2rot=False)')
    key = tuple(int(t.data_ptr()) for t in (v_template, shapedirs, posedirs, J_regressor, lbs_weights)) + \
        (str(betas.device),)
    model = _CACHE.get(key)
    if model is None:
        V = v_template.shape[0]
        tensors = dict(v_template=v_template, shapedirs=shapedirs, posedirs=posedirs, J_regressor=J_regressor,
                       lbs_weights=lbs_weights, parents=torch.as_tensor(parents),
                       faces_tensor=torch.zeros(1, 3, dtype=torch.long))
        model = _ops.SmplxModel(tensors, betas.device)
        _CACHE.clear()
        _CACHE[key] = model
    B = betas.shape[0]
    rot = pose.reshape(B, -1, 3, 3)
    out = _ops.smplx_forward(model, betas, rot, want_v_shaped=return_shaped)
    output = defaultdict(lambda: None, vertices=out['vertices'], joints=out['joints'])
    if return_shaped:
        output['v_shaped'] = out['v_shaped']
    return output
