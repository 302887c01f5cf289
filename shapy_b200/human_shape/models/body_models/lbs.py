"""`lbs()` with the reference signature (regressor/human_shape/models/body_models/lbs.py:99-108),
evaluated by the fused sm_90a kernels (csrc/smplx.cu).  The reference's own TODO reads "Create merged
c++ and CUDA kernel" (lbs.py:97-98)."""
from collections import defaultdict

import torch

from .... import ops as _ops

# one packed model: (key, source tensors, SmplxModel).  The entry holds the source tensors, so their storage cannot be
# freed and handed to new tensors while the key still names it.
_CACHE = {}


def _tensor_key(t):
    """Identity and contents version of a model tensor: an in-place edit bumps `_version`, so a packed model is never
    served for contents it was not built from.  Inference tensors have no version counter: None (never cached)."""
    if t.is_inference():
        return None
    return (int(t.data_ptr()), tuple(t.shape), tuple(t.stride()), t.dtype, str(t.device), t._version)


def lbs(betas, pose, v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights, pose2rot=True,
        return_shaped=True):
    """pose: (B, J, 3, 3) / (B, J*9) rotation matrices (pose2rot=False).  Axis-angle input
    (pose2rot=True) is not on the SHAPY_A path and raises."""
    if pose2rot:
        raise NotImplementedError('shapy_b200 lbs(): pass rotation matrices (pose2rot=False)')
    src = (v_template, shapedirs, posedirs, J_regressor, lbs_weights)
    parts = [_tensor_key(t) for t in src]
    key = None if None in parts else tuple(parts) + (tuple(torch.as_tensor(parents).tolist()), str(betas.device))
    entry = _CACHE.get('lbs')
    if key is not None and entry is not None and entry[0] == key:
        model = entry[2]
    else:
        tensors = dict(v_template=v_template, shapedirs=shapedirs, posedirs=posedirs, J_regressor=J_regressor,
                       lbs_weights=lbs_weights, parents=torch.as_tensor(parents),
                       faces_tensor=torch.zeros(1, 3, dtype=torch.long))
        model = _ops.SmplxModel(tensors, betas.device)
        _CACHE.clear()
        if key is not None:
            _CACHE['lbs'] = (key, src, model)
    B = betas.shape[0]
    rot = pose.reshape(B, -1, 3, 3)
    out = _ops.smplx_forward(model, betas, rot, want_v_shaped=return_shaped)
    output = defaultdict(lambda: None, vertices=out['vertices'], joints=out['joints'])
    if return_shaped:
        output['v_shaped'] = out['v_shaped']
    return output
