"""TEST INFRASTRUCTURE ONLY -- loads the reference's own math files verbatim.

Works only in the build container, where ``/root/reference`` is mounted.  It is
used by ``tools/make_golden.py`` (to write ``tests/golden/*``) and by the
``not gpu`` tests that pin ``oracle/*.py`` restatements against the real
reference code.  Nothing in the product package imports this file, and nothing
on the GPU box can (``/root/reference`` does not exist there).

The reference package ``human_shape`` cannot be imported as a whole (missing
yacs / omegaconf / fvcore / trimesh ...), but its arithmetic files only need
torch / numpy / loguru.  They are loaded by path behind stub parent packages
(SURVEY.md Appendix B):

    regressor/human_shape/utils/rotation_utils.py
    regressor/human_shape/models/body_models/utils.py      (transform_mat, KeypointTensor)
    regressor/human_shape/models/body_models/lbs.py        (lbs, landmarks)
    regressor/human_shape/models/common/networks.py        (MLP, IterativeRegression)
    regressor/human_shape/models/common/pose_utils.py      (ContinuousRotReprDecoder)
    regressor/human_shape/models/backbone/hrnet.py         (HighResolutionNet)
"""
import importlib.util
import io
import os
import sys
import types
from typing import List, NewType

import numpy as np
import torch

REF = os.environ.get('SHAPY_REFERENCE', '/root/reference')
HS = os.path.join(REF, 'regressor', 'human_shape')


def available() -> bool:
    return os.path.isdir(HS)


def _load(name, path, pkg=None):
    spec = importlib.util.spec_from_file_location(name, path)
    m = importlib.util.module_from_spec(spec)
    sys.modules[name] = m
    if pkg:
        m.__package__ = pkg
    spec.loader.exec_module(m)
    return m


_CACHE = {}


def load():
    """Returns a namespace with the reference modules: rot, butils, lbs, net, pu, hrnet."""
    if _CACHE:
        return types.SimpleNamespace(**_CACHE)
    if not available():
        raise RuntimeError(f'reference tree not found at {REF}')
    from loguru import logger
    logger.remove()

    def stub(name):
        m = types.ModuleType(name)
        m.__path__ = []
        sys.modules[name] = m
        return m

    stub('human_shape')
    u = stub('human_shape.utils')
    ty = types.ModuleType('human_shape.utils.typing')
    ty.Tensor = NewType('Tensor', torch.Tensor)
    sys.modules['human_shape.utils.typing'] = ty
    rot = _load('human_shape.utils.rotation_utils', HS + '/utils/rotation_utils.py', 'human_shape.utils')
    for n in ['batch_rodrigues', 'batch_rot2aa', 'rot_mat_to_euler']:
        setattr(u, n, getattr(rot, n))
    u.Tensor = ty.Tensor
    u.IntList = NewType('IntList', List[int])
    u.StringList = NewType('StringList', List[str])
    for n in ['CN', 'Array', 'IntTuple', 'FloatList', 'FloatTuple', 'TensorList']:
        setattr(u, n, object)
    stub('human_shape.models')
    stub('human_shape.models.body_models')
    butils = _load('human_shape.models.body_models.utils', HS + '/models/body_models/utils.py',
                   'human_shape.models.body_models')
    lbs = _load('human_shape.models.body_models.lbs', HS + '/models/body_models/lbs.py',
                'human_shape.models.body_models')
    nn_ = types.ModuleType('human_shape.models.nnutils')
    sys.modules['human_shape.models.nnutils'] = nn_
    il = _load('human_shape.models.nnutils.init_layer', HS + '/models/nnutils/init_layer.py')
    nn_.init_weights = il.init_weights
    stub('human_shape.models.common')
    try:
        import omegaconf  # noqa: F401
    except ImportError:
        oc = types.ModuleType('omegaconf')
        oc.DictConfig = dict
        sys.modules['omegaconf'] = oc
    net = _load('human_shape.models.common.networks', HS + '/models/common/networks.py',
                'human_shape.models.common')
    pu = _load('human_shape.models.common.pose_utils', HS + '/models/common/pose_utils.py',
               'human_shape.models.common')
    hrnet = _load('shapy_ref_hrnet', HS + '/models/backbone/hrnet.py')
    _CACHE.update(rot=rot, butils=butils, lbs=lbs, net=net, pu=pu, hrnet=hrnet)
    return types.SimpleNamespace(**_CACHE)


class AttrDict(dict):
    __getattr__ = dict.__getitem__


def hrnet_cfg():
    """Stage table of regressor/human_shape/config/network_defaults.py:92-132 (HRNet-W48)."""
    def st(**k):
        d = dict(num_modules=1, num_branches=1, num_blocks=(4,), num_channels=(64,),
                 block='BOTTLENECK', fuse_method='SUM')
        d.update(k)
        return AttrDict(d)
    return AttrDict(
        use_old_impl=False, pretrained_layers=('*',), pretrained_path='',
        stage1=st(),
        stage2=st(num_branches=2, num_blocks=(4, 4), num_channels=(48, 96), block='BASIC'),
        stage3=st(num_modules=4, num_branches=3, num_blocks=(4, 4, 4), num_channels=(48, 96, 192), block='BASIC'),
        stage4=st(num_modules=3, num_branches=4, num_blocks=(4, 4, 4, 4), num_channels=(48, 96, 192, 384),
                  block='BASIC'))


def build_hrnet():
    ref = load()
    return ref.hrnet.HighResolutionNet(hrnet_cfg()).eval()


def load_img00():
    """samples/shapy_fit_for_virtual_measurements/img_00.npz (pickled CUDA tensors -> CPU)."""
    import torch.storage
    _orig = torch.load
    saved = torch.storage._load_from_bytes
    torch.storage._load_from_bytes = lambda b: _orig(io.BytesIO(b), map_location='cpu', weights_only=False)
    try:
        d = np.load(os.path.join(REF, 'samples/shapy_fit_for_virtual_measurements/img_00.npz'), allow_pickle=True)
        out = {k: d[k] for k in d.files}
        out['measurements'] = {k: float(v.item()) for k, v in out['measurements'].item().items()}
    finally:
        torch.storage._load_from_bytes = saved
    return out


def smplx_forward_ref(model: dict, betas, global_rot, body_pose, jaw_pose=None, leye_pose=None, reye_pose=None,
                      left_hand_pose=None, right_hand_pose=None, expression=None, transl=None):
    """Re-assembly of SMPLX.forward (body_models.py:628-767) on top of the verbatim lbs.py.

    ``model`` is the dict produced by shapy_b200.synth.make_smplx (torch tensors), in the dtype of ``betas``.
    Pose parts that are not given are identity and a missing expression is zero, as in the reference;
    use_face_contour=True, J14 on.
    """
    ref = load()
    lbs = ref.lbs
    B = betas.shape[0]
    eye = torch.eye(3, dtype=betas.dtype).view(1, 1, 3, 3)
    ident = lambda n: eye.expand(B, n, -1, -1).contiguous()  # noqa: E731
    part = lambda p, n: ident(n) if p is None else p.reshape(B, n, 3, 3)  # noqa: E731
    full_pose = torch.cat([global_rot, body_pose, part(jaw_pose, 1), part(leye_pose, 1), part(reye_pose, 1),
                           part(left_hand_pose, 15), part(right_hand_pose, 15)], dim=1)
    if expression is None:
        expression = torch.zeros(B, model['expr_dirs'].shape[-1], dtype=betas.dtype)
    shape_components = torch.cat([betas, expression], dim=-1)
    shapedirs = torch.cat([model['shapedirs'], model['expr_dirs']], dim=-1)
    out = lbs.lbs(shape_components, full_pose, model['v_template'], shapedirs, model['posedirs'],
                  model['J_regressor'], model['parents'], model['lbs_weights'], pose2rot=False,
                  return_shaped=True)
    vertices, joints = out['vertices'], out['joints']
    lmk_faces_idx = model['lmk_faces_idx'].unsqueeze(0).expand(B, -1)
    lmk_bary = model['lmk_bary_coords'].unsqueeze(0).expand(B, -1, -1)
    dyn_f, dyn_b = lbs.find_dynamic_lmk_idx_and_bcoords(
        vertices, full_pose, model['dynamic_lmk_faces_idx'], model['dynamic_lmk_bary_coords'],
        model['neck_kin_chain'])
    lmk_faces_idx = torch.cat([lmk_faces_idx, dyn_f], 1)
    lmk_bary = torch.cat([lmk_bary.expand(B, -1, -1), dyn_b], 1)
    landmarks = lbs.vertices2landmarks(vertices, model['faces_tensor'], lmk_faces_idx, lmk_bary)
    joints = torch.cat([joints, landmarks], dim=1)
    reg = torch.einsum('ji,bik->bjk', model['extra_joint_regressor'], vertices)
    joints[:, model['source_idxs']] = joints[:, model['source_idxs']] * 0.0 + reg[:, model['target_idxs']] * 1.0
    if transl is not None:
        joints += transl.unsqueeze(dim=1)
        vertices += transl.unsqueeze(dim=1)
    v_shaped = model['v_template'] + lbs.blend_shapes(betas, model['shapedirs'])
    return dict(vertices=vertices, joints=joints, v_shaped=v_shaped, full_pose=full_pose)
