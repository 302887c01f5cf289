"""GPU SMPL-X forward against the float64 oracle (oracle.smplx_oracle.smplx_forward_full, pinned to the reference's own
float64 lbs() by tests/test_oracle_pins.py), run on the same fp32 inputs the kernels receive:

  * every pose width the SMPLX module builds (22, 23, 24, 25, 40, 55 rotated joints), with expression and transl
  * calls of several widths on one model, in rising and falling order (the pose-blend weights are cached per width)
  * the split-fp16 pose-blend GEMM alone, isolated through lbs() on a model whose skinning is the identity
  * shape / expression counts other than 10 / 10, the generic T-pose kernel, and the global-rotation-only forward
  * the dynamic-contour LUT over a sweep of neck angles, and the camera's softplus on both sides of its threshold

Each family asserts the 1e-4 contract and a tight bar set from the errors measured on an H100 (in the comments)."""
import math

import pytest
import torch

from oracle import smplx_oracle
from shapy_b200 import synth

pytestmark = pytest.mark.gpu
TOL = 1e-4          # the contract: 1e-4 of the largest reference value


def err(a, b):
    """max |a - b| / max |b|, in float64."""
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-300))


def rodrigues(aa):
    """(..., 3) axis-angle -> (..., 3, 3) rotations, float64."""
    aa = aa.double()
    th = aa.norm(dim=-1, keepdim=True)
    k = aa / th.clamp_min(1e-300)
    kx, ky, kz = k.unbind(-1)
    z = torch.zeros_like(kx)
    K = torch.stack([z, -kz, ky, kz, z, -kx, -ky, kx, z], -1).view(*aa.shape[:-1], 3, 3)
    s, c = th.sin()[..., None], th.cos()[..., None]
    return torch.eye(3, dtype=torch.float64) + s * K + (1 - c) * (K @ K)


def random_rot(g, B, n, scale=0.3):
    """(B, n, 3, 3) fp32 rotations, axis-angle components ~ N(0, scale)."""
    return rodrigues(torch.randn(B, n, 3, generator=g, dtype=torch.float64) * scale).float()


@pytest.fixture(scope='module')
def model():
    return synth.make_smplx()


@pytest.fixture(scope='module')
def module(model):
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    return SMPLX(data_struct=model, use_face_contour=True).cuda()


# ---------------------------------------------------------------------------------------------- every pose width
# name -> (keyword, first joint, joint count) of the pose parts the SMPLX module takes after global_rot and body_pose
PARTS = dict(jaw=('jaw_pose', 22, 1), leye=('leye_pose', 23, 1), reye=('reye_pose', 24, 1),
             lhand=('left_hand_pose', 25, 15), rhand=('right_hand_pose', 40, 15))
COMBOS = dict(none=(), jaw=('jaw',), leye=('leye',), reye=('reye',), lhand=('lhand',), rhand=('rhand',),
              all=tuple(PARTS))
# largest error over the 21 cases below (vertices / joints / v_shaped), measured on an H100 80GB HBM3 at a 400 W power
# limit: 4.2e-7; 5.0e-7 in the cache-order test.  A plain-fp16 pose blend (~2.5e-4 of a 0.026 m blend) adds ~4e-6 of 1.58 m.
TIGHT_MODULE = 1e-6


def module_inputs(seed, B, combo):
    g = torch.Generator().manual_seed(seed)
    rot = random_rot(g, B, 55)
    kw = dict(global_rot=rot[:, :1], body_pose=rot[:, 1:22], betas=torch.randn(B, 10, generator=g),
              expression=torch.randn(B, 10, generator=g), transl=torch.randn(B, 3, generator=g) * 0.5)
    n_rot = 22
    for name in COMBOS[combo]:
        key, j0, n = PARTS[name]
        kw[key] = rot[:, j0:j0 + n]
        n_rot = max(n_rot, j0 + n)
    # what the oracle sees: the parts given, identity elsewhere
    given = torch.eye(3).expand(B, 55, 3, 3).clone()
    given[:, :22] = rot[:, :22]
    for name in COMBOS[combo]:
        _, j0, n = PARTS[name]
        given[:, j0:j0 + n] = rot[:, j0:j0 + n]
    return kw, given, n_rot


@pytest.mark.parametrize('B', [1, 33, 70])
@pytest.mark.parametrize('combo', list(COMBOS))
def test_pose_widths_module(model, module, combo, B):
    kw, given, n_rot = module_inputs(1000 + B, B, combo)
    out = module(**{k: v.cuda() for k, v in kw.items()}, return_full_pose=True)
    ref = smplx_oracle.smplx_forward_full(model, kw['betas'], given, expression=kw['expression'], transl=kw['transl'])
    assert out['full_pose'].shape == (B, 55, 3, 3)
    assert torch.equal(out['full_pose'].cpu().double(), ref['full_pose'])
    errs = {k: err(out[k]._t if k == 'joints' else out[k], ref[k]) for k in ('vertices', 'joints', 'v_shaped')}
    print(f'pose widths {combo} (n_rot {n_rot}) B={B}:', {k: f'{v:.2e}' for k, v in errs.items()})
    for k, e in errs.items():
        assert e < TOL, (k, e)
        assert e < TIGHT_MODULE, (k, e)


# ---------------------------------------------------------------------------------------------- cache order
WIDTHS = [23, 24, 22, 55, 40, 25]
# the module's pose part that makes each width: the parts before it are materialised as identity
WIDTH_PART = {22: None, 23: 'jaw', 24: 'leye', 25: 'reye', 40: 'lhand', 55: 'rhand'}


def test_pose_width_cache_order(model, module):
    """Pose-blend weights are packed once per padded width (23 and 24 joints share one) and reused.  Every call on a
    shared model, in rising and falling order, must equal the same call on a freshly built model, bit for bit."""
    from shapy_b200 import ops
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    B = 33
    g = torch.Generator().manual_seed(77)
    rot = random_rot(g, B, 55)
    betas, expr = torch.randn(B, 10, generator=g), torch.randn(B, 10, generator=g)
    shared = ops.SmplxModel({**model, 'use_face_contour': True}, 'cuda:0')

    def ops_call(m, n):
        return ops.smplx_forward(m, betas.cuda(), rot[:, :n].contiguous().cuda(), expr=expr.cuda())

    def module_call(mod, n):
        kw = dict(global_rot=rot[:, :1], body_pose=rot[:, 1:22], betas=betas, expression=expr)
        if WIDTH_PART[n]:
            key, j0, k = PARTS[WIDTH_PART[n]]
            kw[key] = rot[:, j0:j0 + k]
        return mod(**{k: v.cuda() for k, v in kw.items()})

    fresh_ops, fresh_mod = {}, {}
    for n in WIDTHS:
        fresh_ops[n] = ops_call(ops.SmplxModel({**model, 'use_face_contour': True}, 'cuda:0'), n)
        fresh_mod[n] = module_call(SMPLX(data_struct=model, use_face_contour=True).cuda(), n)
    worst = 0.0
    for n in WIDTHS + WIDTHS[::-1]:
        a, b = ops_call(shared, n), module_call(module, n)
        for k in ('vertices', 'joints', 'v_shaped'):
            assert torch.equal(a[k], fresh_ops[n][k]), (n, k, err(a[k], fresh_ops[n][k]))
        for k in ('vertices', 'v_shaped'):
            assert torch.equal(b[k], fresh_mod[n][k]), (n, k, err(b[k], fresh_mod[n][k]))
        assert torch.equal(b['joints']._t, fresh_mod[n]['joints']._t), (n, 'module joints')
        given = torch.eye(3).expand(B, 55, 3, 3).clone()
        given[:, :n] = rot[:, :n]
        if n > 22 and WIDTH_PART[n] != 'jaw':
            # the module materialises the parts before the given one as identity; the ops call rotates them
            given_mod = given.clone()
            given_mod[:, 22:PARTS[WIDTH_PART[n]][1]] = torch.eye(3)
        else:
            given_mod = given
        for out, gv in ((a, given), (b, given_mod)):
            ref = smplx_oracle.smplx_forward_full(model, betas, gv, expression=expr)
            for k in ('vertices', 'joints'):
                e = err(out[k]._t if k == 'joints' and hasattr(out[k], '_t') else out[k], ref[k])
                worst = max(worst, e)
                assert e < TIGHT_MODULE, (n, k, e)
    print(f'cache order: largest error vs float64 {worst:.2e}')


def test_lbs_cache_sees_in_place_edit():
    """lbs() caches the packed model; an in-place edit of a model tensor must reach the next call."""
    from shapy_b200.human_shape.models.body_models.lbs import lbs
    g = torch.Generator().manual_seed(3)
    V, J, B = 300, 24, 5
    parents = torch.tensor(synth.SMPLX_PARENTS[:J])
    v_template = (torch.randn(V, 3, generator=g) * 0.3).cuda()
    shapedirs = (torch.randn(V, 3, 4, generator=g) * 0.01).cuda()
    posedirs = (torch.randn((J - 1) * 9, V * 3, generator=g) * 0.01).cuda()
    Jreg = torch.rand(J, V, generator=g)
    Jreg = (Jreg / Jreg.sum(1, keepdim=True)).cuda()
    W = torch.rand(V, J, generator=g)
    W = (W / W.sum(1, keepdim=True)).cuda()
    betas = torch.randn(B, 4, generator=g).cuda()
    rot = random_rot(g, B, J).cuda()
    args = lambda: (betas, rot, v_template, shapedirs, posedirs, Jreg, parents, W)  # noqa: E731
    mdl = dict(v_template=v_template, shapedirs=shapedirs, posedirs=posedirs, J_regressor=Jreg, lbs_weights=W,
               parents=parents, faces_tensor=torch.zeros(1, 3, dtype=torch.long))
    first = lbs(*args(), pose2rot=False)['vertices'].clone()
    posedirs.mul_(2)
    second = lbs(*args(), pose2rot=False)['vertices']
    ref = smplx_oracle.smplx_forward_full(mdl, betas, rot)['vertices']
    assert not torch.equal(first, second)
    assert err(second, ref) < 1e-5, err(second, ref)
    v_template.add_(0.25)
    third = lbs(*args(), pose2rot=False)['vertices']
    assert err(third, smplx_oracle.smplx_forward_full(mdl, betas, rot)['vertices']) < 1e-5


# ---------------------------------------------------------------------------------------------- pose-blend GEMM alone
# (J, V, B, posedirs scale): J sweeps Kp = 9 (J - 1) from 9 to 567 and the partial last k16 step; V sweeps 3V around the
# 384 padding; B sweeps the GEMM's 128-body tiles and the vertex kernel's 32-body tiles; the scale sweeps posedirs
# against kPoseScale = 1024.  The largest V is not crossed with the largest B, to keep the float64 work small.
GEMM_CASES = ([(J, 129, 33, 1e-3) for J in (2, 22, 23, 24, 40, 55, 64)] +
              [(55, V, 33, 1e-3) for V in (1, 127, 128, 129, 10475)] +
              [(23, 128, B, 1e-3) for B in (1, 31, 32, 33, 127, 128, 129, 300)] +
              [(40, 127, 129, s) for s in (1e-5, 1e-3, 1e-1)] +
              [(64, 10475, 3, 1e-1), (2, 1, 300, 1e-5), (24, 10475, 70, 1e-5)])
# largest error / largest |blend| over GEMM_CASES, measured on an H100 80GB HBM3 (400 W): 1.0e-6.  The same GEMM in
# plain fp16 (both operands' lo halves zeroed) gives 2.5e-4 to 4.1e-4 in every case and fails this bar.
TIGHT_GEMM = 2e-5


def blend_model(J, V, scale, g):
    """A model whose forward returns exactly the pose blend: zero template and shape, skinning one-hot on joint 0."""
    parents = torch.tensor([-1] + [(j - 1) // 2 for j in range(1, J)])
    W = torch.zeros(V, J)
    W[:, 0] = 1
    return dict(v_template=torch.zeros(V, 3), shapedirs=torch.zeros(V, 3, 1),
                posedirs=torch.randn((J - 1) * 9, V * 3, generator=g) * scale,
                J_regressor=torch.zeros(J, V), lbs_weights=W, parents=parents)


def lbs_blend(m, rot):
    from shapy_b200.human_shape.models.body_models.lbs import lbs
    B, V = rot.shape[0], m['v_template'].shape[0]
    c = lambda t: t.cuda()  # noqa: E731
    out = lbs(torch.zeros(B, 1).cuda(), c(rot), c(m['v_template']), c(m['shapedirs']), c(m['posedirs']),
              c(m['J_regressor']), m['parents'], c(m['lbs_weights']), pose2rot=False, return_shaped=False)
    return out['vertices'].reshape(B, 3 * V)


def ref_blend(m, rot):
    B = rot.shape[0]
    pf = (rot[:, 1:].double() - torch.eye(3, dtype=torch.float64)).reshape(B, -1)
    return pf @ m['posedirs'].double()


@pytest.mark.parametrize('J,V,B,scale', GEMM_CASES)
def test_pose_blend_gemm(J, V, B, scale):
    g = torch.Generator().manual_seed(J * 1000003 + V * 101 + B)
    m = blend_model(J, V, scale, g)
    rot = random_rot(g, B, J)
    rot[:, 0] = torch.eye(3)
    got, ref = lbs_blend(m, rot), ref_blend(m, rot)
    e = err(got, ref)
    print(f'pose blend J={J} V={V} B={B} scale={scale:g}: {e:.2e} of max |blend| {float(ref.abs().max()):.2e}')
    assert e < TIGHT_GEMM, e


# largest absolute error of the near-identity blend, measured on an H100 80GB HBM3 (400 W): 8.5e-10 m of a 2.6e-6 m
# blend.  That is the split format's floor: features of ~3e-5 / kPoseScale leave hi = 0 and put the value in lo's
# subnormal range, whose spacing is 2^-26 ~ 1.5e-8 per unscaled feature.  Plain fp16 gives 1.7e-6 m.
TIGHT_GEMM_NEAR_ID = 2e-9


def test_pose_blend_gemm_near_identity():
    """Rotations within 1e-4 rad: the features' hi halves are fp16 subnormals, the lo halves carry the value."""
    g = torch.Generator().manual_seed(5)
    J, V, B = 55, 10475, 33
    m = blend_model(J, V, 1e-3, g)
    rot = rodrigues(torch.randn(B, J, 3, generator=g, dtype=torch.float64) * 3e-5).float()
    rot[:, 0] = torch.eye(3)
    got, ref = lbs_blend(m, rot), ref_blend(m, rot)
    e = float((got.double().cpu() - ref).abs().max())
    print(f'pose blend near identity: {e:.2e} m of max |blend| {float(ref.abs().max()):.2e} m')
    assert e < TIGHT_GEMM_NEAR_ID, e


# ---------------------------------------------------------------------------------------------- shape / expression
# largest error over the cases below (vertices / joints / v_shaped / forward_shape), measured on an H100 80GB HBM3
# (400 W): 6.0e-7
TIGHT_SHAPE = 1.5e-6


@pytest.mark.parametrize('NB,NE', [(1, 0), (1, 10), (10, 0), (10, 10), (16, 0), (16, 10), (22, 0), (22, 10)])
def test_shape_expression_counts(model, NB, NE):
    from shapy_b200 import ops
    g = torch.Generator().manual_seed(NB * 100 + NE)
    V = model['v_template'].shape[0]
    m = {k: v for k, v in model.items() if k != 'expr_dirs'}
    m['shapedirs'] = torch.randn(V, 3, NB, generator=g) * 5e-3
    if NE:
        m['expr_dirs'] = torch.randn(V, 3, NE, generator=g) * 5e-3
    packed = ops.SmplxModel({**m, 'use_face_contour': True}, 'cuda:0')
    B = 33
    betas = torch.randn(B, NB, generator=g)
    expr = torch.randn(B, NE, generator=g) if NE else None
    rot = random_rot(g, B, 55)
    worst = {}
    for n_rot in (55, 1):           # n_rot = 1: no pose feature, no GEMM launch
        out = ops.smplx_forward(packed, betas.cuda(), rot[:, :n_rot].contiguous().cuda(),
                                expr=None if expr is None else expr.cuda())
        ref = smplx_oracle.smplx_forward_full(m, betas, rot[:, :n_rot], expression=expr)
        for k in ('vertices', 'joints', 'v_shaped'):
            worst[f'{k}{n_rot}'] = err(out[k], ref[k])
    if NE:
        # expression moves the joints (through J) but not v_shaped
        no_e = smplx_oracle.smplx_forward_full(m, betas, rot[:, :1])
        assert err(ref['joints'], no_e['joints']) > 100 * TIGHT_SHAPE
        assert torch.equal(ref['v_shaped'], no_e['v_shaped'])
    vs = ops.smplx_forward_shape(packed, betas.cuda())     # NB != 10: the generic T-pose kernel
    worst['forward_shape'] = err(vs, smplx_oracle.smplx_forward_full(m, betas, rot[:, :1])['v_shaped'])
    print(f'shape NB={NB} NE={NE}:', {k: f'{v:.2e}' for k, v in worst.items()})
    for k, e in worst.items():
        assert e < TOL, (k, e)
        assert e < TIGHT_SHAPE, (k, e)


# ---------------------------------------------------------------------------------------------- contour LUT, camera
# largest error of the 17 dynamic landmarks over the sweep, measured on an H100 80GB HBM3 (400 W): 3.5e-7; a wrong LUT
# row moves them by centimetres
TIGHT_LUT = 1e-6


def test_dynamic_contour_lut_sweep(model):
    """Neck (joint 12) about y from -60 to +60 degrees in ~0.7 degree steps: LUT rows 0-39, 40-78 and both clamps.
    Angles within 0.05 degrees of a half degree are skipped, where fp32 and float64 may round to different rows."""
    from shapy_b200 import ops
    packed = ops.SmplxModel({**model, 'use_face_contour': True}, 'cuda:0')
    deg = torch.linspace(-60, 60, 172, dtype=torch.float64)
    deg = deg[((deg.abs() % 1) - 0.5).abs() > 0.05]
    B = deg.shape[0]
    aa = torch.zeros(B, 22, 3, dtype=torch.float64)
    aa[:, 12, 1] = deg * math.pi / 180
    rot = rodrigues(aa).float()
    betas = torch.randn(B, 10, generator=torch.Generator().manual_seed(9))
    out = ops.smplx_forward(packed, betas.cuda(), rot.cuda())
    ref = smplx_oracle.smplx_forward_full(model, betas, rot)
    df, _ = smplx_oracle.dynamic_landmarks(ref['full_pose'], model['dynamic_lmk_faces_idx'],
                                           model['dynamic_lmk_bary_coords'], model['neck_kin_chain'])
    rows = {int((model['dynamic_lmk_faces_idx'] == df[b]).all(1).nonzero()[0]) for b in range(B)}
    assert {0, 1, 38, 39, 40, 41, 77, 78} <= rows and len(rows) == 79, sorted(rows)
    D = model['dynamic_lmk_faces_idx'].shape[1]
    e = err(out['joints'][:, -D:], ref['joints'][:, -D:])
    print(f'contour LUT sweep ({B} angles): {e:.2e}')
    assert e < TIGHT_LUT, e


# largest per-body error of the projection, measured on an H100 80GB HBM3 (400 W): 1.1e-7
TIGHT_CAMERA = 5e-7


def test_camera_softplus_threshold(model):
    from shapy_b200 import ops
    packed = ops.SmplxModel({**model, 'use_face_contour': True}, 'cuda:0')
    c0 = torch.tensor([-30.0, -1.0, 0.0, 19.9, 20.0, 20.1, 40.0])
    B = c0.shape[0]
    g = torch.Generator().manual_seed(13)
    cam = torch.cat([c0[:, None], torch.randn(B, 2, generator=g) * 0.1], 1)
    out = ops.smplx_forward(packed, torch.randn(B, 10, generator=g).cuda(), random_rot(g, B, 22).cuda(),
                            camera=cam.cuda())
    cam64, joints = cam.double(), out['joints'].double().cpu()
    ref = torch.nn.functional.softplus(cam64[:, 0]).view(-1, 1, 1) * (joints[:, :, :2] + cam64[:, None, 1:])
    errs = [err(out['proj_joints'][b], ref[b]) for b in range(B)]
    print('camera per body:', [f'{e:.1e}' for e in errs])
    assert max(errs) < TIGHT_CAMERA, errs
