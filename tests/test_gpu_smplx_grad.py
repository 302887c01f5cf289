"""GPU: the posed SMPL-X backward (shapy_smplx_backward) and the 6D decoder's backward, through ops and autograd.

  * against the reference's own autograd (tests/golden/ref_smplx_grad.npz) through SMPLX.forward end to end
  * against float64 autograd of the oracle's forward (tests/smplx_grad_ref.py) at B = 1, 64 and 4096 (rows sampled), every pose
    width, with and without expression, camera, J14 and face contour, on one-hot and mixed cotangents
  * the decoder backward, raw 6D -> decoder -> SMPLX.forward -> a loss on the KeypointTensor joints
  * determinism, batch independence, the unchanged no-grad path, and the batched keypoint fit

Bar: per body and per gradient tensor, max |g - g64| <= 1e-4 max |g64|."""
import os

import numpy as np
import pytest
import torch

from oracle import smplx_oracle
from shapy_b200 import synth
from smplx_grad_ref import LEAVES, forward_differentiable, oracle_grads, pattern

pytestmark = pytest.mark.gpu
TOL = 1e-4
GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'ref_smplx_grad.npz')
PARTS = [('global_rot', 0, 1), ('body_pose', 1, 21), ('jaw_pose', 22, 1), ('leye_pose', 23, 1), ('reye_pose', 24, 1),
         ('left_hand_pose', 25, 15), ('right_hand_pose', 40, 15)]


def check(name, got, ref, tol=TOL):
    got, ref = got.detach().double().cpu(), torch.as_tensor(ref).double().cpu()
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    for b in range(ref.shape[0]):
        scale = float(ref[b].abs().max())
        err = float((got[b] - ref[b]).abs().max())
        assert err <= tol * scale + 1e-30, (name, b, err, scale)


def rodrigues(aa):
    aa = aa.double()
    th = aa.norm(dim=-1, keepdim=True)
    k = aa / th.clamp_min(1e-300)
    kx, ky, kz = k.unbind(-1)
    z = torch.zeros_like(kx)
    K = torch.stack([z, -kz, ky, kz, z, -kx, -ky, kx, z], -1).view(*aa.shape[:-1], 3, 3)
    s, c = th.sin()[..., None], th.cos()[..., None]
    return torch.eye(3, dtype=torch.float64) + s * K + (1 - c) * (K @ K)


@pytest.fixture(scope='module')
def model():
    return synth.make_smplx()


@pytest.fixture(scope='module')
def module(model):
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    return SMPLX(data_struct=model, use_face_contour=True).cuda()


def unwrap(t):
    return t[:] if not torch.is_tensor(t) else t


# ---------------------------------------------------------------------------------------- reference golden
def test_against_reference_golden(module):
    g = np.load(GOLDEN)
    B, V, K = g['betas'].shape[0], module.get_num_verts(), 123
    leaf = {k: torch.from_numpy(g[k]).float().cuda().requires_grad_(True) for k in LEAVES}
    kw = {name: leaf['rot'][:, j0:j0 + n] for name, j0, n in PARTS}
    out = module(betas=leaf['betas'], expression=leaf['expression'], transl=leaf['transl'], camera=leaf['camera'], **kw)
    loss = 0
    for name, shape in (('vertices', (B, V, 3)), ('joints', (B, K, 3)), ('v_shaped', (B, V, 3)),
                        ('proj_joints', (B, K, 2))):
        cot = torch.from_numpy(pattern(g, name, shape)).float().cuda()
        loss = loss + (unwrap(out[name]) * cot).sum()
    loss.backward()
    for k in LEAVES:
        check(k, leaf[k].grad, g[f'grad_{k}'])


# --------------------------------------------------------------------------------------- float64 oracle
def inputs(seed, B, n_rot, expr=True, camera=True):
    gen = torch.Generator().manual_seed(seed)
    rot = rodrigues(torch.randn(B, n_rot, 3, generator=gen, dtype=torch.float64) * 0.4).float()
    if n_rot > 15 and B > 1:                                 # necks turned past both ends of the contour LUT
        rot[0, 12] = rodrigues(torch.tensor([0.0, 1.2, 0.0])).float()
        rot[1, 12] = rodrigues(torch.tensor([0.0, -1.2, 0.0])).float()
    return dict(betas=torch.randn(B, 10, generator=gen), rot=rot,
                expression=torch.randn(B, 10, generator=gen) if expr else None,
                camera=(torch.randn(B, 3, generator=gen) * torch.tensor([3.0, 0.2, 0.2]) +
                        torch.tensor([1.0, 0.0, 0.0])) if camera else None)


def cotangents(kind, seed, B, V, K, m, camera):
    gen = torch.Generator().manual_seed(seed + 1)
    z = lambda *s: torch.zeros(*s)  # noqa: E731
    J, L = 55, m['lmk_faces_idx'].shape[0]
    if kind == 'mixed':
        c = dict(vertices=torch.randn(B, V, 3, generator=gen), joints=torch.randn(B, K, 3, generator=gen),
                 v_shaped=torch.randn(B, V, 3, generator=gen) * 0.5)
        if camera:
            c['proj_joints'] = torch.randn(B, K, 2, generator=gen)
        return c
    if kind == 'proj':
        p = z(B, K, 2)
        p[:, J + 3, 0] = 1.0
        return dict(proj_joints=p)
    j = z(B, K, 3)
    j14 = int(m['source_idxs'][0]) if 'source_idxs' in m else 8
    idx = {'joint': 20, 'j14': j14, 'dyn': min(J + L + 5, K - 1)}[kind]
    j[:, idx, 1] = 1.0
    return dict(joints=j)


def gpu_grads(packed, x, cot):
    from shapy_b200 import ops
    c = lambda t: None if t is None else t.cuda()  # noqa: E731
    return ops.smplx_backward(packed, c(x['betas']), c(x['rot']), expr=c(x['expression']), camera=c(x['camera']),
                              grad_vertices=c(cot.get('vertices')), grad_v_shaped=c(cot.get('v_shaped')),
                              grad_joints=c(cot.get('joints')), grad_proj_joints=c(cot.get('proj_joints')))


def compare_with_oracle(m, packed, x, cot, rows, use_face_contour=True):
    got = gpu_grads(packed, x, cot)
    sub = lambda t: None if t is None else t[rows]  # noqa: E731
    ref, _ = oracle_grads(m, {k: sub(v) for k, v in cot.items()}, sub(x['betas']), sub(x['rot']),
                          expression=sub(x['expression']), camera=sub(x['camera']), use_face_contour=use_face_contour)
    check('betas', got['betas'][rows], ref['betas'])
    check('rot', got['rot'][rows], ref['rot'])
    if x['expression'] is not None:
        check('expression', got['expr'][rows], ref['expression'])
    if x['camera'] is not None:
        check('camera', got['camera'][rows], ref['camera'])
    return got


@pytest.mark.parametrize('kind', ['joint', 'j14', 'dyn', 'proj', 'mixed'])
@pytest.mark.parametrize('n_rot', [1, 22, 25, 55])
@pytest.mark.parametrize('B', [1, 64, 4096])
def test_vs_float64_oracle(model, B, n_rot, kind):
    from shapy_b200 import ops
    packed = ops.SmplxModel(dict(model), 'cuda')
    x = inputs(1000 * n_rot + B, B, n_rot)
    cot = cotangents(kind, B + n_rot, B, packed.V, packed.K, model, True)
    rows = list(range(B)) if B <= 64 else [0, 1, 17, 1000, 2047, 3001, 4095]
    compare_with_oracle(model, packed, x, cot, rows)


@pytest.mark.parametrize('variant', ['no_expression', 'no_camera', 'no_j14', 'no_contour'])
@pytest.mark.parametrize('kind', ['j14', 'dyn', 'mixed'])
def test_vs_float64_oracle_variants(model, variant, kind):
    from shapy_b200 import ops
    m = dict(model)
    if variant == 'no_j14':
        for k in ('extra_joint_regressor', 'source_idxs', 'target_idxs'):
            m.pop(k)
    contour = variant != 'no_contour'
    packed = ops.SmplxModel(dict(m, use_face_contour=contour), 'cuda')
    x = inputs(7, 16, 22, expr=variant != 'no_expression', camera=variant != 'no_camera')
    cot = cotangents(kind, 3, 16, packed.V, packed.K, m, x['camera'] is not None)
    if kind == 'dyn' and not contour:          # no dynamic landmarks: a one-hot on the last static landmark
        cot['joints'] = torch.zeros(16, packed.K, 3)
        cot['joints'][:, packed.K - 1, 2] = 1.0
    compare_with_oracle(m, packed, x, cot, list(range(16)), use_face_contour=contour)


# --------------------------------------------------------------------------------------------- decoder
def test_decoder_backward_vs_float64():
    from shapy_b200 import ops
    gen = torch.Generator().manual_seed(3)
    raw = torch.randn(64, 6 * 22, generator=gen)
    raw[0, :6] = torch.tensor([1e-14, 1.0, 0.0, 0.5, 0.0, 0.2])     # first column below the 1e-12 clamp
    raw[1, :6] = torch.tensor([1.0, 2.0, 0.0, 0.0, 0.0, 0.0])       # second column parallel to the first
    g = torch.randn(64, 22, 3, 3, generator=gen)
    got = ops.decode_rot6d_backward(raw.cuda(), g.cuda())
    r64 = raw.double().requires_grad_(True)
    (smplx_oracle.decode_6d(r64) * g.double()).sum().backward()
    ok = torch.ones(64, dtype=torch.bool)
    ok[:2] = False
    check('raw', got[ok], r64.grad[ok], tol=1e-5)
    assert torch.isfinite(got).all()


def test_end_to_end_from_raw_6d(model, module):
    from shapy_b200.human_shape.models.common.pose_utils import ContinuousRotReprDecoder
    gen = torch.Generator().manual_seed(11)
    B = 8
    raw = (synth.mean_params()[:132] + 0.3 * torch.randn(B, 132, generator=gen)).cuda().requires_grad_(True)
    betas = torch.randn(B, 10, generator=gen).cuda().requires_grad_(True)
    dec = ContinuousRotReprDecoder(22).cuda()
    rot = dec(raw)
    assert rot.requires_grad
    out = module(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=betas)
    wj = torch.randn(B, 123, 3, generator=gen)
    wv = torch.randn(B, module.get_num_verts(), 3, generator=gen) * 0.01
    ws = torch.randn(B, module.get_num_verts(), 3, generator=gen) * 0.01
    loss = out['joints'].mul(wj.cuda()).sum() + (out['vertices'] * wv.cuda()).sum() + (out['v_shaped'] * ws.cuda()).sum()
    loss.backward()
    # float64 oracle: decoder + forward under autograd
    r64 = raw.detach().double().cpu().requires_grad_(True)
    b64 = betas.detach().double().cpu().requires_grad_(True)
    rot64 = smplx_oracle.decode_6d(r64)
    o = forward_differentiable(model, b64, rot64)
    ((o['joints'] * wj.double()).sum() + (o['vertices'] * wv.double()).sum() + (o['v_shaped'] * ws.double()).sum()
     ).backward()
    check('raw', raw.grad, r64.grad)
    check('betas', betas.grad, b64.grad)


# ------------------------------------------------------------------------------ determinism and no-grad path
def test_deterministic_and_batch_independent(model):
    from shapy_b200 import ops
    packed = ops.SmplxModel(dict(model), 'cuda')
    x = inputs(5, 64, 55)
    cot = cotangents('mixed', 5, 64, packed.V, packed.K, model, True)
    a, b = gpu_grads(packed, x, cot), gpu_grads(packed, x, cot)
    one = gpu_grads(packed, {k: None if v is None else v[17:18] for k, v in x.items()},
                    {k: v[17:18] for k, v in cot.items()})
    for k in ('betas', 'rot', 'expr', 'camera'):
        assert torch.equal(a[k], b[k]), k
        assert torch.equal(a[k][17:18], one[k]), k


def test_no_grad_path_unchanged(module):
    from shapy_b200._lib import lib
    x = inputs(9, 32, 22)
    kw = dict(global_rot=x['rot'][:, :1].cuda(), body_pose=x['rot'][:, 1:].cuda(), betas=x['betas'].cuda(),
              expression=x['expression'].cuda(), camera=x['camera'].cuda(), transl=torch.ones(32, 3).cuda())

    def run(requires_grad, grad_mode):
        args = {k: v.clone().requires_grad_(requires_grad) for k, v in kw.items()}
        torch.cuda.synchronize()
        n0 = lib().shapy_launch_count()
        with torch.set_grad_enabled(grad_mode):
            out = module(**args)
        torch.cuda.synchronize()
        return out, lib().shapy_launch_count() - n0

    base, n_base = run(False, True)
    for rg, gm in ((False, False), (True, False), (True, True)):
        out, n = run(rg, gm)
        assert n == n_base, (rg, gm, n, n_base)
        for k in ('vertices', 'v_shaped', 'proj_joints'):
            assert torch.equal(out[k].detach(), base[k]), (rg, gm, k)
        assert torch.equal(unwrap(out['joints']).detach(), unwrap(base['joints']))
        assert (out['vertices'].grad_fn is not None) == (rg and gm)


# ------------------------------------------------------------------------------------------------ fit
FIT = {}
# Fraction of the 256 bodies whose keypoint RMS error is under 1 cm after the default 600 Adam iterations (lr 0.05),
# set from the first run on an H100 80GB HBM3 (700 W): 0.035, with the median loss down 15.6x (median RMS 0.18 m).
# On the seeded synthetic model most bodies stall in a local minimum of the pose from the mean-pose start; the bar
# guards against regressions, it does not claim what a real SMPL-X model reaches.
RMS_BAR = 1e-2
FRAC_BAR = 0.03


def _targets(module, B, seed=31):
    gen = torch.Generator().manual_seed(seed)
    bstar = torch.randn(B, 10, generator=gen).clamp(-2, 2)
    raw = synth.mean_params()[:132] + 0.3 * torch.randn(B, 132, generator=gen)
    from shapy_b200 import ops
    with torch.no_grad():
        rot = ops.decode_rot6d(raw.cuda())
        kp = module(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=bstar.cuda())['joints'][:].clone()
    return kp


def _fit(module, kp, iterations=600):
    from shapy_b200.fit import fit_body_to_keypoints
    mean = synth.mean_params()
    B = kp.shape[0]
    init = {'global_rot': mean[:6].expand(B, 6), 'body_pose': mean[6:132].expand(B, 126)}
    return fit_body_to_keypoints(module, kp, iterations=iterations, init=init)


def test_fit_256_bodies(module):
    kp = _targets(module, 256)
    res = _fit(module, kp)
    start = _fit(module, kp, iterations=0)['loss']
    rms = ((res['keypoints'] - kp).pow(2).sum(-1).mean(1)).sqrt()
    frac = float((rms < RMS_BAR).float().mean())
    print('fit_keypoints_256', {'frac_rms_1cm': frac, 'median_loss': float(res['loss'].median()),
                                'median_start': float(start.median()), 'median_rms': float(rms.median())})
    FIT['res'], FIT['kp'] = res, kp
    assert torch.isfinite(res['loss']).all()
    assert float(res['loss'].median()) < 0.1 * float(start.median())
    assert frac >= FRAC_BAR, frac


def test_fit_8_bodies_alone_equal_their_batch_rows(module):
    if 'res' not in FIT:
        pytest.skip('needs test_fit_256_bodies')
    rows = [3, 40, 77, 101, 150, 199, 230, 255]
    res8 = _fit(module, FIT['kp'][rows].contiguous())
    for k in ('global_rot', 'body_pose', 'betas', 'transl'):
        assert torch.equal(res8[k], FIT['res'][k][rows]), k
