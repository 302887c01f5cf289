"""GPU: the 2D keypoint Levenberg-Marquardt step (shapy_fit_lm_keypoints_2d_step) against its NumPy restatement
(tests/kp2d_lm_oracle.py, pinned by tests/test_fit_lm_kp2d_cpu.py) at P = 7, 54, 55 (the 48 KB shared-memory opt-in)
and 96, and fit_body_to_keypoints_2d end to end on the synthetic SMPL-X: loss definition, monotone losses, no host
synchronisation, determinism, batch independence, time to quality against Adam, and robustness to outliers."""
import math

import numpy as np
import pytest
import torch

import kp2d_lm_oracle as o2
from shapy_b200 import synth

pytestmark = pytest.mark.gpu


def _bits(t):
    return t.contiguous().view(torch.int32)


def _rodrigues(aa):
    aa = aa.double()
    th = aa.norm(dim=-1, keepdim=True)
    k = aa / th.clamp_min(1e-300)
    kx, ky, kz = k.unbind(-1)
    z = torch.zeros_like(kx)
    K = torch.stack([z, -kz, ky, kz, z, -kx, -ky, kx, z], -1).view(*aa.shape[:-1], 3, 3)
    s, c = th.sin()[..., None], th.cos()[..., None]
    return torch.eye(3, dtype=torch.float64) + s * K + (1 - c) * (K @ K)


# ------------------------------------------------------------------------------------------------ step kernel
# (n_rot, nb): P = 3 n_rot + nb + 3 = 7, 54, 55 (twice) and 96; K: 2K = 2, 16 (the staging boundary), 18 and 254 rows
STEP_SHAPES = [(1, 1), (8, 27), (12, 16), (17, 1), (22, 27)]
STEP_K = [1, 8, 9, 127]
# (robust_sigma, pose_prior_weight, betas_weight)
TERMS = [(math.inf, 0.0, 0.0), (0.3, 0.5, 0.1)]


def _step_case(n_rot, nb, K, terms):
    """Six bodies with random Jacobians: body 0's trial hits its targets (accepted), body 1's state does and its trial
    is far (rejected), body 2 has a weighted NaN trial keypoint (rejected), 3 to 5 random.  With K >= 8 keypoint 7 has
    weight 0 and NaN targets, keypoints and rows in state and trial."""
    sigma, pw, bw = terms
    B, P = 6, 3 * n_rot + nb + 3
    gen = torch.Generator().manual_seed(1000 * n_rot + 10 * nb + K + (3 if pw else 0))
    rn = lambda *s: torch.randn(*s, generator=gen)  # noqa: E731
    rot = _rodrigues(rn(B, n_rot, 3).double() * 0.5).float()
    trot = (rot.double() @ _rodrigues(rn(B, n_rot, 3).double() * 0.05)).float()
    anchor = (rot.double() @ _rodrigues(rn(B, n_rot, 3).double() * 0.1)).float()
    betas = rn(B, nb)
    cam = rn(B, 3) * torch.tensor([0.5, 0.1, 0.1])
    tbetas, tcam = betas + 0.05 * rn(B, nb), cam + 0.01 * rn(B, 3)
    anchor[0], tbetas[0] = trot[0], 0.9 * betas[0]          # the priors favour body 0's trial and body 1's state too
    anchor[1], tbetas[1] = rot[1], 1.1 * betas[1]
    kp, jac = rn(B, K, 3), rn(B, 3 * K, P)
    tkp, tjac = kp + 0.05 * rn(B, K, 3), jac + 0.1 * rn(B, 3 * K, P)
    kp[0] = tkp[0] + 0.5
    tkp[1] = kp[1] + 0.5
    tg = torch.stack([torch.from_numpy(o2.project(kp[b].numpy(), cam[b].numpy())).float() for b in range(B)])
    tg += 0.05 * rn(B, K, 2)
    tg[0] = torch.from_numpy(o2.project(tkp[0].numpy(), tcam[0].numpy())).float()
    tg[1] = torch.from_numpy(o2.project(kp[1].numpy(), cam[1].numpy())).float()
    tkp[2, 0, 1] = float('nan')
    w = torch.rand(B, K, generator=gen) + 0.5
    if K >= 8:
        w[:, 7] = 0.0
        tg[:, 7] = float('nan')
        for t in (kp, tkp):
            t[:, 7] = float('nan')
        for t in (jac, tjac):
            t[:, 21:24] = float('nan')
    return dict(rot=rot, betas=betas, cam=cam, kp=kp, jac=jac, trot=trot, tbetas=tbetas, tcam=tcam, tkp=tkp,
                tjac=tjac, tg=tg, w=w, anchor=anchor, lam=torch.rand(B, generator=gen) + 0.01,
                sigma=sigma, pw=pw, bw=bw)


def _run_step(c, first):
    from shapy_b200 import ops
    B = c['rot'].shape[0]
    n = lambda t: t.numpy()  # noqa: E731
    kw = dict(sigma=c['sigma'], pose_w=c['pw'], betas_w=c['bw'])
    s_np = []
    for b in range(B):
        s = {'rot': n(c['rot'][b]), 'betas': n(c['betas'][b]), 'camera': n(c['cam'][b]), 'keypoints': n(c['kp'][b]),
             'jac': n(c['jac'][b]), 'lambda': n(c['lam'][b]), 'accepted': 0}
        s['loss'] = np.float32(o2.loss(n(c['tg'][b]), n(c['w'][b]), s['keypoints'], s['camera'], c['sigma'], s['rot'],
                                       n(c['anchor'][b]), c['pw'], s['betas'], c['bw']))
        s_np.append(s)
    cu = lambda t: t.cuda().contiguous()  # noqa: E731
    state = {'rot': cu(c['rot']), 'betas': cu(c['betas']), 'camera': cu(c['cam']), 'keypoints': cu(c['kp']),
             'jac': cu(c['jac']), 'loss': cu(torch.tensor(np.array([s['loss'] for s in s_np]))),
             'lambda': cu(c['lam']), 'accepted': torch.zeros(B, dtype=torch.int32, device='cuda')}
    trial = {'rot': cu(c['trot']), 'betas': cu(c['tbetas']), 'camera': cu(c['tcam'])}
    ops.fit_lm_keypoints_2d_step(state, trial, cu(c['tg']), cu(c['w']), c['sigma'], c['pw'], c['bw'], 10.0, 3.0, first,
                                 cu(c['tkp']), cu(c['tjac']), pose_anchor=cu(c['anchor']))
    got = {k: v.cpu().numpy() for k, v in state.items()}
    nxt = {k: v.cpu().numpy() for k, v in trial.items()}
    flags, worst = [], 0.0
    for b in range(B):
        tr = {'rot': n(c['trot'][b]), 'betas': n(c['tbetas'][b]), 'camera': n(c['tcam'][b])}
        new, want, acc = o2.lm_keypoints_2d_step(s_np[b], n(c['tg'][b]), n(c['w'][b]), 10.0, 3.0, first, tr,
                                                 n(c['tkp'][b]), n(c['tjac'][b]), anchor=n(c['anchor'][b]), **kw)
        flags.append(acc)
        assert got['accepted'][b] == new['accepted'], b
        # softplus' exp / log1p may round differently on the device: loss and lambda to fp32 rounding
        assert np.isclose(got['lambda'][b], new['lambda'], rtol=3e-7, atol=0), (b, got['lambda'][b], new['lambda'])
        assert np.isclose(got['loss'][b], new['loss'], rtol=3e-7, atol=0, equal_nan=True), (b, got['loss'][b],
                                                                                          new['loss'])
        for k in ('rot', 'betas', 'camera', 'keypoints', 'jac'):
            assert np.array_equal(got[k][b], new[k], equal_nan=True), (b, k)
        for k in ('rot', 'betas', 'camera'):
            bar = 2e-6 * max(1.0, np.abs(want[k]).max())
            err = np.abs(nxt[k][b] - want[k]).max()
            assert err <= bar, (b, k, err)
            worst = max(worst, err / bar)
    if first:
        assert all(flags)
    else:
        assert flags[:3] == [True, False, False], flags
    return worst


@pytest.mark.parametrize('terms', TERMS, ids=['lsq', 'robust_priors'])
@pytest.mark.parametrize('first', [False, True])
@pytest.mark.parametrize('K', STEP_K)
@pytest.mark.parametrize('n_rot,nb', STEP_SHAPES)
def test_step_kernel_vs_oracle(n_rot, nb, K, first, terms):
    worst = _run_step(_step_case(n_rot, nb, K, terms), first)
    print(f'[kp2d] step P={3 * n_rot + nb + 3} K={K} first={first} terms={terms}: trial error / bar {worst:.3f}')


def test_argument_errors_raise_before_any_launch():
    from shapy_b200 import _lib, ops
    from shapy_b200.fit import fit_body_to_keypoints_2d
    L = _lib.lib()
    z = lambda *s: torch.zeros(*s, device='cuda')  # noqa: E731
    B, K, n_rot, nb = 2, 5, 22, 10
    P = 3 * n_rot + nb + 3
    st = {'rot': z(B, n_rot, 3, 3), 'betas': z(B, nb), 'camera': z(B, 3), 'keypoints': z(B, K, 3),
          'jac': z(B, 3 * K, P), 'loss': z(B), 'lambda': z(B), 'accepted': torch.zeros(B, dtype=torch.int32,
                                                                                     device='cuda')}
    tr = {'rot': z(B, n_rot, 3, 3), 'betas': z(B, nb), 'camera': z(B, 3)}
    anchor = z(B, n_rot, 3, 3)

    def step(sigma=1.0, pw=0.0, bw=0.0, up=10.0, down=3.0, anc=anchor, n_rot=n_rot, null_jac=False):
        P = 3 * n_rot + nb + 3
        p = [_lib.ptr(st[k]) for k in ('rot', 'betas', 'camera', 'keypoints')] + \
            [None if null_jac else _lib.ptr(z(B, 3 * K, P))] + [_lib.ptr(st[k]) for k in ('loss', 'lambda', 'accepted')]
        return L.shapy_fit_lm_keypoints_2d_step(B, K, n_rot, nb, _lib.ptr(z(B, K, 2)), _lib.ptr(z(B, K)),
                                                _lib.ptr(anc) if anc is not None else None, sigma, pw, bw, up, down,
                                                1, *p, _lib.ptr(tr['rot']), _lib.ptr(tr['betas']),
                                                _lib.ptr(tr['camera']), _lib.ptr(z(B, K, 3)), _lib.ptr(z(B, 3 * K, P)),
                                                None)
    torch.cuda.synchronize()
    n0 = L.shapy_launch_count()
    for kw in (dict(sigma=0.0), dict(sigma=-1.0), dict(sigma=float('nan')), dict(pw=-1.0), dict(bw=-0.5),
               dict(up=0.5), dict(down=0.9), dict(pw=1.0, anc=None), dict(null_jac=True), dict(n_rot=0)):
        assert step(**kw) == -1, kw
    assert step(n_rot=30) == -3                    # P = 103 > 96
    with pytest.raises(ValueError):
        ops.fit_lm_keypoints_2d_step(st, tr, z(B, K, 2), z(B, K), 0.0, 0.0, 0.0, 10.0, 3.0, True, z(B, K, 3),
                                     z(B, 3 * K, P))
    with pytest.raises(ValueError):
        ops.fit_lm_keypoints_2d_step(st, tr, z(B, K, 2), z(B, K), None, 1.0, 0.0, 10.0, 3.0, True, z(B, K, 3),
                                     z(B, 3 * K, P))
    for kw in (dict(robust_sigma=0.0), dict(pose_prior_weight=-1.0), dict(betas_weight=-1.0), dict(method='gn')):
        with pytest.raises(ValueError):
            fit_body_to_keypoints_2d(None if 'method' in kw else _FakeModel(), z(B, 123, 2), **kw)
    for bad in (z(123, 2), z(2, 123), z(2, 123, 3)):       # not (B, K, 2)
        with pytest.raises(ValueError):
            fit_body_to_keypoints_2d(_FakeModel(), bad)
    st0 = {k: v[:0].contiguous() for k, v in st.items()}
    tr0 = {k: v[:0].contiguous() for k, v in tr.items()}
    ops.fit_lm_keypoints_2d_step(st0, tr0, z(0, K, 2), z(0, K), None, 0.0, 0.0, 10.0, 3.0, True, z(0, K, 3),
                                 z(0, 3 * K, P))
    assert L.shapy_launch_count() == n0


class _FakeModel:
    num_betas = 10
    shapedirs = torch.zeros(1)


# ------------------------------------------------------------------------------------------------ fit
def _model(variant):
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    m = dict(synth.make_smplx())
    if variant == 'no_contour_no_j14':
        for k in ('extra_joint_regressor', 'source_idxs', 'target_idxs'):
            m.pop(k)
        return SMPLX(data_struct=m, use_face_contour=False).cuda()
    return SMPLX(data_struct=m, use_face_contour=True).cuda()


_MODELS = {}


def _get(variant='full'):
    if variant not in _MODELS:
        _MODELS[variant] = _model(variant)
    return _MODELS[variant]


def _problem(module, B, seed=41):
    """Ground truth: betas ~ N(0, 1) clipped to 2, raw pose = mean + 0.3 N(0, 1), a random camera; targets its
    projected keypoints; the start a perturbed copy standing in for a regressor's prediction."""
    from shapy_b200 import ops
    gen = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=gen)  # noqa: E731
    bstar = rn(B, module.num_betas).clamp(-2, 2)
    raw = synth.mean_params()[:132] + 0.3 * rn(B, 132)
    cam = torch.stack([1.0 + 0.2 * rn(B), 0.1 * rn(B), 0.1 * rn(B)], 1)
    with torch.no_grad():
        rot = ops.decode_rot6d(raw.cuda())
        out = module(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=bstar.cuda(), camera=cam.cuda())
    init = {'global_rot': (raw[:, :6] + 0.1 * rn(B, 6)).cuda(), 'body_pose': (raw[:, 6:] + 0.1 * rn(B, 126)).cuda(),
            'betas': (bstar + 0.5 * rn(B, module.num_betas)).cuda(), 'camera': (cam + 0.05 * rn(B, 3)).cuda()}
    return out['proj_joints'].clone(), out['joints'][:].clone(), init


def _rms2d(res, x, w=None):
    d = (res['proj_joints'] - x).pow(2).sum(-1)
    if w is None:
        return d.mean(1).sqrt()
    return ((d * w).sum(1) / w.sum(1)).sqrt()


def _lm_loop(module, x, w, init, iterations, sigma=None, pw=0.0, bw=0.0):
    """The LM loop of fit_body_to_keypoints_2d written out, keeping every iteration's state loss."""
    from shapy_b200 import ops
    from shapy_b200.fit import LM_DOWN, LM_UP
    packed = module.packed(x.device)
    B, K = x.shape[:2]
    nb = init['betas'].shape[1]
    P = 3 * 22 + nb + 3
    rot0 = ops.decode_rot6d(torch.cat([init['global_rot'], init['body_pose']], 1)).contiguous()
    trial = {'rot': rot0.clone(), 'betas': init['betas'].clone().contiguous(), 'camera': init['camera'].clone()}
    mk = lambda *s: torch.empty(*s, device='cuda')  # noqa: E731
    state = {'rot': mk(B, 22, 3, 3), 'betas': mk(B, nb), 'camera': mk(B, 3), 'keypoints': mk(B, K, 3),
             'jac': mk(B, 3 * K, P), 'loss': mk(B), 'lambda': mk(B),
             'accepted': torch.zeros(B, dtype=torch.int32, device='cuda')}
    losses = []
    for it in range(iterations + 1):
        tkp, tjac = ops.smplx_keypoint_jacobian(packed, trial['betas'], trial['rot'])
        ops.fit_lm_keypoints_2d_step(state, trial, x, w, sigma, pw, bw, LM_UP, LM_DOWN, it == 0, tkp, tjac,
                                     pose_anchor=rot0 if pw > 0 else None)
        losses.append(state['loss'].clone())
    return state, torch.stack(losses)


@pytest.mark.parametrize('variant', ['full', 'no_contour_no_j14'])
def test_lm_loss_definition_and_monotone_losses(variant):
    """At sigma = inf without priors the kernel's loss equals sum w |proj_joints - x|^2 of shapy_smplx_forward's
    proj_joints (fp32 rounding); with a robust loss and priors every body's loss is non-increasing at every iteration,
    and fit_body_to_keypoints_2d's returned loss is the kernel's."""
    from shapy_b200 import ops
    from shapy_b200.fit import fit_body_to_keypoints_2d
    module = _get(variant)
    x, _, init = _problem(module, 64, seed=5)
    w = (torch.rand(64, x.shape[1], generator=torch.Generator().manual_seed(6)) + 0.5).cuda()
    w[:, 3] = 0.0
    x[:, 3] = float('nan')
    state, losses = _lm_loop(module, x, w, init, 0)
    out = ops.smplx_forward(module.packed(x.device), state['betas'], state['rot'], camera=state['camera'],
                            want_v_shaped=False)
    keep = w > 0
    d = torch.where(keep[..., None], out['proj_joints'] - torch.where(keep[..., None], x, 0.0), 0.0)
    ref = (w * d.double().pow(2).sum(-1)).sum(1)
    rel = ((state['loss'].double() - ref).abs() / ref).max()
    print(f'[kp2d] {variant}: loss vs forward proj_joints, max relative {float(rel):.2e}')
    assert float(rel) <= 1e-5
    for sigma, pw, bw in ((None, 0.0, 0.0), (0.05, 0.5, 0.01)):
        state, losses = _lm_loop(module, x, w, init, 20, sigma, pw, bw)
        assert bool(torch.isfinite(losses).all())
        assert bool((losses[1:] <= losses[:-1]).all())
        ratio = float(losses[-1].median()) / float(losses[0].median())
        print(f'[kp2d] {variant} sigma={sigma}: median loss after 20 iterations / start {ratio:.3f}')
        assert ratio < 0.5                   # first run on an H100: 0.000 to 0.310
    res = fit_body_to_keypoints_2d(module, x, w, init=init, method='lm', iterations=20, robust_sigma=0.05,
                                   pose_prior_weight=0.5, betas_weight=0.01)
    for k in ('betas', 'camera'):
        assert torch.equal(_bits(res[k]), _bits(state[k])), k
    # the returned loss comes from SMPLX.forward's proj_joints, the kernel's from the Jacobian launch's keypoints
    assert float(((res['loss'] - state['loss']).abs() / state['loss']).max()) <= 1e-2
    assert res['proj_joints'].shape == x.shape and res['keypoints'].shape == (64, x.shape[1], 3)


def test_lm_loop_never_synchronises():
    from shapy_b200.fit import fit_body_to_keypoints_2d
    module = _get()
    x, _, init = _problem(module, 32, seed=7)
    fit_body_to_keypoints_2d(module, x, init=init, method='lm', iterations=1, robust_sigma=0.1,
                             pose_prior_weight=1.0)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        res = fit_body_to_keypoints_2d(module, x, init=init, method='lm', iterations=3, robust_sigma=0.1,
                                       pose_prior_weight=1.0, betas_weight=0.01)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert res['betas'].shape == (32, 10)


def test_lm_deterministic_and_batch_independent():
    from shapy_b200.fit import fit_body_to_keypoints_2d
    module = _get()
    x, _, init = _problem(module, 64, seed=8)
    kw = dict(method='lm', iterations=15, robust_sigma=0.1, pose_prior_weight=0.5)
    r1 = fit_body_to_keypoints_2d(module, x, init=init, **kw)
    r2 = fit_body_to_keypoints_2d(module, x, init=init, **kw)
    rows = [0, 5, 17, 33, 63]
    r8 = fit_body_to_keypoints_2d(module, x[rows].contiguous(), init={k: v[rows].contiguous() for k, v in init.items()},
                                  **kw)
    for k in ('global_rot', 'body_pose', 'betas', 'camera', 'loss'):
        assert torch.equal(_bits(r1[k]), _bits(r2[k])), k
        assert torch.equal(_bits(r8[k]), _bits(r1[k][rows])), k


def test_init_from_the_regressor_stage_output():
    """The regressor's stage dict (raw_global_rot, raw_body_pose, decoded matrices, betas, camera) works as-is."""
    from shapy_b200 import ops
    from shapy_b200.fit import fit_body_to_keypoints_2d
    module = _get()
    x, _, init = _problem(module, 8, seed=9)
    raw = torch.cat([init['global_rot'], init['body_pose']], 1)
    rot = ops.decode_rot6d(raw)
    stage = {'raw_global_rot': init['global_rot'], 'raw_body_pose': init['body_pose'], 'global_rot': rot[:, :1],
             'body_pose': rot[:, 1:], 'betas': init['betas'], 'camera': init['camera']}
    a = fit_body_to_keypoints_2d(module, x, init=stage, method='lm', iterations=3)
    b = fit_body_to_keypoints_2d(module, x, init=init, method='lm', iterations=3)
    assert torch.equal(_bits(a['betas']), _bits(b['betas'])) and torch.equal(_bits(a['camera']), _bits(b['camera']))


# Time to quality, 256 bodies, LM(50) against Adam(600); bars set just below / above the first run on an H100 80GB
# HBM3 (700 W): LM 29.7 % of the bodies within the RMS threshold and a median root-aligned joint error of 0.192 m,
# Adam(600) 0 % and 0.238 m (README.md).
RMS_THRESHOLD = 2e-3             # 2D RMS in the crop frame ([-1, 1] over the crop: ~0.26 px of a 256 px crop)
LM_FRAC_BAR = 0.28
LM_MPJPE_BAR = 0.20


def test_time_to_quality_256_bodies_vs_adam():
    from shapy_b200.fit import fit_body_to_keypoints_2d
    from shapy_b200.metrics import PointError, build_alignment
    module = _get()
    x, joints, init = _problem(module, 256)
    lm = fit_body_to_keypoints_2d(module, x, init=init, method='lm')
    adam = fit_body_to_keypoints_2d(module, x, init=init)
    pe = PointError(build_alignment('root'))
    frac, mpjpe = {}, {}
    for k, r in (('lm', lm), ('adam', adam)):
        frac[k] = float((_rms2d(r, x) < RMS_THRESHOLD).float().mean())
        pe(r['keypoints'].contiguous(), joints)
        mpjpe[k] = float(pe.last_mean.median())
    print('fit_keypoints_2d_256', {'frac_rms2d': frac, 'median_root_mpjpe_m': mpjpe,
                                   'median_rms2d': {k: float(_rms2d(r, x).median()) for k, r in (('lm', lm),
                                                                                                  ('adam', adam))}})
    assert frac['lm'] >= LM_FRAC_BAR and mpjpe['lm'] <= LM_MPJPE_BAR
    assert frac['lm'] >= frac['adam']


def test_robust_fit_beats_least_squares_on_outliers():
    """10 % of the keypoints moved by 0.3 in the crop frame: the Geman-McClure fit's inlier RMS beats the
    least-squares fit's."""
    from shapy_b200.fit import fit_body_to_keypoints_2d
    module = _get()
    x, _, init = _problem(module, 128, seed=43)
    gen = torch.Generator().manual_seed(44)
    out = (torch.rand(x.shape[:2], generator=gen) < 0.1).cuda()
    xo = torch.where(out[..., None], x + 0.3 * torch.randn(x.shape, generator=gen).cuda(), x)
    inl = (~out).float()
    rms = {}
    for name, sigma in (('lsq', None), ('robust', 0.02)):
        r = fit_body_to_keypoints_2d(module, xo, init=init, method='lm', robust_sigma=sigma, pose_prior_weight=0.01)
        rms[name] = float(_rms2d(r, x, inl).median())
    print('fit_keypoints_2d_outliers, median inlier RMS', rms)
    assert rms['robust'] < rms['lsq']          # first run: 0.0103 against 0.216


def test_keypoint_jacobian_2d_vs_oracle_and_forward():
    """fit.keypoint_jacobian_2d against the float64 restatement's projection of the same 3D Jacobian, and its
    proj_joints against SMPLX.forward's."""
    from shapy_b200 import ops
    from shapy_b200.fit import keypoint_jacobian, keypoint_jacobian_2d
    module = _get()
    gen = torch.Generator().manual_seed(50)
    B = 8
    rot = _rodrigues(torch.randn(B, 22, 3, generator=gen, dtype=torch.float64) * 0.4).float().cuda()
    betas = torch.randn(B, 10, generator=gen).cuda()
    cam = (torch.randn(B, 3, generator=gen) * torch.tensor([3.0, 0.2, 0.2])).cuda()
    cam[0, 0] = 25.0                                       # past softplus' threshold
    res = keypoint_jacobian_2d(module, rot, betas, cam)
    r3 = keypoint_jacobian(module, rot, betas)
    fwd = ops.smplx_forward(module.packed(), betas, rot, camera=cam, want_v_shaped=False)['proj_joints']
    K = r3['keypoints'].shape[1]
    assert res['jacobian'].shape == (B, 2 * K, 79) and res['proj_joints'].shape == (B, K, 2)
    for b in range(B):
        kp, j3, c = (r3['keypoints'][b].double().cpu().numpy(), r3['jacobian'][b].double().cpu().numpy(),
                     cam[b].double().cpu().numpy())
        want = o2.jacobian_2d(kp, j3, c)
        got = res['jacobian'][b].double().cpu().numpy()
        assert np.abs(got - want).max() <= 1e-6 * np.abs(want).max(), b
        assert np.abs(res['proj_joints'][b].double().cpu().numpy() - o2.project(kp, c)).max() <= 1e-6 * max(
            1.0, np.abs(o2.project(kp, c)).max()), b
    rel = ((res['proj_joints'] - fwd).abs().amax((1, 2)) / fwd.abs().amax((1, 2))).max()
    assert float(rel) <= 2e-6


def test_cli_fits_raw_openpose_detections(tmp_path):
    """python -m shapy_b200.fit --keypoints-2d with img_00's raw OpenPose detections, its crop descriptor and the
    OpenPose -> SMPL-X map, started from SHAPY's img_00 prediction (on the synthetic model)."""
    import os
    from shapy_b200 import fit
    from shapy_b200 import keypoints2d as k2d
    g = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
    ref = np.load(os.path.join(g, 'ref_openpose.npz'))
    kmap_path = os.path.join(g, 'openpose_smplx_map.json')
    row = int(np.nonzero(ref['file_index'] == [str(f) for f in ref['files']].index('img_00.json'))[0][0])
    raw = ref['raw'][row:row + 1]
    center, scale = k2d.bbox_from_keypoints(k2d.threshold_confidence(raw, k2d.load_keypoint_map(kmap_path)))
    np.savez(tmp_path / 'kp.npz', openpose=raw, center=center, scale=scale)
    body = np.load(os.path.join(g, 'img00_body.npz'))
    np.savez(tmp_path / 'pred.npz', **{k: body[k] for k in ('raw_global_rot', 'raw_body_pose', 'betas', 'camera')})
    out = tmp_path / 'fit.npz'
    fit.main(['--synthetic', '--keypoints-2d', str(tmp_path / 'kp.npz'), '--keypoint-map', kmap_path, '--init',
              str(tmp_path / 'pred.npz'), '--method', 'lm', '--iterations', '10', '--robust-sigma', '0.05',
              '--pose-prior-weight', '1.0', '--output', str(out)])
    r = np.load(out)
    K = r['keypoints'].shape[1]                              # the CLI's synthetic model has no face contour
    assert r['proj_joints'].shape == (1, K, 2) and np.isfinite(r['loss']).all() and np.isfinite(r['camera']).all()
