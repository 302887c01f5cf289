"""GPU: the whole-body 2D fit.  The expression-aware keypoint Jacobian (shapy_smplx_keypoint_jacobian_expr) against
the 22-joint launch at psi = 0, the float64 restatement and the forward, on every model shape; the wide LM step
(shapy_fit_lm_keypoints_2d_expressive_step and its perspective entry) against tests/kp2d_lm_oracle.py at P = 7 to 200,
bit for bit against today's 2D steps at n_rot = 22 without expression over a 50-iteration loop, its argument errors;
and fit_body_to_keypoints_2d(pose_width=55, fit_expression=True) end to end: launches, no host synchronisation,
monotone losses, determinism, batch independence, Adam, the command line and quality."""
import time

import numpy as np
import pytest
import torch

import kp2d_lm_oracle as o2
import kp_lm_oracle
import lm_harness as harness
from lm_harness import TOL, VARIANTS, bits, variant_model
from shapy_b200 import synth

pytestmark = pytest.mark.gpu

F, PP = harness.F, harness.PP


# ------------------------------------------------------------------------------------------------ Jacobian
_PACKED = {}


def _packed(name):
    from shapy_b200 import ops
    if name not in _PACKED:
        _PACKED[name] = ops.SmplxModel(dict(variant_model(name), use_face_contour=True), 'cuda')
    return _PACKED[name]


@pytest.mark.parametrize('n_rot', [22, 25, 40, 55])
@pytest.mark.parametrize('name', [n for n in VARIANTS if VARIANTS[n][1] > 0])
def test_jacobian_expr(name, n_rot):
    from shapy_b200 import ops
    m, pk = variant_model(name), _packed(name)
    NB, NE, _ = VARIANTS[name]
    B = 3
    x = harness.inputs(500 * NB + n_rot, B, n_rot, NB, NE)
    betas, rot, transl = x['betas'].cuda(), x['rot'].cuda(), x['transl'].cuda()
    expr = x['expression'].cuda()
    # psi = 0: the keypoints and every shared column are the 22-joint launch's bits
    kp0, jac0 = ops.smplx_keypoint_jacobian(pk, betas, rot, transl)
    kpz, jacz = ops.smplx_keypoint_jacobian(pk, betas, rot, transl, expr=torch.zeros_like(expr))
    P0 = 3 * n_rot + NB
    assert jacz.shape == (B, 3 * pk.K, P0 + NE + 3)
    assert torch.equal(bits(kp0), bits(kpz))
    assert torch.equal(bits(jac0[..., :P0]), bits(jacz[..., :P0]))
    assert torch.equal(bits(jac0[..., P0:]), bits(jacz[..., P0 + NE:]))
    # psi != 0: every column against the float64 restatement, the keypoints against the forward
    kp, jac = ops.smplx_keypoint_jacobian(pk, betas, rot, transl, expr=expr)
    out = ops.smplx_forward(pk, betas, rot, expr=expr, want_vertices=True, want_v_shaped=False, want_joints=True)
    fj = out['joints'] + transl[:, None]
    assert float((kp - fj).abs().max()) <= 1e-5 * float(fj.abs().max())
    kp, jac = kp.double().cpu().numpy(), jac.double().cpu().numpy()
    worst = 0.0
    for b in range(B):
        k64, j64 = kp_lm_oracle.keypoint_jacobian(m, x['betas'][b], x['rot'][b], x['transl'][b],
                                                  expr=x['expression'][b])
        assert np.abs(kp[b] - k64).max() <= 1e-5 * np.abs(k64).max(), b
        for block, cols in (('rot', slice(0, 3 * n_rot)), ('betas', slice(3 * n_rot, P0)),
                            ('expression', slice(P0, P0 + NE))):
            err, scale = np.abs(jac[b][:, cols] - j64[:, cols]).max(), np.abs(j64[:, cols]).max()
            assert err <= TOL * scale, (b, block, err, scale)
            worst = max(worst, err / (TOL * scale))
        assert np.array_equal(jac[b][:, P0 + NE:], np.tile(np.eye(3), (pk.K, 1)))
    print(f'[expressive] jacobian {name} n_rot={n_rot}: worst error / bar {worst:.3f}')


def test_jacobian_expr_needs_an_expression_basis():
    from shapy_b200 import ops
    pk = _packed('nb10_ne0')
    z = torch.zeros(1, 10, device='cuda')
    with pytest.raises(RuntimeError):
        ops.smplx_keypoint_jacobian(pk, z, torch.eye(3, device='cuda').expand(1, 22, 3, 3).contiguous(),
                                    expr=torch.zeros(1, 0, device='cuda'))


# ------------------------------------------------------------------------------------------------ step kernel
# (n_rot, nb, ne): P = 7, 79 (n_rot 22), 96, 97, 188 and 200
STEP_SHAPES = [(1, 1, 0), (22, 10, 0), (22, 10, 10), (27, 6, 6), (27, 7, 6), (55, 10, 10), (55, 27, 5),
               (55, 16, 16)]
STEP_K = [9, 127]


@pytest.mark.parametrize('persp', [False, True], ids=['weak', 'persp'])
@pytest.mark.parametrize('terms', range(3), ids=['lsq', 'robust_joint_priors', 'robust_scalar_prior'])
@pytest.mark.parametrize('first', [False, True])
@pytest.mark.parametrize('K', STEP_K)
@pytest.mark.parametrize('n_rot,nb,ne', STEP_SHAPES)
def test_step_kernel_vs_oracle(n_rot, nb, ne, K, first, terms, persp):
    """The wide step on lm_harness.kp2d_case with ne expression columns; terms indexes lm_harness.EXPR_TERMS."""
    t = harness.EXPR_TERMS['persp' if persp else 'weak'][terms]
    worst = harness.kp2d_run(first, n_rot=n_rot, nb=nb, K=K, terms=t, persp=persp, ne=ne)
    print(f'[expressive] step P={3 * n_rot + nb + ne + 3} K={K} first={first} terms={t} persp={persp}: trial '
          f'error / bar {worst:.3f}')


def test_step_errors():
    from shapy_b200 import _lib, ops
    L = _lib.lib()
    B, K = 2, 9
    z = lambda *s: torch.zeros(*s, device='cuda')  # noqa: E731

    def mk(n_rot, nb, ne):
        n_rot, ne = max(n_rot, 1), max(ne, 0)
        P = 3 * n_rot + nb + ne + 3
        st = {'rot': z(B, n_rot, 3, 3), 'betas': z(B, nb), 'expression': z(B, ne), 'camera': z(B, 3),
              'keypoints': z(B, K, 3), 'jac': z(B, 3 * K, P), 'loss': z(B), 'lambda': z(B),
              'accepted': torch.zeros(B, dtype=torch.int32, device='cuda')}
        tr = {'rot': z(B, n_rot, 3, 3), 'betas': z(B, nb), 'expression': z(B, ne), 'camera': z(B, 3)}
        return st, tr, z(B, K, 3), z(B, 3 * K, P)

    def raw(n_rot=22, nb=10, ne=10, sigma=1.0, pw=0.0, bw=0.0, ew=0.0, up=10.0, down=3.0, anc=True, jw=False,
            null_expr=False):
        st, tr, tkp, tjac = mk(n_rot, nb, ne)
        p = _lib.ptr
        anchor = z(B, n_rot, 3, 3)
        e = (lambda t: None) if null_expr else p  # noqa: E731
        return L.shapy_fit_lm_keypoints_2d_expressive_step(
            B, K, n_rot, nb, ne, p(z(B, K, 2)), p(z(B, K)), p(anchor) if anc else None, p(z(n_rot)) if jw else None,
            sigma, pw, bw, ew, up, down, 1, p(st['rot']), p(st['betas']), e(st['expression']), p(st['camera']),
            p(st['keypoints']), p(st['jac']), p(st['loss']), p(st['lambda']), p(st['accepted']), p(tr['rot']),
            p(tr['betas']), e(tr['expression']), p(tr['camera']), p(tkp), p(tjac), _lib.stream_ptr())

    torch.cuda.synchronize()
    n0 = L.shapy_launch_count()
    for kw in (dict(sigma=0.0), dict(sigma=float('nan')), dict(pw=-1.0), dict(bw=-0.5), dict(ew=-1.0),
               dict(up=0.5), dict(down=0.9), dict(pw=1.0, anc=False), dict(jw=True, anc=False), dict(null_expr=True),
               dict(n_rot=0), dict(ne=-1)):
        assert raw(**kw) == -1, kw
    assert raw(n_rot=55, nb=16, ne=17) == -3                  # P = 201
    assert L.shapy_launch_count() == n0
    assert raw(n_rot=55, nb=16, ne=16) == 0                   # P = 200
    assert raw(n_rot=22, nb=10, ne=0, null_expr=True) == 0    # no expression: no expression arrays
    torch.cuda.synchronize()
    st, tr, tkp, tjac = mk(22, 10, 10)
    with pytest.raises(ValueError):
        ops.fit_lm_keypoints_2d_expressive_step(st, tr, z(B, K, 2), z(B, K), None, 0.0, 0.0, 0.0, 10.0, 3.0, True,
                                                tkp, tjac, pose_anchor=z(B, 22, 3, 3), joint_weights=torch.ones(22))
    with pytest.raises(ValueError):
        ops.fit_lm_keypoints_2d_expressive_step(st, tr, z(B, K, 2), z(B, K), None, 0.0, 0.0, -1.0, 10.0, 3.0, True,
                                                tkp, tjac)
    with pytest.raises(RuntimeError):
        ops.fit_lm_keypoints_2d_expressive_step(st, tr, z(B, K, 2), z(B, K), None, 0.0, 0.0, 0.0, 10.0, 3.0, True,
                                                tkp, tjac[..., 1:])
    st, tr, tkp, tjac = mk(55, 16, 17)
    with pytest.raises(RuntimeError, match='at most 200'):
        ops.fit_lm_keypoints_2d_expressive_step(st, tr, z(B, K, 2), z(B, K), None, 0.0, 0.0, 0.0, 10.0, 3.0, True,
                                                tkp, tjac)


# ------------------------------------------------------------------------------------------------ fits
def _problem(module, B, seed=41, persp=False):
    """The 2D recipe's ground truth (betas, raw body pose, camera or translation) plus hands (raw 6D = identity + 0.3
    N), jaw (identity + 0.2 N) and psi ~ N(0, 1); targets the exact projections of every keypoint; the start the
    recipe's perturbed one with hands and jaw at identity and psi = 0."""
    from shapy_b200 import ops
    gen = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=gen)  # noqa: E731
    ident = torch.tensor([1.0, 0.0, 0.0, 1.0, 0.0, 0.0])
    bstar = rn(B, module.num_betas).clamp(-2, 2)
    raw = synth.mean_params()[:132] + 0.3 * rn(B, 132)
    jaw = ident + 0.2 * rn(B, 6)
    lh, rh = ident.repeat(15) + 0.3 * rn(B, 90), ident.repeat(15) + 0.3 * rn(B, 90)
    psi = rn(B, module.num_expression_coeffs)
    with torch.no_grad():
        full = torch.cat([raw, jaw, ident.repeat(B, 2), lh, rh], 1).cuda()
        rot = ops.decode_rot6d(full)
        kw = dict(global_rot=rot[:, :1], body_pose=rot[:, 1:22], jaw_pose=rot[:, 22:23], leye_pose=rot[:, 23:24],
                  reye_pose=rot[:, 24:25], left_hand_pose=rot[:, 25:40], right_hand_pose=rot[:, 40:55],
                  betas=bstar.cuda(), expression=psi.cuda())
        if persp:
            tr = torch.stack([0.2 * rn(B), 0.2 * rn(B), 4.0 + rn(B).abs()], 1).cuda()
            out = module(transl=tr, **kw)
            j = out['joints'][:]
            x = F * j[..., :2] / j[..., 2:] + torch.tensor(PP, device='cuda')
            last = ('transl', tr + torch.cat([0.05 * rn(B, 2), 0.2 * rn(B, 1)], 1).cuda())
        else:
            cam = torch.stack([1.0 + 0.2 * rn(B), 0.1 * rn(B), 0.1 * rn(B)], 1).cuda()
            out = module(camera=cam, **kw)
            x = out['proj_joints']
            last = ('camera', cam + 0.05 * rn(B, 3).cuda())
    init = {'global_rot': (raw[:, :6] + 0.1 * rn(B, 6)).cuda(), 'body_pose': (raw[:, 6:] + 0.1 * rn(B, 126)).cuda(),
            'betas': (bstar + 0.5 * rn(B, module.num_betas)).cuda(), last[0]: last[1]}
    truth = dict(rot=rot, psi=psi.cuda(), joints=out['joints'][:].clone())
    return x.clone(), init, truth


def _fit(module, x, init, persp=False, **kw):
    from shapy_b200.fit import fit_body_to_keypoints_2d
    extra = dict(focal_length=F, principal_point=PP) if persp else {}
    return fit_body_to_keypoints_2d(module, x, init=init, method='lm', **extra, **kw)


def _wide_loop(module, x, w, init, iterations, persp=False):
    """The wide LM loop written out, keeping every iteration's state loss."""
    from shapy_b200 import ops
    from shapy_b200.fit import LM_DOWN, LM_UP
    packed = module.packed(x.device)
    B, K = x.shape[:2]
    nb, ne, n_rot = module.num_betas, module.num_expression_coeffs, 55
    ident = torch.tensor([1.0, 0.0, 0.0, 1.0, 0.0, 0.0], device='cuda')
    raw = torch.cat([init['global_rot'], init['body_pose'], ident.repeat(B, 33)], 1)
    lk = 'transl' if persp else 'camera'
    trial = {'rot': ops.decode_rot6d(raw).contiguous(), 'betas': init['betas'].clone().contiguous(),
             'expression': torch.zeros(B, ne, device='cuda'), lk: init[lk].clone().contiguous()}
    mk = lambda *s: torch.empty(*s, device='cuda')  # noqa: E731
    state = {'rot': mk(B, n_rot, 3, 3), 'betas': mk(B, nb), 'expression': mk(B, ne), lk: mk(B, 3),
             'keypoints': mk(B, K, 3), 'jac': mk(B, 3 * K, 3 * n_rot + nb + ne + 3), 'loss': mk(B), 'lambda': mk(B),
             'accepted': torch.zeros(B, dtype=torch.int32, device='cuda')}
    intr = torch.tensor([F, *PP], device='cuda').repeat(B, 1) if persp else None
    losses = []
    for it in range(iterations + 1):
        tkp, tjac = ops.smplx_keypoint_jacobian(packed, trial['betas'], trial['rot'], expr=trial['expression'])
        ops.fit_lm_keypoints_2d_expressive_step(state, trial, x, w, 0.1 if not persp else 10.0, 0.0, 0.01, 0.001,
                                                LM_UP, LM_DOWN, it == 0, tkp, tjac, intrinsics=intr)
        losses.append(state['loss'].clone())
    return torch.stack(losses), state


@pytest.mark.parametrize('persp', [False, True], ids=['weak', 'persp'])
def test_equals_todays_step_over_50_iterations(persp):
    """n_rot = 22 without expression: the wide step and today's 2D step (weak or perspective) give the same bits
    over a 50-iteration loop: state, loss, lambda and accepted count."""
    from shapy_b200 import ops
    from shapy_b200.fit import LM_DOWN, LM_UP
    module = harness.smplx_module()
    B = 48
    x, init, _ = _problem(module, B, seed=5, persp=persp)
    x = x.contiguous()
    w = torch.ones(B, x.shape[1], device='cuda')
    w[:, 3] = 0.0
    packed = module.packed('cuda')
    lk = 'transl' if persp else 'camera'
    intr = torch.tensor([F, *PP], device='cuda').repeat(B, 1) if persp else None
    rot0 = ops.decode_rot6d(torch.cat([init['global_rot'], init['body_pose']], 1)).contiguous()
    K, nb = x.shape[1], module.num_betas
    runs = []
    for wide in (False, True):
        trial = {'rot': rot0.clone(), 'betas': init['betas'].clone().contiguous(), lk: init[lk].clone().contiguous()}
        mk = lambda *s: torch.empty(*s, device='cuda')  # noqa: E731
        state = {'rot': mk(B, 22, 3, 3), 'betas': mk(B, nb), lk: mk(B, 3), 'keypoints': mk(B, K, 3),
                 'jac': mk(B, 3 * K, 66 + nb + 3), 'loss': mk(B), 'lambda': mk(B),
                 'accepted': torch.zeros(B, dtype=torch.int32, device='cuda')}
        if wide:
            trial['expression'] = torch.zeros(B, 0, device='cuda')
            state['expression'] = torch.zeros(B, 0, device='cuda')
        sigma = 10.0 if persp else 0.1
        for it in range(51):
            tkp, tjac = ops.smplx_keypoint_jacobian(packed, trial['betas'], trial['rot'])
            args = (sigma, 2.0, 0.01)
            if wide:
                ops.fit_lm_keypoints_2d_expressive_step(state, trial, x, w, *args, 0.0, LM_UP, LM_DOWN, it == 0, tkp,
                                                        tjac, pose_anchor=rot0, intrinsics=intr)
            elif persp:
                ops.fit_lm_keypoints_2d_perspective_step(state, trial, x, w, intr, *args, LM_UP, LM_DOWN, it == 0,
                                                         tkp, tjac, pose_anchor=rot0)
            else:
                ops.fit_lm_keypoints_2d_step(state, trial, x, w, *args, LM_UP, LM_DOWN, it == 0, tkp, tjac,
                                             pose_anchor=rot0)
        runs.append((state, trial))
    (s0, t0), (s1, t1) = runs
    for k in ('rot', 'betas', lk, 'keypoints', 'jac', 'loss', 'lambda', 'accepted'):
        assert torch.equal(s0[k].view(torch.int32), s1[k].view(torch.int32)), k
    for k in ('rot', 'betas', lk):
        assert torch.equal(bits(t0[k]), bits(t1[k])), k
    assert int(s1['accepted'].sum()) > B


@pytest.mark.parametrize('persp', [False, True], ids=['weak', 'persp'])
def test_wide_loop_monotone_deterministic_and_batch_independent(persp):
    module = harness.smplx_module()
    B = 24
    x, init, _ = _problem(module, B, seed=9, persp=persp)
    w = torch.ones(B, x.shape[1], device='cuda')
    losses, st = _wide_loop(module, x, w, init, 12, persp)
    d = losses[1:] - losses[:-1]
    assert bool((d <= 0).all()), float(d.max())
    assert float(losses[-1].mean()) < float(losses[0].mean())
    again, st2 = _wide_loop(module, x, w, init, 12, persp)
    assert torch.equal(bits(losses), bits(again))
    idx = torch.tensor([3, 17, 5], device='cuda')
    sub, st3 = _wide_loop(module, x[idx].contiguous(), w[idx].contiguous(), {k: v[idx] for k, v in init.items()}, 12,
                          persp)
    assert torch.equal(bits(losses[:, idx]), bits(sub))
    for k in ('rot', 'betas', 'expression'):
        assert torch.equal(bits(st[k]), bits(st2[k]))
        assert torch.equal(bits(st[k][idx]), bits(st3[k]))


def test_lm_fit_launches_and_never_synchronises():
    module = harness.smplx_module()
    B = 16
    x, init, _ = _problem(module, B, seed=3)
    kw = dict(pose_width=55, fit_expression=True, robust_sigma=0.1, pose_prior_weight=1.0, expression_weight=0.01)
    _fit(module, x, init, iterations=1, **kw)
    counts = []
    for it in (3, 5):
        n, res = harness.launches_without_sync(lambda: _fit(module, x, init, iterations=it, **kw))
        counts.append(n)
    assert counts[1] - counts[0] == 2 * 2, counts          # two launches per iteration
    assert res['full_pose_mat'].shape == (B, 55, 3, 3) and res['expression'].shape == (B, 10)
    assert res['left_hand_pose'].shape == (B, 90) and res['jaw_pose'].shape == (B, 6)
    assert res['body_pose'].shape == (B, 126) and res['body_pose_mat'].shape == (B, 21, 3, 3)


def test_fit_arguments():
    module = harness.smplx_module()
    x, init, _ = _problem(module, 2, seed=1)
    with pytest.raises(ValueError):
        _fit(module, x, init, pose_width=30)
    with pytest.raises(ValueError):
        _fit(module, x, init, pose_width=55, groups=torch.tensor([0, 0]))
    with pytest.raises(ValueError):
        _fit(module, x, init, fit_expression=True, share_pose=True, groups=torch.tensor([0, 0]))
    with pytest.raises(ValueError):
        _fit(module, x, init, pose_width=25, pose_prior_weight=np.ones(25))        # joint 0 must be 0
    jw = np.zeros(55)
    jw[1:22], jw[22:] = 1.0, 0.1
    res = _fit(module, x, init, pose_width=55, pose_prior_weight=jw, iterations=2)
    assert bool(torch.isfinite(res['loss']).all())


def test_adam_loss_matches_the_oracle():
    """Adam's returned loss at its final parameters equals the step oracle's loss there (float64, per body)."""
    from shapy_b200.fit import fit_body_to_keypoints_2d
    module = harness.smplx_module()
    B = 4
    x, init, _ = _problem(module, B, seed=13)
    jw = np.zeros(55)
    jw[1:22], jw[22:] = 0.5, 0.2
    res = fit_body_to_keypoints_2d(module, x, init=init, method='adam', iterations=20, pose_width=55,
                                   fit_expression=True, robust_sigma=0.2, pose_prior_weight=jw, betas_weight=0.01,
                                   expression_weight=0.05)
    from shapy_b200 import ops
    anchor = ops.decode_rot6d(torch.cat([init['global_rot'], init['body_pose'],
                                         torch.tensor([1.0, 0, 0, 1.0, 0, 0], device='cuda').repeat(B, 33)], 1))
    n = lambda t: t.detach().double().cpu().numpy()  # noqa: E731
    for b in range(B):
        want = o2.loss(n(x[b]), np.ones(x.shape[1]), n(res['keypoints'][b]), n(res['camera'][b]), 0.2,
                       n(res['full_pose_mat'][b]), n(anchor[b]), 0.0, n(res['betas'][b]), 0.01, joint_w=jw,
                       expr=n(res['expression'][b]), expr_w=0.05)
        assert abs(float(res['loss'][b]) - want) <= 1e-4 * abs(want), (b, float(res['loss'][b]), want)


def test_cli_fits_raw_openpose_detections_with_hands_and_face(tmp_path):
    """python -m shapy_b200.fit --keypoints-2d with img_00's raw OpenPose detections (body, hands and face) and the
    OpenPose -> SMPL-X map, --pose-width 55 --fit-expression, on the synthetic model."""
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
    out = tmp_path / 'fit.npz'
    fit.main(['--synthetic', '--keypoints-2d', str(tmp_path / 'kp.npz'), '--keypoint-map', kmap_path, '--method',
              'lm', '--iterations', '5', '--robust-sigma', '0.05', '--pose-prior-weight', '1.0', '--pose-width', '55',
              '--fit-expression', '--expression-weight', '0.01', '--output', str(out)])
    r = np.load(out)
    assert r['full_pose_mat'].shape == (1, 55, 3, 3) and r['expression'].shape == (1, 10)
    assert r['right_hand_pose'].shape == (1, 90) and r['jaw_pose'].shape == (1, 6)
    assert np.isfinite(r['loss']).all() and np.isfinite(r['full_pose_mat']).all()


# ------------------------------------------------------------------------------------------------ quality
def _quality(module, x, init, truth, persp, **kw):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = _fit(module, x, init, persp=persp, iterations=50, **kw)
    torch.cuda.synchronize()
    return res, time.perf_counter() - t0


def test_quality_whole_body():
    """256 synthetic bodies with hands, jaw and expression, exact targets: today's 22-joint fit on all keypoints (a),
    on the body keypoints alone (b), the whole-body fit (c) and (c) under the perspective camera (d)."""
    module = harness.smplx_module()
    B = 256
    x, init, truth = _problem(module, B, seed=77)
    xp, initp, truthp = _problem(module, B, seed=77, persp=True)
    K = x.shape[1]
    wall = torch.ones(B, K, device='cuda')
    wbody = torch.zeros(B, K, device='cuda')
    wbody[:, :22] = 1.0
    hands = torch.arange(25, 55, device='cuda')
    face = torch.arange(76, K, device='cuda') if K > 76 else torch.arange(55, K, device='cuda')
    rows = {}
    _fit(module, x, init, iterations=1, pose_width=55, fit_expression=True)             # warm-up
    for name, (xx, ii, tt, persp, kw) in {
            'a': (x, init, truth, False, dict(weights=wall)),
            'b': (x, init, truth, False, dict(weights=wbody)),
            'c': (x, init, truth, False, dict(weights=wall, pose_width=55, fit_expression=True,
                                              expression_weight=1e-4)),
            'd': (xp, initp, truthp, True, dict(weights=wall, pose_width=55, fit_expression=True,
                                                expression_weight=1e-4))}.items():
        res, sec = _quality(module, xx, ii, tt, persp, **kw)
        scale = 1.0 if not persp else 1.0 / F                # RMS in crop units (persp: pixels / f)
        d2 = (res['proj_joints'] - xx).pow(2).sum(-1)
        rms = (d2.mean(1).sqrt() * scale)
        rms_h = (d2[:, hands].mean(1).sqrt() * scale).median()
        rms_f = (d2[:, face].mean(1).sqrt() * scale).median()
        j = res['keypoints'][:, :22]
        jt = tt['joints'][:, :22]
        mpj = ((j - j[:, :1]) - (jt - jt[:, :1])).norm(dim=-1).mean(1).median()
        if 'full_pose_mat' in res:
            R = res['full_pose_mat'][:, 25:55]
        else:
            R = torch.eye(3, device='cuda').expand(B, 30, 3, 3)
        rel = R.transpose(-1, -2) @ tt['rot'][:, 25:55]
        geo = torch.acos(((rel.diagonal(dim1=-2, dim2=-1).sum(-1) - 1) / 2).clamp(-1, 1)).mean(1).median()
        psi = res.get('expression', torch.zeros_like(tt['psi']))
        epsi = (psi - tt['psi']).norm(dim=1).median()
        rows[name] = dict(share=float((rms < 2e-3).float().mean()), rms_hand=float(rms_h), rms_face=float(rms_f),
                          mpjpe=float(mpj), hand_geo=float(geo), psi_err=float(epsi), sec=sec)
        print(f'[expressive] quality ({name}): ' + ', '.join(f'{k} {v:.4g}' for k, v in rows[name].items()))
    a, c, d = rows['a'], rows['c'], rows['d']
    # bars just past the values measured on an H100 (the fits are deterministic).  (c) explains the hand points that
    # (a) cannot and has the lower body-joint error; under the weak-perspective camera it barely improves on (a) at the
    # face landmarks, which (d) explains
    assert c['rms_hand'] < 0.11 < a['rms_hand'] and c['mpjpe'] < 0.16 < a['mpjpe']
    assert c['rms_face'] < 0.32 and c['share'] >= 0.2 and c['hand_geo'] < 0.46 and c['psi_err'] < 2.8
    assert d['rms_hand'] < 0.018 and d['rms_face'] < 0.055 and d['share'] >= 0.24 and d['mpjpe'] < 0.16
