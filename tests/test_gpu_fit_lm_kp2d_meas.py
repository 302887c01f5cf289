"""GPU: the stacked 2D keypoint + measurement Levenberg-Marquardt step (shapy_fit_lm_keypoints_2d_measurements_step)
against its NumPy restatement (tests/kp2d_lm_oracle.py with `meas`, pinned by tests/test_fit_lm_kp2d_meas_cpu.py) and against
shapy_fit_lm_keypoints_2d_step when every measurement is dropped; and fit_body_to_keypoints_2d with known measurements
end to end on the synthetic SMPL-X: unchanged without them, deterministic, batch independent, monotone, never
synchronising, and the quality with known height and mass against the keypoints alone."""
import math

import numpy as np
import pytest
import torch

import kp2d_lm_oracle as o2
import lm_harness as harness
from lm_harness import bits, rodrigues
from shapy_b200 import synth

pytestmark = pytest.mark.gpu
NAMES, N_ROT = harness.NAMES, harness.N_ROT
# (robust_sigma, pose_prior_weight, betas_weight)
TERMS = [(math.inf, 0.0, 0.0), (0.3, 0.5, 0.1)]


@pytest.fixture(scope='module')
def model():
    return harness.smplx_and_measurements()


# ------------------------------------------------------------------------------------------------ step
def _evaluate(packed, lm, faces, rot, betas, exact):
    from shapy_b200 import ops
    c = lambda t: t.cuda().contiguous()  # noqa: E731
    kp, jac = ops.smplx_keypoint_jacobian(packed, c(betas), c(rot))
    meas, mjac, _ = ops.measure_jacobian_betas(packed, lm, ops.smplx_forward_shape(packed, c(betas)), faces,
                                               exact=exact)
    return [t.cpu() for t in (kp, jac, meas, mjac)]


def _step_case(model, terms, exact=False):
    """Eight bodies of the synthetic model: the state at one pose, shape and camera, the trial at a nearby one.  Body 0
    targets the trial (accepted), 1 the state (rejected), 2 the trial with a dropped measurement whose value and row
    are NaN in state and trial (accepted), 3 a weighted NaN trial measurement (rejected), 4 to 7 random targets.
    Keypoint 7 has weight 0 and NaN targets, keypoints and rows in state and trial."""
    smplx, bm = model
    sigma, pw, bw = terms
    packed, faces, lm = smplx.packed(), smplx.faces_i32, bm.landmarks()
    B = 8
    gen = torch.Generator().manual_seed(41)                   # the rotations and betas of test_gpu_fit_lm_kp_meas.py
    rn = lambda *s: torch.randn(*s, generator=gen)  # noqa: E731
    rot = rodrigues(torch.randn(B, N_ROT, 3, generator=gen, dtype=torch.float64) * 0.3).float()
    betas = rn(B, 10).clamp(-2, 2)
    cam = torch.stack([1.0 + 0.2 * rn(B), 0.1 * rn(B), 0.1 * rn(B)], 1)
    trot = (rot.double() @ rodrigues(rn(B, N_ROT, 3).double() * 0.02)).float()
    anchor = (rot.double() @ rodrigues(rn(B, N_ROT, 3).double() * 0.05)).float()
    tbetas, tcam = betas + 0.05 * rn(B, 10), cam + 0.01 * rn(B, 3)
    for b in (0, 2):                                          # the priors favour the accepted trials ...
        anchor[b], tbetas[b] = trot[b], 0.9 * betas[b]
    anchor[1], tbetas[1] = rot[1], 1.1 * betas[1]             # ... and body 1's state
    tcam[1, 1] += 0.05                                        # body 1's trial clearly worse
    kp, jac, meas, mjac = _evaluate(packed, lm, faces, rot, betas, exact)
    tkp, tjac, tmeas, tmjac = _evaluate(packed, lm, faces, trot, tbetas, exact)
    assert all(bool(torch.isfinite(t).all()) for t in (meas, tmeas, mjac, tmjac))
    K = packed.K
    proj = lambda k, c: torch.stack([torch.from_numpy(o2.project(k[b].numpy(), c[b].numpy())).float()  # noqa: E731
                                     for b in range(B)])
    ps, pt = proj(kp, cam), proj(tkp, tcam)
    tg = ps + 0.02 * rn(B, K, 2)
    mt = tmeas * (1 + 0.02 * rn(B, 5))
    for b in (0, 2, 3):
        tg[b], mt[b] = pt[b], tmeas[b]
    tg[1], mt[1] = ps[1], meas[1]
    w = torch.rand(B, K, generator=gen) + 0.5
    w[:, 7] = 0.0
    tg[:, 7] = float('nan')
    for t in (kp, tkp):
        t[:, 7] = float('nan')
    for t in (jac, tjac):
        t[:, 21:24] = float('nan')
    mw = torch.tensor([1.0, 100.0, 2000.0, 1000.0, 1000.0]).repeat(B, 1)
    mw[2, 2] = 0.0
    for t in (meas, tmeas, mjac, tmjac):
        t[2, 2] = float('nan')
    tmeas[3, 3] = float('nan')
    return dict(rot=rot, betas=betas, cam=cam, kp=kp, jac=jac, meas=meas, mjac=mjac, trot=trot, tbetas=tbetas,
                tcam=tcam, tkp=tkp, tjac=tjac, tmeas=tmeas, tmjac=tmjac, tg=tg, w=w, mt=mt, mw=mw, anchor=anchor,
                lam=torch.rand(B, generator=gen) + 0.01, sigma=sigma, pw=pw, bw=bw)


def _state(c, with_meas=True):
    """The state and trial tensors on the device, the state's loss from the oracle (float32)."""
    B = c['rot'].shape[0]
    n = lambda t: t.numpy()  # noqa: E731
    loss = torch.tensor([o2.loss(n(c['tg'][b]), n(c['w'][b]), n(c['kp'][b]), n(c['cam'][b]), c['sigma'],
                                 n(c['rot'][b]), n(c['anchor'][b]), c['pw'], n(c['betas'][b]), c['bw'],
                                 meas=(n(c['mt'][b]), n(c['mw'][b]), n(c['meas'][b]))) for b in range(B)]).float()
    cu = lambda t: t.cuda().contiguous()  # noqa: E731
    state = {'rot': cu(c['rot']), 'betas': cu(c['betas']), 'camera': cu(c['cam']), 'keypoints': cu(c['kp']),
             'jac': cu(c['jac']), 'loss': cu(loss), 'lambda': cu(c['lam']),
             'accepted': torch.zeros(B, dtype=torch.int32, device='cuda')}
    if with_meas:
        state.update(meas=cu(c['meas']), meas_jac=cu(c['mjac']))
    trial = {'rot': cu(c['trot']), 'betas': cu(c['tbetas']), 'camera': cu(c['tcam'])}
    return state, trial


def _meas_step(c, state, trial, first):
    from shapy_b200 import ops
    cu = lambda t: t.cuda().contiguous()  # noqa: E731
    ops.fit_lm_keypoints_2d_measurements_step(state, trial, cu(c['tg']), cu(c['w']), c['sigma'], c['pw'], c['bw'],
                                              cu(c['mt']), cu(c['mw']), 10.0, 3.0, first, cu(c['tkp']), cu(c['tjac']),
                                              cu(c['tmeas']), cu(c['tmjac']), pose_anchor=cu(c['anchor']))


@pytest.mark.parametrize('derivative', ['reference', 'exact'])
@pytest.mark.parametrize('terms', TERMS, ids=['lsq', 'robust_priors'])
@pytest.mark.parametrize('first', [False, True])
def test_step_kernel_vs_oracle(model, first, terms, derivative):
    c = _step_case(model, terms, exact=derivative == 'exact')
    B = c['rot'].shape[0]
    state, trial = _state(c)
    s0 = {k: v.cpu().numpy() for k, v in state.items()}
    _meas_step(c, state, trial, first)
    n = lambda t: t.numpy()  # noqa: E731
    oracle = []
    for b in range(B):
        s = {k: s0[k][b] for k in s0}
        s['accepted'] = 0
        tr = {'rot': n(c['trot'][b]), 'betas': n(c['tbetas'][b]), 'camera': n(c['tcam'][b])}
        oracle.append(o2.lm_keypoints_2d_step(
            s, n(c['tg'][b]), n(c['w'][b]), 10.0, 3.0, first, tr, n(c['tkp'][b]), n(c['tjac'][b]), sigma=c['sigma'],
            anchor=n(c['anchor'][b]), pose_w=c['pw'], betas_w=c['bw'], meas=(n(c['mt'][b]), n(c['mw'][b])),
            trial_meas=(n(c['tmeas'][b]), n(c['tmjac'][b]))))
    got = harness.numpy_of(state)
    keys = ('rot', 'betas', 'camera')
    # softplus' exp / log1p may round differently on the device: loss and lambda to fp32 rounding
    flags, worst = harness.check_step(harness.rows_of(got, B), harness.rows_of(harness.numpy_of(trial), B), oracle,
                                 keys + ('keypoints', 'jac', 'meas', 'meas_jac'), keys, exact=False)
    if first:
        assert all(flags) and np.isnan(got['loss'][3])
    else:
        assert flags[:4] == [True, False, True, False], flags
    print(f'[kp2dm] step first={first} terms={terms} {derivative}: accepted {flags}, trial error / bar {worst:.3f}')


@pytest.mark.parametrize('terms', TERMS, ids=['lsq', 'robust_priors'])
@pytest.mark.parametrize('first', [False, True])
def test_dropped_measurements_equal_the_2d_step_bit_for_bit(model, first, terms):
    """Every measurement weight <= 0, NaN in the measurements and their rows, state and trial: torch.equal to
    shapy_fit_lm_keypoints_2d_step on state and trial."""
    from shapy_b200 import ops
    c = _step_case(model, terms)
    for k in ('meas', 'tmeas', 'mjac', 'tmjac'):
        c[k][:] = float('nan')
    c['mw'][:] = 0.0
    c['mw'][:, 1] = -1.0
    a_state, a_trial = _state(c)
    b_state = {k: v.clone() for k, v in a_state.items() if k not in ('meas', 'meas_jac')}
    b_trial = {k: v.clone() for k, v in a_trial.items()}
    _meas_step(c, a_state, a_trial, first)
    cu = lambda t: t.cuda().contiguous()  # noqa: E731
    ops.fit_lm_keypoints_2d_step(b_state, b_trial, cu(c['tg']), cu(c['w']), c['sigma'], c['pw'], c['bw'], 10.0, 3.0,
                                 first, cu(c['tkp']), cu(c['tjac']), pose_anchor=cu(c['anchor']))
    for k in ('rot', 'betas', 'camera', 'keypoints', 'jac', 'loss', 'lambda', 'accepted'):
        assert torch.equal(bits(a_state[k]), bits(b_state[k])), k
    for k in ('rot', 'betas', 'camera'):
        assert torch.equal(bits(a_trial[k]), bits(b_trial[k])), k
    assert bool(torch.isfinite(a_state['loss']).all())


# ------------------------------------------------------------------------------------------------ fit
def _problem(module, bm, B, seed=41):
    """The recipe of tests/test_gpu_fit_lm_keypoints_2d.py (_problem: same seed, same draws in the same order), plus the
    generating betas and their measurements."""
    from shapy_b200 import ops
    gen = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=gen)  # noqa: E731
    bstar = rn(B, module.num_betas).clamp(-2, 2)
    raw = synth.mean_params()[:132] + 0.3 * rn(B, 132)
    cam = torch.stack([1.0 + 0.2 * rn(B), 0.1 * rn(B), 0.1 * rn(B)], 1)
    with torch.no_grad():
        rot = ops.decode_rot6d(raw.cuda())
        out = module(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=bstar.cuda(), camera=cam.cuda())
        tgt = harness.measure(module, bm, bstar.cuda())
    init = {'global_rot': (raw[:, :6] + 0.1 * rn(B, 6)).cuda(), 'body_pose': (raw[:, 6:] + 0.1 * rn(B, 126)).cuda(),
            'betas': (bstar + 0.5 * rn(B, module.num_betas)).cuda(), 'camera': (cam + 0.05 * rn(B, 3)).cuda()}
    return dict(x=out['proj_joints'].clone(), joints=out['joints'][:].clone(), init=init, bstar=bstar.cuda(), tgt=tgt,
                tg={k: tgt[:, i].contiguous() for i, k in enumerate(NAMES)})


def _lm_loop(module, bm, p, w, iterations, sigma=None, pw=0.0, bw=0.0, measurements=None, exact=False):
    """The LM loop of fit_body_to_keypoints_2d written out over the ops, keeping every iteration's state loss; without
    measurements, the two launches of the keypoint-only fit."""
    from shapy_b200 import ops
    from shapy_b200.fit import LM_DOWN, LM_UP, _measurement_terms
    x, init = p['x'], p['init']
    packed = module.packed(x.device)
    B, K = x.shape[:2]
    nb = init['betas'].shape[1]
    P = 3 * N_ROT + nb + 3
    rot0 = ops.decode_rot6d(torch.cat([init['global_rot'], init['body_pose']], 1)).contiguous()
    trial = {'rot': rot0.clone(), 'betas': init['betas'].clone().contiguous(), 'camera': init['camera'].clone()}
    mk = lambda *s: torch.empty(*s, device='cuda')  # noqa: E731
    state = {'rot': mk(B, N_ROT, 3, 3), 'betas': mk(B, nb), 'camera': mk(B, 3), 'keypoints': mk(B, K, 3),
             'jac': mk(B, 3 * K, P), 'loss': mk(B), 'lambda': mk(B),
             'accepted': torch.zeros(B, dtype=torch.int32, device='cuda')}
    anchor = rot0 if pw > 0 else None
    if measurements is not None:
        state.update(meas=mk(B, 5), meas_jac=mk(B, 5, nb))
        mt, mw = _measurement_terms(measurements, None, B, x.device)
        faces, lm = module.faces_i32, bm.landmarks()
    losses = []
    for it in range(iterations + 1):
        tkp, tjac = ops.smplx_keypoint_jacobian(packed, trial['betas'], trial['rot'])
        if measurements is None:
            ops.fit_lm_keypoints_2d_step(state, trial, x, w, sigma, pw, bw, LM_UP, LM_DOWN, it == 0, tkp, tjac,
                                         pose_anchor=anchor)
        else:
            tm, tmj, _ = ops.measure_jacobian_betas(packed, lm, ops.smplx_forward_shape(packed, trial['betas']), faces,
                                                    exact=exact)
            ops.fit_lm_keypoints_2d_measurements_step(state, trial, x, w, sigma, pw, bw, mt.contiguous(),
                                                      mw.contiguous(), LM_UP, LM_DOWN, it == 0, tkp, tjac, tm, tmj,
                                                      pose_anchor=anchor)
        losses.append(state['loss'].clone())
    return state, torch.stack(losses)


def test_fit_without_measurements_is_unchanged(model):
    """measurements=None: the same bits as the keypoint-only loop over ops.smplx_keypoint_jacobian and
    ops.fit_lm_keypoints_2d_step, and no 'measurements' in the result."""
    from shapy_b200.fit import fit_body_to_keypoints_2d
    module, bm = model
    p = _problem(module, bm, 32, seed=5)
    w = torch.ones(32, p['x'].shape[1], device='cuda')
    state, _ = _lm_loop(module, bm, p, w, 12, 0.05, 0.5, 0.01)
    res = fit_body_to_keypoints_2d(module, p['x'], init=p['init'], method='lm', iterations=12, robust_sigma=0.05,
                                   pose_prior_weight=0.5, betas_weight=0.01, body_measurements=bm)
    assert 'measurements' not in res
    for k in ('betas', 'camera'):
        assert torch.equal(bits(res[k]), bits(state[k])), k
    assert torch.equal(bits(res['global_rot_mat']), bits(state['rot'][:, :1]))
    assert torch.equal(bits(res['body_pose_mat']), bits(state['rot'][:, 1:]))


@pytest.mark.parametrize('derivative', ['reference', 'exact'])
def test_lm_losses_monotone_and_returned_by_the_fit(model, derivative):
    """With known height and mass, a robust loss and both priors, every body's loss is non-increasing at every
    iteration; fit_body_to_keypoints_2d returns the loop's parameters and measurements, and its loss is the total."""
    from shapy_b200.fit import fit_body_to_keypoints_2d
    module, bm = model
    p = _problem(module, bm, 64, seed=5)
    w = (torch.rand(64, p['x'].shape[1], generator=torch.Generator().manual_seed(6)) + 0.5).cuda()
    w[:, 3] = 0.0
    p['x'][:, 3] = float('nan')
    meas = {k: p['tg'][k] for k in (('height', 'mass') if derivative == 'reference' else NAMES)}
    state, losses = _lm_loop(module, bm, p, w, 20, 0.05, 0.5, 0.01, meas, exact=derivative == 'exact')
    fin = torch.isfinite(losses[0])          # a body whose weighted circumference is NaN at the start never moves
    assert float(fin.float().mean()) >= 0.9
    losses = losses[:, fin]
    assert bool(torch.isfinite(losses).all())
    assert bool((losses[1:] <= losses[:-1]).all())
    ratio = float(losses[-1].median()) / float(losses[0].median())
    print(f'[kp2dm] {derivative}: median loss after 20 iterations / start {ratio:.4f}')
    assert ratio < 0.5
    res = fit_body_to_keypoints_2d(module, p['x'], w, init=p['init'], method='lm', iterations=20, robust_sigma=0.05,
                                   pose_prior_weight=0.5, betas_weight=0.01, body_measurements=bm, measurements=meas,
                                   circumference_derivative=derivative)
    for k in ('betas', 'camera'):
        assert torch.equal(bits(res[k]), bits(state[k])), k
    assert torch.equal(bits(res['measurements']), bits(state['meas']))
    torch.testing.assert_close(res['measurements'][fin], harness.measure(module, bm, res['betas'])[fin], rtol=1e-6,
                               atol=1e-7, equal_nan=True)
    # the returned loss comes from SMPLX.forward's proj_joints, the kernel's from the Jacobian launch's keypoints
    assert float(((res['loss'] - state['loss']).abs() / state['loss'])[fin].max()) <= 1e-2


def test_lm_deterministic_and_batch_independent(model):
    from shapy_b200.fit import fit_body_to_keypoints_2d
    module, bm = model
    p = _problem(module, bm, 64, seed=8)
    kw = dict(method='lm', iterations=15, robust_sigma=0.1, pose_prior_weight=0.5, body_measurements=bm)
    meas = {k: p['tg'][k] for k in ('height', 'mass')}
    r1 = fit_body_to_keypoints_2d(module, p['x'], init=p['init'], measurements=meas, **kw)
    r2 = fit_body_to_keypoints_2d(module, p['x'], init=p['init'], measurements=meas, **kw)
    rows = [0, 5, 17, 33, 63]
    r8 = fit_body_to_keypoints_2d(module, p['x'][rows].contiguous(),
                                  init={k: v[rows].contiguous() for k, v in p['init'].items()},
                                  measurements={k: v[rows].contiguous() for k, v in meas.items()}, **kw)
    for k in ('global_rot', 'body_pose', 'betas', 'camera', 'measurements', 'loss'):
        assert torch.equal(bits(r1[k]), bits(r2[k])), k
        if k != 'loss':                   # the returned loss is summed by torch, whose reduction order follows the batch
            assert torch.equal(bits(r8[k]), bits(r1[k][rows])), k
    one = fit_body_to_keypoints_2d(module, p['x'][17:18].contiguous(),
                                   init={k: v[17:18].contiguous() for k, v in p['init'].items()},
                                   measurements={k: v[17:18].contiguous() for k, v in meas.items()}, **kw)
    for k in ('betas', 'camera', 'measurements'):
        assert torch.equal(bits(one[k]), bits(r1[k][17:18])), k


def test_lm_loop_never_synchronises(model):
    from shapy_b200.fit import fit_body_to_keypoints_2d
    module, bm = model
    p = _problem(module, bm, 32, seed=7)
    kw = dict(init=p['init'], method='lm', robust_sigma=0.1, pose_prior_weight=1.0, betas_weight=0.01,
              body_measurements=bm, measurements=p['tg'])
    fit_body_to_keypoints_2d(module, p['x'], iterations=1, **kw)      # packs the model, builds the incidence table
    _, res = harness.launches_without_sync(lambda: fit_body_to_keypoints_2d(module, p['x'], iterations=3, **kw))
    assert res['measurements'].shape == (32, 5)


def test_adam_counts_the_betas_regulariser_once(model):
    """Adam with measurements: 'measurements' returned, and the loss is the 2D loss + the measurement terms, the
    betas regulariser once."""
    from shapy_b200.fit import _kp2d_loss, _measurement_loss, _measurement_terms, fit_body_to_keypoints_2d
    module, bm = model
    p = _problem(module, bm, 8, seed=9)
    meas = {k: p['tg'][k] for k in ('height', 'mass')}
    res = fit_body_to_keypoints_2d(module, p['x'], init=p['init'], iterations=5, betas_weight=0.3,
                                   body_measurements=bm, measurements=meas)
    assert res['measurements'].shape == (8, 5)
    mt, mw = _measurement_terms(meas, None, 8, 'cuda')
    w = torch.ones(8, p['x'].shape[1], device='cuda')
    want = _kp2d_loss(res['proj_joints'], p['x'], w, None, 0.0, None, None, 0.3, res['betas']) + \
        _measurement_loss(mt, mw, res['measurements'], res['betas'], 0.0)
    torch.testing.assert_close(res['loss'], want, rtol=1e-5, atol=1e-7)


class _FakeModel:
    num_betas = 10
    shapedirs = torch.zeros(1)


def test_argument_errors_and_empty_batch(model):
    from shapy_b200 import _lib, ops
    from shapy_b200.fit import fit_body_to_keypoints_2d
    module, bm = model
    L = _lib.lib()
    K = module.packed().K
    z = lambda *s: torch.zeros(*s, device='cuda')  # noqa: E731
    with pytest.raises(ValueError):
        fit_body_to_keypoints_2d(_FakeModel(), z(2, K, 2), measurements={'height': 1.7})    # no body_measurements
    with pytest.raises(ValueError):
        fit_body_to_keypoints_2d(_FakeModel(), z(2, K, 2), circumference_derivative='numeric')
    with pytest.raises(ValueError):
        fit_body_to_keypoints_2d(module, z(4, K, 2), method='lm', body_measurements=bm,
                                 measurements={'height': z(3) + 1.7})
    torch.cuda.synchronize()
    n0 = L.shapy_launch_count()

    def step(B=2, n_rot=22, nb=10, null=None, sigma=1.0, pw=0.0, bw=0.0, up=10.0, down=3.0, anchor=True):
        P = 3 * n_rot + nb + 3
        p = [_lib.ptr(t) for t in (z(B, n_rot, 3, 3), z(B, nb), z(B, 3), z(B, K, 3), z(B, 3 * K, P), z(B, 5),
                                   z(B, 5, nb), z(B), z(B), torch.zeros(B, dtype=torch.int32, device='cuda'))]
        q = [_lib.ptr(t) for t in (z(B, n_rot, 3, 3), z(B, nb), z(B, 3), z(B, K, 3), z(B, 3 * K, P), z(B, 5),
                                   z(B, 5, nb))]
        mt = [_lib.ptr(z(B, 5)), _lib.ptr(z(B, 5))]
        if null == 'meas_jac':
            p[6] = None
        elif null == 'trial_meas':
            q[5] = None
        elif null == 'meas_weights':
            mt[1] = None
        elif null == 'jac':
            p[4] = None
        return L.shapy_fit_lm_keypoints_2d_measurements_step(
            B, K, n_rot, nb, _lib.ptr(z(B, K, 2)), _lib.ptr(z(B, K)), _lib.ptr(z(B, n_rot, 3, 3)) if anchor else None,
            sigma, pw, bw, *mt, up, down, 1, *p, *q, None)
    assert step(n_rot=30) == -3                     # P = 103 > 96
    for kw in (dict(null='meas_jac'), dict(null='trial_meas'), dict(null='meas_weights'), dict(null='jac'),
               dict(sigma=0.0), dict(sigma=float('nan')), dict(pw=-1.0), dict(bw=-0.5), dict(up=0.5), dict(down=0.9),
               dict(pw=1.0, anchor=False), dict(n_rot=0)):
        assert step(**kw) == -1, kw
    st = {'rot': z(0, 22, 3, 3), 'betas': z(0, 10), 'camera': z(0, 3), 'keypoints': z(0, K, 3), 'jac': z(0, 3 * K, 79),
          'meas': z(0, 5), 'meas_jac': z(0, 5, 10), 'loss': z(0), 'lambda': z(0),
          'accepted': torch.zeros(0, dtype=torch.int32, device='cuda')}
    tr = {'rot': z(0, 22, 3, 3), 'betas': z(0, 10), 'camera': z(0, 3)}
    args = (z(0, K, 3), z(0, 3 * K, 79), z(0, 5), z(0, 5, 10))
    ops.fit_lm_keypoints_2d_measurements_step(st, tr, z(0, K, 2), z(0, K), None, 0.0, 0.0, z(0, 5), z(0, 5), 10.0, 3.0,
                                              True, *args)
    with pytest.raises(ValueError):
        ops.fit_lm_keypoints_2d_measurements_step(st, tr, z(0, K, 2), z(0, K), None, 1.0, 0.0, z(0, 5), z(0, 5), 10.0,
                                                  3.0, True, *args)                          # prior without anchor
    with pytest.raises(RuntimeError):
        ops.fit_lm_keypoints_2d_measurements_step(st, tr, z(0, K, 2), z(0, K), None, 0.0, 0.0, z(0, 4), z(0, 5), 10.0,
                                                  3.0, True, *args)                          # targets not (B, 5)
    assert L.shapy_launch_count() == n0


# Quality, 256 bodies, 50 LM iterations, the problem of tests/test_gpu_fit_lm_keypoints_2d.py (seed 41, perturbed
# start): keypoints alone against keypoints + known height and mass, with all keypoints and with the 22 posed body
# joints only.  Bars just below the first run on an H100 80GB HBM3 (700 W), with / without the measurements:
#   all keypoints: height < 1 mm 0.402 / 0.371, mass < 1 % 0.938 / 0.887, 2D RMS < 2e-3 0.289 / 0.297, median
#     |beta - beta*| 1.24 / 1.32, median root-aligned joint error 0.191 / 0.192 m.  Seven bodies in ten do not converge
#     in the image from this start, with or without measurements, and those decide the shares;
#   body joints: height 0.961 / 0.180, mass 0.961 / 0.938, 2D RMS 1.0 / 1.0, |beta - beta*| 0.95 / 1.10, joint error
#     0.125 / 0.127 m: the height is what the keypoints cannot see; the joint error is depth and pose, not size.
QUALITY_BARS = {'all': {'height_1mm': 0.38, 'mass_1pct': 0.92, 'frac_rms2d': 0.27},
                'body': {'height_1mm': 0.94, 'mass_1pct': 0.94, 'frac_rms2d': 0.98}}


@pytest.mark.parametrize('which', ['all', 'body'])
def test_fit_quality_256_bodies(model, which):
    from shapy_b200.fit import fit_body_to_keypoints_2d
    module, bm = model
    p = _problem(module, bm, 256)
    w = torch.ones(p['x'].shape[1], device='cuda')
    if which == 'body':                       # only the posed skeleton joints of the 22 fitted rotations
        w[N_ROT:] = 0.0
    kw = dict(init=p['init'], method='lm')
    hm = dict(body_measurements=bm, measurements={k: p['tg'][k] for k in ('height', 'mass')})
    kpo = fit_body_to_keypoints_2d(module, p['x'], w, **kw)
    comb = fit_body_to_keypoints_2d(module, p['x'], w, **hm, **kw)
    start = fit_body_to_keypoints_2d(module, p['x'], w, iterations=0, **hm, **kw)['loss']
    qk, qc = harness.quality_2d(module, bm, p, kpo, w), harness.quality_2d(module, bm, p, comb, w)
    print(f'fit_kp2d_meas_lm_256[{which}]', {'keypoints_only': qk, 'height_mass': qc,
                                             'median_loss': float(comb['loss'].median()),
                                             'median_start': float(start.median())})
    fin = torch.isfinite(start)
    assert bool((comb['loss'][fin] <= start[fin] * (1 + 1e-2)).all())
    for k in ('height_1mm', 'mass_1pct'):
        assert qc[k] > qk[k], (k, qc[k], qk[k])
    if which == 'body':                       # where the image is fitted, the known height is what was missing
        assert qc['height_1mm'] >= qk['height_1mm'] + 0.5
    assert qc['frac_rms2d'] >= 0.9 * qk['frac_rms2d'], (qc['frac_rms2d'], qk['frac_rms2d'])
    assert all(qc[k] >= QUALITY_BARS[which][k] for k in QUALITY_BARS[which]), qc
