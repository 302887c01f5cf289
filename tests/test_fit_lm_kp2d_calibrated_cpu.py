"""CPU: the float64 restatement of the calibrated 2D keypoint LM step (tests/kp2d_calibrated_lm_oracle.py) pinned to
central differences of its projection (every column, random extrinsics, several views) and of its loss, the depth rule
per view, one identity view against the perspective oracle, a plain fp64 LM on a noiseless 4-camera rig;
fit.calibrated_start against a float64 SMPL-X forward, and the default translation start on noiseless rays."""
import math

import numpy as np
import pytest
import torch

import kp2d_calibrated_lm_oracle as oc
import kp2d_lm_oracle as o2
from lm_harness import expm, toy_problem

INTR = np.array([1000.0, 500.0, 480.0])
T0 = np.array([0.1, -0.2, 0.3])                # the toy body's world translation


def _look_at(azimuth_deg, radius=6.0, height=0.0, target=np.zeros(3)):
    """Extrinsics (12,) of a camera on a circle of `radius` about the vertical (world y) axis, at `height`, looking at
    `target`: camera y along world -y (down), z towards the target."""
    a = math.radians(azimuth_deg)
    centre = target + np.array([radius * math.sin(a), height, -radius * math.cos(a)])
    z = (target - centre) / np.linalg.norm(target - centre)
    y = np.array([0.0, -1.0, 0.0])
    y = y - (y @ z) * z
    y /= np.linalg.norm(y)
    x = np.cross(y, z)
    R = np.stack([x, y, z])
    return np.concatenate([R.reshape(9), -R @ centre])


def _rand_ext(rng):
    """A random view 5-8 m from the origin, looking near it."""
    ext = _look_at(rng.uniform(0, 360), rng.uniform(5, 8), rng.uniform(-1, 1), rng.normal(size=3) * 0.2)
    R = ext[:9].reshape(3, 3) @ expm(rng.normal(size=3) * 0.05)
    return np.concatenate([R.reshape(9), ext[9:]])


def _views(rng, kp, V=3, noise=20.0):
    ext = np.stack([_rand_ext(rng) for _ in range(V)])
    intr = np.stack([INTR * np.array([rng.uniform(0.8, 1.2), 1.0, 1.0]) for _ in range(V)])
    tg = np.stack([oc.project(kp, T0, intr[v], ext[v]) for v in range(V)]) + rng.normal(size=(V, len(kp), 2)) * noise
    w = rng.uniform(0.5, 1.5, (V, len(kp)))
    w[:, 3], tg[:, 3] = 0.0, np.nan
    return tg, w, intr, ext


def _case(seed, V=3):
    evaluate, rng = toy_problem(seed)
    rot = np.stack([expm(rng.normal(size=3) * 0.5) for _ in range(2)])
    beta = np.array([0.3])
    kp, jac = evaluate(rot, beta)
    return evaluate, rng, rot, beta, kp, jac, _views(rng, kp, V)


def _at(evaluate, rot, beta, theta):
    """(rotations, betas, t, keypoints) at the offsets theta = [delta_0, delta_1 | beta | t]."""
    R = np.stack([rot[j] @ expm(theta[3 * j:3 * j + 3]) for j in range(2)])
    b = beta + theta[6:7]
    kp, _ = evaluate(R, b)
    return R, b, T0 + theta[7:], kp


def test_rows_vs_central_differences_on_every_column():
    evaluate, _, rot, beta, kp, jac, (tg, w, intr, ext) = _case(21)
    jac[:, 7:] = 7.0                          # the 3D transl columns are not read: J_t = I
    h = 1e-6
    for v in range(len(ext)):
        J2 = oc.jacobian_calibrated(kp, jac, T0, intr[v], ext[v])
        fd = np.zeros((24, 10))
        for i in range(10):
            e = np.zeros(10)
            e[i] = h
            a, b = _at(evaluate, rot, beta, e), _at(evaluate, rot, beta, -e)
            fd[:, i] = (oc.project(a[3], a[2], intr[v], ext[v]) - oc.project(b[3], b[2], intr[v], ext[v])).reshape(-1) \
                / (2 * h)
        assert np.abs(J2 - fd).max() <= 1e-6 * np.abs(fd).max(), v


def _meas(rng, beta):
    """A linear measurement block m(beta) = m0 + Jm beta: (meas_targets, meas_weights, meas, meas_jac) at beta."""
    Jm = rng.normal(size=(5, 1))
    m0 = rng.normal(size=5)
    mt, mw = m0 + rng.normal(size=5) * 0.1, np.array([3.0, 0.0, 2.0, 1.0, 5.0])
    return lambda b: (mt, mw, m0 + Jm @ b, Jm)


@pytest.mark.parametrize('sigma,pose_w,betas_w,meas', [(math.inf, 0.0, 0.0, False), (30.0, 0.0, 0.0, False),
                                                       (30.0, 5e3, 2e3, True), (math.inf, 1e4, 0.0, True)])
def test_gradient_is_half_the_loss_gradient(sigma, pose_w, betas_w, meas):
    """g = sum_views J^T W r + priors + measurement rows equals half the central-difference gradient of the loss; a
    dropped keypoint with NaN target and rows is never read."""
    evaluate, rng, rot, beta, kp, jac, views = _case(22)
    anchor = np.stack([r @ expm(rng.normal(size=3) * 0.2) for r in rot])
    jac[9:12] = np.nan
    mf = _meas(rng, beta) if meas else None
    _, g, _ = oc.normal_equations(views, kp, jac, T0, sigma, rot, anchor, pose_w, beta, betas_w,
                                  mf(beta) if meas else None)

    def L(theta):
        R, b, t, k = _at(evaluate, rot, beta, theta)
        return oc.loss(views, k, t, sigma, R, anchor, pose_w, b, betas_w, mf(b)[:3] if meas else None)

    h = 1e-6
    fd = np.zeros(10)
    for i in range(10):
        e = np.zeros(10)
        e[i] = h
        fd[i] = (L(e) - L(-e)) / (2 * h)
    assert np.abs(2 * g - fd).max() <= 1e-6 * np.abs(fd).max(), (2 * g, fd)


def test_depth_rule_per_view():
    """A weighted keypoint behind any one view makes the loss +inf (a dropped one is ignored), as does a bad focal
    length in any view; a trial breaking it is rejected, a start breaking it reports NaN and does not move."""
    evaluate, _, rot, beta, kp, jac, (tg, w, intr, ext) = _case(23)
    views = (tg, w, intr, ext)
    assert math.isfinite(oc.loss(views, kp, T0))
    # move keypoint 5 to just behind view 1's camera plane, which the other views still see in front
    R1, T1 = ext[1, :9].reshape(3, 3), ext[1, 9:]
    Y = oc.camera_points(kp, T0, ext[1])
    behind = kp.copy()
    behind[5] = R1.T @ (np.array([Y[5, 0], Y[5, 1], -0.1]) - T1) - T0
    assert oc.camera_points(behind, T0, ext[0])[5, 2] > 0 and oc.camera_points(behind, T0, ext[2])[5, 2] > 0
    assert oc.loss(views, behind, T0) == math.inf
    w2 = w.copy()
    w2[1, 5] = 0.0                             # dropped in that view only
    assert math.isfinite(oc.loss((tg, w2, intr, ext), behind, T0))
    for f in (0.0, -1000.0, math.nan, math.inf):
        bad = intr.copy()
        bad[2, 0] = f
        assert oc.loss((tg, w, bad, ext), kp, T0) == math.inf
    state = {'rot': rot, 'betas': beta, 'transl': T0, 'keypoints': kp, 'jac': jac, 'lambda': np.float32(1e-3),
             'loss': np.float32(oc.loss(views, kp, T0))}
    trial = {'rot': rot, 'betas': beta, 'transl': T0}
    new, nxt, acc = oc.lm_keypoints_2d_calibrated_step(state, views, 10.0, 3.0, False, trial, behind, jac)
    assert not acc and new['loss'] == state['loss']
    new, nxt, acc = oc.lm_keypoints_2d_calibrated_step({}, views, 10.0, 3.0, True, trial, behind, jac)
    assert acc and math.isnan(new['loss'])
    assert all(np.array_equal(nxt[k], np.asarray(trial[k], np.float32)) for k in ('rot', 'betas', 'transl'))


@pytest.mark.parametrize('first', [True, False])
@pytest.mark.parametrize('sigma,pose_w,betas_w', [(math.inf, 0.0, 0.0), (30.0, 5e3, 2e3)])
def test_one_identity_view_is_the_perspective_step(first, sigma, pose_w, betas_w):
    evaluate, rng, rot, beta, kp, jac, _ = _case(24)
    t = np.array([0.1, -0.2, 5.0])
    tg = o2.project(kp, t, INTR) + rng.normal(size=(12, 2)) * 20.0
    w = rng.uniform(0.5, 1.5, 12)
    w[3], tg[3] = 0.0, np.nan
    ident = np.concatenate([np.eye(3).reshape(9), np.zeros(3)])
    views = (tg[None], w[None], INTR[None], ident[None])
    anchor = np.stack([r @ expm(rng.normal(size=3) * 0.2) for r in rot])
    A1, g1, d1 = oc.normal_equations(views, kp, jac, t, sigma, rot, anchor, pose_w, beta, betas_w)
    A2, g2, d2 = o2.normal_equations(tg, w, kp, jac, t, sigma, rot, anchor, pose_w, beta, betas_w, intr=INTR)
    for a, b in ((A1, A2), (g1, g2), (d1, d2)):
        assert np.abs(a - b).max() <= 1e-12 * np.abs(b).max()
    assert abs(oc.loss(views, kp, t, sigma, rot, anchor, pose_w, beta, betas_w) -
               o2.loss(tg, w, kp, t, sigma, rot, anchor, pose_w, beta, betas_w, intr=INTR)) <= 1e-12 * abs(o2.loss(
                   tg, w, kp, t, sigma, rot, anchor, pose_w, beta, betas_w, intr=INTR))
    trial_kp, trial_jac = evaluate(np.stack([r @ expm(rng.normal(size=3) * 0.05) for r in rot]), beta + 0.05)
    state = {'rot': rot, 'betas': beta, 'transl': t, 'keypoints': kp, 'jac': jac, 'lambda': np.float32(1e-2),
             'loss': np.float32(o2.loss(tg, w, kp, t, sigma, rot, anchor, pose_w, beta, betas_w, intr=INTR))}
    trial = {'rot': rot, 'betas': beta + 0.05, 'transl': t + 0.01}
    kw = dict(sigma=sigma, anchor=anchor, pose_w=pose_w, betas_w=betas_w, dtype=np.float64)
    n1, x1, a1 = oc.lm_keypoints_2d_calibrated_step(state, views, 10.0, 3.0, first, trial, trial_kp, trial_jac, **kw)
    n2, x2, a2 = o2.lm_keypoints_2d_step(state, tg, w, 10.0, 3.0, first, trial, trial_kp, trial_jac, intr=INTR, **kw)
    assert a1 == a2 and n1['accepted'] == n2['accepted']
    assert abs(n1['lambda'] - n2['lambda']) <= 1e-12 * n2['lambda']
    for k in ('rot', 'betas', 'transl'):
        assert np.abs(x1[k] - x2[k]).max() <= 1e-12 * max(1.0, np.abs(x2[k]).max()), k


@pytest.mark.parametrize('sigma', [math.inf, 50.0])
def test_fp64_lm_on_a_noiseless_four_camera_rig_recovers_pose_shape_and_world_translation(sigma):
    evaluate, rng = toy_problem(25)
    R1, R2 = expm(rng.normal(size=3) * 0.6), expm(rng.normal(size=3) * 0.6)
    bstar, tstar = np.array([0.6]), np.array([0.3, -0.1, 0.4])
    kp, _ = evaluate(np.stack([R1, R2]), bstar)
    ext = np.stack([_look_at(a) for a in (0.0, 90.0, 180.0, 270.0)])
    intr = np.tile(INTR, (4, 1))
    tg = np.stack([oc.project(kp, tstar, intr[v], ext[v]) for v in range(4)])
    w = np.ones((4, 12))
    w[1, 2], tg[1, 2] = 0.0, np.nan
    views = (tg, w, intr, ext)
    trial = {'rot': np.stack([R1 @ expm(rng.normal(size=3) * 0.2), R2 @ expm(rng.normal(size=3) * 0.2)]),
             'betas': np.zeros(1), 'transl': tstar + np.array([0.1, 0.1, -0.2])}
    state, losses = {}, []
    for it in range(60):
        k, j = evaluate(trial['rot'], trial['betas'])
        state, trial, _ = oc.lm_keypoints_2d_calibrated_step(state, views, 10.0, 3.0, it == 0, trial, k, j,
                                                             sigma=sigma, dtype=np.float64)
        losses.append(float(state['loss']))
    assert all(b <= a for a, b in zip(losses, losses[1:])), losses
    assert losses[-1] < 1e-12, losses
    assert np.abs(state['transl'] - tstar).max() < 1e-6 and np.abs(state['betas'] - bstar).max() < 1e-6
    assert np.abs(state['rot'][0] - R1).max() < 1e-6 and np.abs(state['rot'][1] - R2).max() < 1e-6


def _smplx():
    from shapy_b200 import synth
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    return SMPLX(data_struct=synth.make_smplx())


def test_calibrated_start_matches_a_float64_forward():
    """A body posed in one camera's frame (R_c, t_c) and the world body calibrated_start maps it to are the same points
    in that camera: R_v X_world + T_v = X_camera, vertex for vertex, in a float64 SMPL-X forward."""
    from oracle import smplx_oracle
    from shapy_b200.fit import calibrated_start
    module = _smplx()
    model = {k: v for k, v in module.state_dict().items()}
    model['parents'] = module.parents
    gen = torch.Generator().manual_seed(3)
    B = 6
    rot = smplx_oracle.decode_6d(torch.randn(B * 22, 6, generator=gen, dtype=torch.float64)).reshape(B, 22, 3, 3)
    betas = torch.randn(B, module.num_betas, generator=gen, dtype=torch.float64)
    tc = torch.randn(B, 3, generator=gen, dtype=torch.float64) + torch.tensor([0.0, 0.0, 4.0], dtype=torch.float64)
    rng = np.random.default_rng(4)
    ext = torch.from_numpy(np.stack([_rand_ext(rng) for _ in range(B)]))
    Rv, Tv = ext[:, :9].reshape(B, 3, 3), ext[:, 9:]
    R0w, tw = calibrated_start(module, rot[:, 0], tc, betas, Rv, Tv)
    # the vertices: the dynamic face-contour landmarks among the joints follow the head's global rotation, so they are
    # not a rigid function of the body
    cam = smplx_oracle.smplx_forward_full(model, betas, rot, transl=tc)['vertices']
    world_rot = torch.cat([R0w.double()[:, None], rot[:, 1:]], 1)
    world = smplx_oracle.smplx_forward_full(model, betas, world_rot, transl=tw.double())['vertices']
    back = torch.einsum('bij,bkj->bki', Rv, world) + Tv[:, None]
    err = float((back - cam).abs().max())
    print(f'[kp2d calibrated] calibrated_start: max vertex error {err:.2e} m')
    assert err <= 1e-5                          # float32 rotations, translations and J_0


def test_default_translation_start_is_exact_on_noiseless_rays():
    """Views of one body whose weighted keypoints' centroids project a world point p: the start is p (to the ray
    weight's 1e-6 pull); with one view, the point START_DEPTH in front of it on its ray."""
    from shapy_b200.fit import START_DEPTH, _ray_start
    rng = np.random.default_rng(5)
    V, K = 4, 7
    p = np.array([0.3, -0.4, 0.2])
    ext = np.stack([_look_at(a, radius=3.0) for a in (0.0, 90.0, 180.0, 270.0)])
    intr = np.tile(INTR, (V, 1))
    x = np.zeros((V, K, 2))
    for v in range(V):
        c = oc.project(p[None], np.zeros(3), intr[v], ext[v])[0]
        d = rng.normal(size=(K - 1, 2)) * 30.0
        x[v, :K - 1] = c + d - d.mean(0)           # the weighted keypoints' centroid is p's projection
        x[v, K - 1] = 1e4                          # dropped
    w = np.ones((V, K))
    w[:, K - 1] = 0.0
    f = lambda a: torch.from_numpy(np.ascontiguousarray(a)).float()  # noqa: E731
    R, T = f(ext[:, :9].reshape(V, 3, 3)), f(ext[:, 9:])
    off = torch.tensor([0, 2, 4], dtype=torch.int32)
    got = _ray_start(f(x), f(w), f(intr), R, T, off).double().numpy()
    assert np.abs(got - p).max() <= 1e-5, got
    one = _ray_start(f(x[:1]), f(w[:1]), f(intr[:1]), R[:1], T[:1], torch.tensor([0, 1], dtype=torch.int32))
    Y = oc.camera_points(one.double().numpy(), np.zeros(3), ext[0])[0]
    assert abs(Y[2] - START_DEPTH) <= 1e-5
    c = oc.project(p[None], np.zeros(3), intr[0], ext[0])[0]
    assert np.abs(INTR[0] * Y[:2] / Y[2] + INTR[1:] - c).max() <= 1e-3      # on view 0's ray through p
