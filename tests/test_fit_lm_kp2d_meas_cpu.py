"""CPU: the float64 restatement of the stacked 2D keypoint + measurement LM step (tests/kp2d_lm_oracle.py) pinned to
J^T W J and J^T W r of the explicitly stacked Jacobian (projected keypoint rows, pose-prior rows, measurement rows), to
the step without measurements when every measurement is dropped, on NaN in dropped and in weighted measurements, and run as a plain
fp64 LM on a small nonlinear problem."""
import math

import numpy as np
import pytest

import kp2d_lm_oracle as o2
from lm_harness import expm, toy_problem

P = 10              # toy_problem: two rotations, one betas, the camera
MW = np.array([1.0, 100.0, 2000.0, 1000.0, 1000.0])


def _measure(beta):
    """Five toy measurements of the one betas, smooth and nonlinear, and their (5, 1) Jacobian."""
    a = np.array([70.0, 1.7, 1.0, 0.9, 1.0])
    b = np.array([9.0, 0.08, 0.07, 0.06, 0.05])
    c = np.array([0.8, 0.004, 0.01, 0.008, 0.006])
    x = float(beta[0])
    return a + b * x + c * x * x, (b + 2.0 * c * x)[:, None]


def _case(seed, sigma=0.3, pose_w=0.5, betas_w=0.2):
    evaluate, rng = toy_problem(seed)
    rot = np.stack([expm(rng.normal(size=3) * 0.5) for _ in range(2)])
    beta, cam = np.array([0.3]), np.array([0.4, 0.05, -0.1])
    anchor = np.stack([r @ expm(rng.normal(size=3) * 0.2) for r in rot])
    kp, jac = evaluate(rot, beta)
    tg = o2.project(kp, cam) + rng.normal(size=(12, 2)) * 0.2
    w = rng.uniform(0.5, 1.5, 12)
    w[3], tg[3] = 0.0, np.nan
    jac[9:12] = np.nan
    meas, mjac = _measure(beta)
    mt = meas * (1 + 0.05 * rng.normal(size=5))
    return dict(evaluate=evaluate, rng=rng, rot=rot, beta=beta, cam=cam, anchor=anchor, kp=kp, jac=jac, tg=tg, w=w,
                meas=meas, mjac=mjac, mt=mt, sigma=sigma, pose_w=pose_w, betas_w=betas_w)


@pytest.mark.parametrize('sigma,pose_w,betas_w', [(math.inf, 0.0, 0.0), (0.3, 0.5, 0.2)])
def test_normal_equations_equal_the_stacked_jacobian(sigma, pose_w, betas_w):
    """A = J^T W J and g = J^T W r + betas_w beta with J the projected keypoint rows (IRLS weights), the pose-prior
    rows and the measurement rows stacked explicitly; the measurement rows do not count for the first lambda."""
    c = _case(11, sigma, pose_w, betas_w)
    mw = MW.copy()
    mw[2] = 0.0                                              # a dropped measurement, NaN value and row
    meas, mjac = c['meas'].copy(), c['mjac'].copy()
    meas[2], mjac[2] = np.nan, np.nan
    A, g, dg = o2.normal_equations(c['tg'], c['w'], c['kp'], c['jac'], c['cam'], sigma, c['rot'], c['anchor'], pose_w,
                                   c['beta'], betas_w, meas=(c['mt'], mw, meas, mjac))
    J2 = o2.jacobian_2d(c['kp'], c['jac'], c['cam'])
    p = o2.project(c['kp'], c['cam'])
    rows, wts, res = [], [], []
    for k in range(12):
        if not c['w'][k] > 0:
            continue
        d = p[k] - c['tg'][k]
        q = 1.0 if not math.isfinite(sigma) else sigma ** 2 / (sigma ** 2 + d @ d)
        for ax in range(2):
            rows.append(J2[2 * k + ax])
            wts.append(c['w'][k] * q * q)
            res.append(d[ax])
    nk = len(rows)
    if pose_w > 0:
        D = np.stack([o2.rot_tangent(c['rot'][1], a) for a in range(3)], 1)
        for e in range(9):
            row = np.zeros(P)
            row[3:6] = D[e]
            rows.append(row)
            wts.append(0.5 * pose_w)
            res.append((c['rot'][1] - c['anchor'][1]).reshape(9)[e])
    for m in range(5):
        if mw[m] > 0:
            row = np.zeros(P)
            row[6] = c['mjac'][m, 0]
            rows.append(row)
            wts.append(mw[m])
            res.append(c['meas'][m] - c['mt'][m])
    J, W, r = np.array(rows), np.array(wts), np.array(res)
    gw = J.T @ (W * r)
    gw[6] += float(np.float32(betas_w)) * c['beta'][0]
    Aw = J.T @ (W[:, None] * J)
    assert np.allclose(A, Aw, rtol=1e-12, atol=1e-12 * np.abs(Aw).max())
    assert np.allclose(g, gw, rtol=1e-12, atol=1e-12 * np.abs(gw).max())
    assert np.allclose(dg, np.diag(J[:nk].T @ (W[:nk, None] * J[:nk])), rtol=1e-12, atol=1e-12)
    assert A[6, 6] > dg[6]


def _step_inputs(c, seed=3):
    rng = np.random.default_rng(seed)
    trot = np.stack([r @ expm(rng.normal(size=3) * 0.02) for r in c['rot']])
    tbeta, tcam = c['beta'] + 0.02, c['cam'] + 0.01 * rng.normal(size=3)
    tkp, tjac = c['evaluate'](trot, tbeta)
    tjac[9:12] = np.nan
    tmeas, tmjac = _measure(tbeta)
    state = {'rot': c['rot'], 'betas': c['beta'], 'camera': c['cam'], 'keypoints': c['kp'], 'jac': c['jac'],
             'meas': c['meas'], 'meas_jac': c['mjac'], 'lambda': np.float64(0.05), 'accepted': 0}
    trial = {'rot': trot, 'betas': tbeta, 'camera': tcam}
    return state, trial, tkp, tjac, tmeas, tmjac


def _kw(c):
    return dict(sigma=c['sigma'], anchor=c['anchor'], pose_w=c['pose_w'], betas_w=c['betas_w'], dtype=np.float64)


def _same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k]), equal_nan=True), k


@pytest.mark.parametrize('first', [False, True])
def test_dropped_measurements_reproduce_the_2d_oracle_exactly(first):
    """Every measurement weight <= 0, NaN in the dropped values and rows: state, lambda, loss and next trial equal
    the step without measurements (meas None) exactly, with the robust loss and both priors on."""
    c = _case(12)
    state, trial, tkp, tjac, tmeas, tmjac = _step_inputs(c)
    nan5, nan51 = np.full(5, np.nan), np.full((5, 1), np.nan)
    state = dict(state, meas=nan5, meas_jac=nan51)
    s2 = {k: v for k, v in state.items() if k not in ('meas', 'meas_jac')}
    for s in (state, s2):
        s['loss'] = np.float64(1e9 if not first else np.nan)
    mw = np.array([0.0, -1.0, 0.0, 0.0, -0.0])
    got = o2.lm_keypoints_2d_step(state, c['tg'], c['w'], 10.0, 3.0, first, trial, tkp, tjac, meas=(c['mt'], mw),
                                  trial_meas=(nan5, nan51), **_kw(c))
    want = o2.lm_keypoints_2d_step(s2, c['tg'], c['w'], 10.0, 3.0, first, trial, tkp, tjac, **_kw(c))
    assert got[2] == want[2] and got[2]
    _same({k: v for k, v in got[0].items() if k not in ('meas', 'meas_jac')}, want[0])
    _same(got[1], want[1])


def test_nan_in_a_dropped_measurement_changes_nothing_and_a_weighted_nan_rejects():
    c = _case(13)
    state, trial, tkp, tjac, tmeas, tmjac = _step_inputs(c)
    mw = MW.copy()
    mw[3] = 0.0
    state['loss'] = np.float64(o2.loss(c['tg'], c['w'], c['kp'], c['cam'], c['sigma'], c['rot'], c['anchor'],
                                       c['pose_w'], c['beta'], c['betas_w'], meas=(c['mt'], mw, c['meas'])) * 10)
    args = (c['tg'], c['w'], 10.0, 3.0, False, trial, tkp, tjac)
    kw = dict(_kw(c), meas=(c['mt'], mw))
    base = o2.lm_keypoints_2d_step(state, *args, trial_meas=(tmeas, tmjac), **kw)
    assert base[2]
    # NaN in the dropped measurement, state and trial
    sn = dict(state, meas=state['meas'].copy(), meas_jac=state['meas_jac'].copy())
    tmn, tjn = tmeas.copy(), tmjac.copy()
    for t in (sn['meas'], sn['meas_jac'], tmn, tjn):
        t[3] = np.nan
    got = o2.lm_keypoints_2d_step(sn, *args, trial_meas=(tmn, tjn), **kw)
    assert got[2]
    skip = lambda d: {k: np.delete(v, 3, 0) if k in ('meas', 'meas_jac') else v for k, v in d.items()}  # noqa: E731
    _same(skip(got[0]), skip(base[0]))
    _same(got[1], base[1])
    # a weighted NaN trial measurement: rejected, the state kept, lambda up, the step from the state
    tmn = tmeas.copy()
    tmn[1] = np.nan
    new, nxt, acc = o2.lm_keypoints_2d_step(state, *args, trial_meas=(tmn, tmjac), **kw)
    assert not acc and new['accepted'] == 0 and new['lambda'] == state['lambda'] * 10.0
    for k in ('rot', 'betas', 'camera', 'keypoints', 'meas', 'meas_jac', 'loss'):
        assert np.array_equal(new[k], state[k], equal_nan=True), k
    assert np.isfinite(nxt['betas']).all() and not np.array_equal(nxt['betas'], state['betas'])


@pytest.mark.parametrize('sigma', [math.inf, 0.5])
def test_fp64_lm_loss_non_increasing_and_height_fixes_the_scale(sigma):
    """The targets are the projection of (R*, beta*, c*) and the measurements those of beta*: every iteration's loss is
    non-increasing and the fit ends at a zero of the total loss, the measurements matched."""
    evaluate, rng = toy_problem(8)
    R1, R2 = expm(rng.normal(size=3) * 0.6), expm(rng.normal(size=3) * 0.6)
    bstar, cstar = np.array([0.6]), np.array([0.5, 0.1, -0.05])
    kp, _ = evaluate(np.stack([R1, R2]), bstar)
    tg = o2.project(kp, cstar)
    w = np.ones(12)
    w[2], tg[2] = 0.0, np.nan
    mt, _ = _measure(bstar)
    mw = np.array([1.0, 100.0, 0.0, 0.0, 0.0])              # mass and height
    trial = {'rot': np.stack([R1 @ expm(rng.normal(size=3) * 0.2), R2 @ expm(rng.normal(size=3) * 0.2)]),
             'betas': np.zeros(1), 'camera': np.array([0.3, 0.0, 0.0])}
    state, losses = {}, []
    for it in range(60):
        k, j = evaluate(trial['rot'], trial['betas'])
        m, mj = _measure(trial['betas'])
        state, trial, _ = o2.lm_keypoints_2d_step(state, tg, w, 10.0, 3.0, it == 0, trial, k, j, sigma=sigma,
                                                  meas=(mt, mw), trial_meas=(m, mj), dtype=np.float64)
        losses.append(float(state['loss']))
    assert all(b <= a for a, b in zip(losses, losses[1:])), losses
    assert losses[-1] < 1e-14, losses
    assert abs(float(state['betas'][0]) - 0.6) < 1e-6 and np.abs(state['meas'][:2] - mt[:2]).max() < 1e-6
