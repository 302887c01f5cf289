"""CPU: the float64 restatement of the 2D keypoint LM step (tests/kp2d_lm_oracle.py) pinned to central differences of
its float64 loss (projected Jacobian, IRLS weights, pose-prior rows), to the 3D oracle's normal equations at sigma = inf
without priors, and run as a plain fp64 LM on a small nonlinear problem with rotations and a camera."""
import math

import numpy as np
import pytest

import kp2d_lm_oracle as o2
from test_fit_lm_keypoints_cpu import _rodrigues


def _skew(d):
    return np.array([[0.0, -d[2], d[1]], [d[2], 0.0, -d[0]], [-d[1], d[0], 0.0]])


def _expm(d):
    return _rodrigues(np.asarray(d, np.float64)).numpy()


def _problem(seed, K=12):
    """Keypoints kp = R0 p (first half), R0 R1 p (second half) + beta q + t: two chained rotations, one betas, and
    its (3K, 10) Jacobian with the transl columns last (P = 3 * 2 + 1 + 3)."""
    rng = np.random.default_rng(seed)
    p = rng.normal(size=(K, 3))
    q = rng.normal(size=(K, 3)) * 0.2
    t = rng.normal(size=3) * 0.1
    half = K // 2

    def evaluate(rot, beta):
        kp = np.zeros((K, 3))
        kp[:half] = p[:half] @ rot[0].T
        kp[half:] = p[half:] @ (rot[0] @ rot[1]).T
        kp += beta[0] * q + t
        jac = np.zeros((3 * K, 10))
        for k in range(K):
            x = kp[k] - beta[0] * q[k] - t
            for a in range(3):
                jac[3 * k:3 * k + 3, a] = np.cross(rot[0][:, a], x)
                if k >= half:
                    jac[3 * k:3 * k + 3, 3 + a] = np.cross((rot[0] @ rot[1])[:, a], x)
            jac[3 * k:3 * k + 3, 6] = q[k]
            jac[3 * k:3 * k + 3, 7:] = np.eye(3)
        return kp, jac
    return evaluate, rng


def _full_loss(evaluate, rot, beta, cam, theta, tg, w, sigma, anchor, pose_w, betas_w):
    """The loss at the offsets theta = [delta_0, delta_1 | beta | c0 c1 c2] in float64."""
    R = np.stack([rot[j] @ _expm(theta[3 * j:3 * j + 3]) for j in range(2)])
    b = beta + theta[6:7]
    c = cam + theta[7:]
    kp, _ = evaluate(R, b)
    return o2.loss(tg, w, kp, c, sigma, R, anchor, pose_w, b, betas_w)


@pytest.mark.parametrize('sigma,pose_w,betas_w', [(math.inf, 0.0, 0.0), (0.3, 0.0, 0.0), (0.3, 0.5, 0.2),
                                                  (math.inf, 2.0, 0.0)])
def test_gradient_is_half_the_loss_gradient(sigma, pose_w, betas_w):
    """g = J^T W r + priors equals half the central-difference gradient of the loss: pins the projected Jacobian,
    the IRLS weights w rho'(e) and the pose-prior rows; a dropped keypoint with NaN target is never read."""
    evaluate, rng = _problem(5)
    rot = np.stack([_expm(rng.normal(size=3) * 0.5) for _ in range(2)])
    beta, cam = np.array([0.3]), np.array([0.4, 0.05, -0.1])
    anchor = np.stack([r @ _expm(rng.normal(size=3) * 0.2) for r in rot])
    kp, jac = evaluate(rot, beta)
    tg = o2.project(kp, cam) + rng.normal(size=(12, 2)) * 0.2
    w = rng.uniform(0.5, 1.5, 12)
    w[3], tg[3] = 0.0, np.nan
    jac[9:12] = np.nan
    _, g, _ = o2.normal_equations(tg, w, kp, jac, cam, sigma, rot, anchor, pose_w, beta, betas_w)
    h = 1e-6
    fd = np.zeros(10)
    for i in range(10):
        e = np.zeros(10)
        e[i] = h
        fd[i] = (_full_loss(evaluate, rot, beta, cam, e, tg, w, sigma, anchor, pose_w, betas_w) -
                 _full_loss(evaluate, rot, beta, cam, -e, tg, w, sigma, anchor, pose_w, betas_w)) / (2 * h)
    assert np.abs(2 * g - fd).max() <= 1e-6 * np.abs(fd).max(), (2 * g, fd)


def test_projected_jacobian_and_prior_block_vs_central_differences():
    evaluate, rng = _problem(6)
    rot = np.stack([_expm(rng.normal(size=3) * 0.5) for _ in range(2)])
    beta, cam = np.array([-0.2]), np.array([-0.3, 0.1, 0.2])
    kp, jac = evaluate(rot, beta)
    J2 = o2.jacobian_2d(kp, jac, cam)
    h = 1e-6

    def proj(theta):
        R = np.stack([rot[j] @ _expm(theta[3 * j:3 * j + 3]) for j in range(2)])
        k, _ = evaluate(R, beta + theta[6:7])
        return o2.project(k, cam + theta[7:]).reshape(-1), (R[1] / math.sqrt(2)).reshape(-1)

    fd, fdp = np.zeros((24, 10)), np.zeros((9, 10))
    for i in range(10):
        e = np.zeros(10)
        e[i] = h
        (a, pa), (b, pb) = proj(e), proj(-e)
        fd[:, i], fdp[:, i] = (a - b) / (2 * h), (pa - pb) / (2 * h)
    assert np.abs(J2 - fd).max() <= 1e-7 * np.abs(fd).max()
    # the pose-prior rows (R_1 - R0_1) / sqrt(2): their normal-matrix block equals Jp^T Jp of the differences
    anchor = rot.copy()
    A0, _, _ = o2.normal_equations(np.zeros((12, 2)), np.zeros(12), kp, jac, cam, math.inf, rot, anchor, 0.0, beta)
    A1, _, dg = o2.normal_equations(np.zeros((12, 2)), np.zeros(12), kp, jac, cam, math.inf, rot, anchor, 3.0, beta)
    assert np.abs((A1 - A0) - 3.0 * fdp.T @ fdp).max() <= 1e-7 and np.array_equal(dg, np.diag(A0))


def test_normal_equations_equal_the_3d_rows_after_the_camera_transform():
    """sigma = inf and no priors: A and g equal those of the 3D oracle's rows restricted to x and y, with the rotation
    and betas columns scaled by s and the transl columns replaced by the camera's."""
    evaluate, rng = _problem(7)
    rot = np.stack([_expm(rng.normal(size=3) * 0.5) for _ in range(2)])
    beta, cam = np.array([0.1]), np.array([0.7, -0.05, 0.02])
    kp, jac = evaluate(rot, beta)
    tg = o2.project(kp, cam) + rng.normal(size=(12, 2)) * 0.1
    w = rng.uniform(0.5, 1.5, 12)
    A, g, _ = o2.normal_equations(tg, w, kp, jac, cam, math.inf, rot, None, 0.0, beta)
    s, ds = o2.softplus(cam[0])
    xy = np.concatenate([np.arange(0, 36, 3), np.arange(1, 36, 3)])
    xy.sort()
    J = jac[xy].copy()
    J[:, :7] *= s
    J[:, 7] = ds * (kp[:, :2] + cam[1:]).reshape(-1)
    J[:, 8:] = np.tile(np.eye(2) * s, (12, 1))
    W = np.repeat(w, 2)
    r = (s * (kp[:, :2] + cam[1:]) - tg).reshape(-1)
    assert np.allclose(A, J.T @ (W[:, None] * J), rtol=1e-12, atol=1e-12)
    assert np.allclose(g, J.T @ (W * r), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize('sigma', [math.inf, 0.5])
def test_fp64_lm_recovers_rotations_shape_and_camera(sigma):
    evaluate, rng = _problem(8)
    R1, R2 = _expm(rng.normal(size=3) * 0.6), _expm(rng.normal(size=3) * 0.6)
    bstar, cstar = np.array([0.6]), np.array([0.5, 0.1, -0.05])
    kp, _ = evaluate(np.stack([R1, R2]), bstar)
    tg = o2.project(kp, cstar)
    w = np.ones(12)
    w[2], tg[2] = 0.0, np.nan
    trial = {'rot': np.stack([R1 @ _expm(rng.normal(size=3) * 0.2), R2 @ _expm(rng.normal(size=3) * 0.2)]),
             'betas': np.zeros(1), 'camera': np.array([0.3, 0.0, 0.0])}
    state, losses = {}, []
    for it in range(60):
        k, j = evaluate(trial['rot'], trial['betas'])
        state, trial, _ = o2.lm_keypoints_2d_step(state, tg, w, 10.0, 3.0, it == 0, trial, k, j, sigma=sigma,
                                                  dtype=np.float64)
        losses.append(float(state['loss']))
    assert all(b <= a for a, b in zip(losses, losses[1:])), losses
    assert losses[-1] < 1e-16, losses
