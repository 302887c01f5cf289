"""CPU: the float64 restatement of the perspective 2D keypoint LM step (tests/kp2d_lm_oracle.py with intrinsics) pinned to
central differences of its projection and loss (all columns, t included), the depth rule, a plain fp64 LM on a small
nonlinear problem with rotations, a betas and the translation; fit.perspective_start against the crop projection; and
PerspectiveCamera against the reference class's outputs."""
import math
import os

import numpy as np
import pytest
import torch

import kp2d_lm_oracle as o2
from lm_harness import expm, toy_problem

INTR = np.array([1000.0, 500.0, 480.0])
T0 = np.array([0.1, -0.2, 5.0])              # the toy keypoints are ~N(0, 1): 5 m keeps them in front


def _case(seed, sigma_noise=20.0):
    evaluate, rng = toy_problem(seed)
    rot = np.stack([expm(rng.normal(size=3) * 0.5) for _ in range(2)])
    beta = np.array([0.3])
    kp, jac = evaluate(rot, beta)
    tg = o2.project(kp, T0, INTR) + rng.normal(size=(12, 2)) * sigma_noise
    w = rng.uniform(0.5, 1.5, 12)
    w[3], tg[3] = 0.0, np.nan
    return evaluate, rng, rot, beta, kp, jac, tg, w


def _at(evaluate, rot, beta, theta):
    """(rotations, betas, t, keypoints) at the offsets theta = [delta_0, delta_1 | beta | t]."""
    R = np.stack([rot[j] @ expm(theta[3 * j:3 * j + 3]) for j in range(2)])
    b = beta + theta[6:7]
    kp, _ = evaluate(R, b)
    return R, b, T0 + theta[7:], kp


def test_projected_jacobian_vs_central_differences_on_every_column():
    evaluate, _, rot, beta, kp, jac, _, _ = _case(11)
    jac[:, 7:] = 7.0                          # the 3D transl columns are not read: J_t = I
    J2 = o2.jacobian_persp(kp, jac, T0, INTR)
    h = 1e-6
    fd = np.zeros((24, 10))
    for i in range(10):
        e = np.zeros(10)
        e[i] = h
        a, b = _at(evaluate, rot, beta, e), _at(evaluate, rot, beta, -e)
        fd[:, i] = (o2.project(a[3], a[2], INTR) - o2.project(b[3], b[2], INTR)).reshape(-1) / (2 * h)
    assert np.abs(J2 - fd).max() <= 1e-6 * np.abs(fd).max()


@pytest.mark.parametrize('sigma,pose_w,betas_w', [(math.inf, 0.0, 0.0), (30.0, 0.0, 0.0), (30.0, 5e3, 2e3),
                                                  (math.inf, 1e4, 0.0)])
def test_gradient_is_half_the_loss_gradient(sigma, pose_w, betas_w):
    """g = J^T W r + priors equals half the central-difference gradient of the loss: the perspective rows, the IRLS
    weights, the pose-prior rows and betas_w beta; a dropped keypoint with NaN target and rows is never read."""
    evaluate, rng, rot, beta, kp, jac, tg, w = _case(12)
    anchor = np.stack([r @ expm(rng.normal(size=3) * 0.2) for r in rot])
    jac[9:12] = np.nan
    _, g, _ = o2.normal_equations(tg, w, kp, jac, T0, sigma, rot, anchor, pose_w, beta, betas_w, intr=INTR)

    def L(theta):
        R, b, t, k = _at(evaluate, rot, beta, theta)
        return o2.loss(tg, w, k, t, sigma, R, anchor, pose_w, b, betas_w, intr=INTR)

    h = 1e-6
    fd = np.zeros(10)
    for i in range(10):
        e = np.zeros(10)
        e[i] = h
        fd[i] = (L(e) - L(-e)) / (2 * h)
    assert np.abs(2 * g - fd).max() <= 1e-6 * np.abs(fd).max(), (2 * g, fd)


def test_depth_rule():
    """A weighted keypoint at Y_z <= 0 makes the loss +inf and the trial is rejected; a dropped one is ignored; a bad
    focal length is +inf; a start behind the camera reports NaN and does not move."""
    evaluate, _, rot, beta, kp, jac, tg, w = _case(13)
    assert math.isfinite(o2.loss(tg, w, kp, T0, intr=INTR))
    behind = kp.copy()
    behind[5, 2] = -T0[2] - 0.1              # Y_z = -0.1
    assert o2.loss(tg, w, behind, T0, intr=INTR) == math.inf
    behind[5, 2] = -T0[2]                    # Y_z = 0
    assert o2.loss(tg, w, behind, T0, intr=INTR) == math.inf
    dropped = kp.copy()
    dropped[3, 2] = -T0[2] - 1.0             # keypoint 3 has weight 0
    assert o2.loss(tg, w, dropped, T0, intr=INTR) == o2.loss(tg, w, kp, T0, intr=INTR)
    for f in (0.0, -1000.0, math.nan, math.inf):
        assert o2.loss(tg, w, kp, T0, intr=[f, 500.0, 480.0]) == math.inf
    state = {'rot': rot, 'betas': beta, 'transl': T0, 'keypoints': kp, 'jac': jac, 'lambda': np.float32(1e-3),
             'loss': np.float32(o2.loss(tg, w, kp, T0, intr=INTR))}
    trial = {'rot': rot, 'betas': beta, 'transl': T0}
    new, nxt, acc = o2.lm_keypoints_2d_step(state, tg, w, 10.0, 3.0, False, trial, behind, jac, intr=INTR)
    assert not acc and new['loss'] == state['loss']
    new, nxt, acc = o2.lm_keypoints_2d_step({}, tg, w, 10.0, 3.0, True, trial, behind, jac, intr=INTR)
    assert acc and math.isnan(new['loss'])
    assert all(np.array_equal(nxt[k], np.asarray(trial[k], np.float32)) for k in ('rot', 'betas', 'transl'))


@pytest.mark.parametrize('sigma', [math.inf, 50.0])
def test_fp64_lm_recovers_rotations_shape_and_translation(sigma):
    evaluate, rng = toy_problem(14)
    R1, R2 = expm(rng.normal(size=3) * 0.6), expm(rng.normal(size=3) * 0.6)
    bstar, tstar = np.array([0.6]), np.array([0.3, -0.1, 4.0])
    kp, _ = evaluate(np.stack([R1, R2]), bstar)
    tg = o2.project(kp, tstar, INTR)
    w = np.ones(12)
    w[2], tg[2] = 0.0, np.nan
    trial = {'rot': np.stack([R1 @ expm(rng.normal(size=3) * 0.2), R2 @ expm(rng.normal(size=3) * 0.2)]),
             'betas': np.zeros(1), 'transl': tstar + np.array([0.1, 0.1, 0.8])}
    state, losses = {}, []
    for it in range(60):
        k, j = evaluate(trial['rot'], trial['betas'])
        state, trial, _ = o2.lm_keypoints_2d_step(state, tg, w, 10.0, 3.0, it == 0, trial, k, j, sigma=sigma,
                                                  intr=INTR, dtype=np.float64)
        losses.append(float(state['loss']))
    assert all(b <= a for a, b in zip(losses, losses[1:])), losses
    assert losses[-1] < 1e-12, losses
    assert np.abs(state['transl'] - tstar).max() < 1e-6 and np.abs(state['betas'] - bstar).max() < 1e-6


def _crop_to_pixels(u, center, scale):
    """The inverse of keypoints2d.to_crop without its +1 and rounding: x = center + u h / 2."""
    return center[:, None] + u * (100.0 * scale)[:, None, None]


def test_perspective_start_reproduces_the_crop_projection():
    from shapy_b200.fit import perspective_start
    gen = torch.Generator().manual_seed(3)
    B = 16
    cam = torch.stack([0.9 + 0.3 * torch.randn(B, generator=gen), 0.1 * torch.randn(B, generator=gen),
                       0.1 * torch.randn(B, generator=gen)], 1).double()
    center = torch.rand(B, 2, generator=gen).double() * 800 + 100
    scale = torch.rand(B, generator=gen).double() * 3 + 2
    f, pp = 1200.0, torch.tensor([512.0, 384.0], dtype=torch.float64)
    t = perspective_start(cam.float(), center, scale, f, pp).double()
    s = torch.nn.functional.softplus(cam[:, 0])
    # points in the plane Y_z = t_z: exact
    X = torch.randn(B, 40, 3, generator=gen).double() * 0.5
    X[..., 2] = 0.0
    crop = s[:, None, None] * (X[..., :2] + cam[:, None, 1:3])
    want = _crop_to_pixels(crop, center, scale)
    Y = X + t[:, None]
    got = f * Y[..., :2] / Y[..., 2:] + pp
    assert float((got - want).abs().max()) <= 1e-3                 # pixels; float32 t
    # a posed body with depth extent |dz| <= d: a point moves towards the principal point by dz / (t_z + dz) of its
    # offset, at most d / (t_z - d)
    d = 0.2
    X[..., 2] = (torch.rand(B, 40, generator=gen).double() * 2 - 1) * d
    Y = X + t[:, None]
    got = f * Y[..., :2] / Y[..., 2:] + pp
    bound = (want - pp).abs() * (d / (t[:, 2] - d))[:, None, None] + 1e-3
    assert bool(((got - want).abs() <= bound).all())
    assert float((got - want).abs().max()) > 1.0                   # and the depth does show


def test_perspective_camera_matches_the_reference_class():
    """ref_persp_camera.npz: the reference's PerspectiveCamera (regressor/human_shape/models/camera/
    camera_projection.py) on random points with a rotation, translation, per-body focal length and camera centre, and
    with the defaults of the focal length (5000), rotation and camera centre."""
    from shapy_b200.human_shape.models.camera.camera_projection import PerspectiveCamera
    g = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'ref_persp_camera.npz'))
    pts, R, t, f, c = (torch.from_numpy(g[k]) for k in ('points', 'rotation', 'translation', 'focal_length', 'center'))
    cam = PerspectiveCamera()
    out = cam(pts, focal_length=f, translation=t, rotation=R, camera_center=c)
    assert torch.allclose(out, torch.from_numpy(g['full']), rtol=1e-6, atol=1e-3)
    out = cam(pts + torch.tensor([0.0, 0.0, 5.0]), translation=torch.zeros(pts.shape[0], 3))
    assert torch.allclose(out, torch.from_numpy(g['defaults']), rtol=1e-6, atol=1e-3)
