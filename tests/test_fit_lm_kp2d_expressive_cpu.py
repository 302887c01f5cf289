"""CPU: the float64 restatement of the whole-body 2D keypoint LM step (tests/kp2d_lm_oracle.py).  Its expression
and wide rotation columns against central differences of the float64 forward (tests/smplx_grad_ref.py); its packed
solve against a dense solve at P = 7, 79, 188 and 200; at n_rot = 22 a width-0 expression is the step without one, for
the weak-perspective and perspective cameras; a plain fp64 LM loop over the wide parameters never raises the loss.  The
command line refuses the wide flags outside the single-image 2D fit."""
import math

import numpy as np
import pytest
import torch

import kp2d_lm_oracle as o2
from kp_lm_oracle import keypoint_jacobian
from oracle.lm_oracle import cholesky_solve
from shapy_b200 import synth
from smplx_grad_ref import forward_differentiable
from lm_harness import expm


def _model():
    return dict(synth.make_smplx())


def _rotations(rng, n, scale):
    return np.stack([expm(rng.normal(size=3) * scale) for _ in range(n)])


def test_expression_and_wide_rotation_columns_vs_central_differences():
    m = _model()
    rng = np.random.default_rng(3)
    n_rot, NB, NE = 55, 10, 10
    rot = _rotations(rng, n_rot, 0.3)
    beta, psi = rng.normal(size=NB) * 0.5, rng.normal(size=NE)
    kp, jac = keypoint_jacobian(m, beta, rot, expr=psi)
    out = forward_differentiable(m, torch.tensor(beta)[None], torch.tensor(rot)[None], torch.tensor(psi)[None])
    assert np.abs(kp - out['joints'][0].numpy()).max() <= 1e-9
    h = 1e-6
    o = 3 * n_rot + NB

    def joints(rot_, psi_):
        return forward_differentiable(m, torch.tensor(beta)[None], torch.tensor(rot_)[None],
                                      torch.tensor(psi_)[None])['joints'][0].numpy().reshape(-1)
    for l in (0, 4, NE - 1):                      # expression columns
        e = np.zeros(NE)
        e[l] = h
        fd = (joints(rot, psi + e) - joints(rot, psi - e)) / (2 * h)
        assert np.abs(jac[:, o + l] - fd).max() <= 1e-6 * max(1.0, np.abs(fd).max()), l
    for j, a in ((22, 0), (24, 1), (30, 2), (54, 1)):   # jaw, right eye, hand joints
        d = np.zeros(3)
        d[a] = h
        rp, rm = rot.copy(), rot.copy()
        rp[j], rm[j] = rot[j] @ expm(d), rot[j] @ expm(-d)
        fd = (joints(rp, psi) - joints(rm, psi)) / (2 * h)
        assert np.abs(jac[:, 3 * j + a] - fd).max() <= 1e-6 * max(1.0, np.abs(fd).max()), (j, a)


@pytest.mark.parametrize('P', [7, 79, 188, 200])
def test_packed_solve_is_the_dense_solve(P):
    rng = np.random.default_rng(P)
    X = rng.normal(size=(P + 20, P))
    A = X.T @ X + 0.1 * np.eye(P)
    g = rng.normal(size=P)
    y, ok = o2.packed_solve(A.copy(), g.copy())
    yd, okd = cholesky_solve(A.copy(), g.copy())
    assert ok and okd
    assert np.array_equal(y, yd)                  # the same operations in the same order
    ref = np.linalg.solve(A, -g)
    assert np.abs(y - ref).max() <= 1e-9 * np.abs(ref).max()
    A[3, 3] = -1.0
    assert not o2.packed_solve(A, g)[1]


def _toy(seed, n_rot, nb, ne, K):
    rng = np.random.default_rng(seed)
    P = 3 * n_rot + nb + ne + 3
    return rng, dict(rot=_rotations(rng, n_rot, 0.4), betas=rng.normal(size=nb), expression=rng.normal(size=ne),
                     kp=rng.normal(size=(K, 3)) * 0.4, jac=rng.normal(size=(3 * K, P)) * 0.3)


@pytest.mark.parametrize('persp', [False, True])
@pytest.mark.parametrize('first', [False, True])
def test_no_expression_at_22_joints_is_todays_oracle(first, persp):
    rng, c = _toy(5 + persp, 22, 10, 0, 30)
    lk = 'transl' if persp else 'camera'
    last = np.array([0.1, -0.2, 4.0]) if persp else np.array([1.0, 0.1, -0.1])
    intr = np.array([1000.0, 500.0, 480.0]) if persp else None
    tg = o2.project(c['kp'], last, intr) + \
        rng.normal(size=(30, 2)) * (5.0 if persp else 0.02)
    w = rng.uniform(0.5, 1.5, 30)
    anchor = np.stack([r @ expm(rng.normal(size=3) * 0.1) for r in c['rot']])
    f32 = lambda x: np.asarray(x, np.float32)  # noqa: E731
    state = {'rot': f32(c['rot']), 'betas': f32(c['betas']), lk: f32(last), 'keypoints': f32(c['kp']),
             'jac': f32(c['jac']), 'loss': np.float32(50.0), 'lambda': np.float32(0.3), 'accepted': 0}
    trial = {'rot': f32(np.stack([r @ expm(rng.normal(size=3) * 0.05) for r in c['rot']])),
             'betas': f32(c['betas'] + 0.05), lk: f32(last + 0.01)}
    tkp, tjac = f32(c['kp'] + 0.01), f32(c['jac'] * 1.01)
    sigma = 20.0 if persp else 0.3
    kw = dict(sigma=sigma, anchor=anchor, pose_w=2.0, betas_w=0.1)
    want = o2.lm_keypoints_2d_step(state, tg, w, 10.0, 3.0, first, trial, tkp, tjac, intr=intr, **kw)
    sx = dict(state, expression=np.zeros(0, np.float32))
    tx = dict(trial, expression=np.zeros(0, np.float32))
    got = o2.lm_keypoints_2d_step(sx, tg, w, 10.0, 3.0, first, tx, tkp, tjac, intr=intr, **kw)
    assert got[2] == want[2]
    for k in ('rot', 'betas', lk, 'keypoints', 'jac', 'loss', 'lambda', 'accepted'):
        assert np.array_equal(got[0][k], want[0][k]), k
    for k in ('rot', 'betas', lk):
        assert np.array_equal(got[1][k], want[1][k]), k


@pytest.mark.parametrize('persp', [False, True])
def test_fp64_lm_loop_never_raises_the_loss(persp):
    """A plain fp64 LM (dtype float64) over 25 rotations, betas and the expression on the synthetic SMPL-X, the
    Jacobian from the float64 restatement, with a robust loss, per-joint priors and both regularisers."""
    m = _model()
    rng = np.random.default_rng(11 + persp)
    n_rot, NB, NE = 25, 10, 10
    rot_t = _rotations(rng, n_rot, 0.25)
    beta_t, psi_t = rng.normal(size=NB) * 0.5, rng.normal(size=NE)
    lk = 'transl' if persp else 'camera'
    last_t = np.array([0.1, -0.2, 4.0]) if persp else np.array([1.0, 0.05, -0.05])
    intr = np.array([1000.0, 500.0, 480.0]) if persp else None
    kp_t, _ = keypoint_jacobian(m, beta_t, rot_t, expr=psi_t)
    tg = o2.project(kp_t, last_t, intr)
    K = tg.shape[0]
    w = np.ones(K)
    jw = np.zeros(n_rot)
    jw[1:22], jw[22:] = 0.5, 0.1
    trial = {'rot': np.stack([r @ expm(rng.normal(size=3) * 0.1) for r in rot_t]), 'betas': beta_t + 0.3,
             'expression': np.zeros(NE), lk: last_t + (np.array([0.02, 0.02, 0.3]) if persp else 0.05)}
    anchor = trial['rot'].copy()
    state = {'accepted': 0}
    kw = dict(sigma=30.0 if persp else 0.2, anchor=anchor, joint_w=jw, betas_w=0.01, expr_w=0.001, intr=intr,
              dtype=np.float64)
    losses = []
    for it in range(8):
        kp, jac = keypoint_jacobian(m, trial['betas'], trial['rot'], expr=trial['expression'])
        state, trial, _ = o2.lm_keypoints_2d_step(state, tg, w, 10.0, 3.0, it == 0, trial, kp, jac, **kw)
        losses.append(float(state['loss']))
    assert all(b <= a for a, b in zip(losses, losses[1:])), losses
    assert losses[-1] < 0.5 * losses[0], losses
    assert math.isfinite(losses[-1])


@pytest.mark.parametrize('extra', [['--calibrated'], ['--sequence'], []])
@pytest.mark.parametrize('wide', [['--pose-width', '55'], ['--fit-expression'], ['--expression-weight', '0.1']])
def test_cli_refuses_the_wide_flags_outside_the_single_image_2d_fit(tmp_path, wide, extra):
    """The calibrated and sequence fits, and the betas fit without --keypoints-2d, have no hands or expression: the
    command line refuses the wide flags there instead of fitting the 22-joint body."""
    from shapy_b200.fit import main
    kp = [] if extra == [] else ['--keypoints-2d', str(tmp_path / 'kp.npz')]
    with pytest.raises(SystemExit, match='--pose-width'):
        main(['--synthetic', *kp, *extra, *wide])
