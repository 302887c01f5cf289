"""CPU: the float64 restatement of the keypoint Jacobian (tests/kp_lm_oracle.py) against float64 central differences
of the SMPL-X forward with R_j Exp(delta_j) substituted, and its keypoint LM step on a small nonlinear least-squares
problem with rotations."""
import numpy as np
import torch

import kp_lm_oracle
from lm_harness import keypoints_at, rodrigues
from shapy_b200 import synth


def test_oracle_jacobian_vs_central_differences():
    model = synth.make_smplx()
    gen = torch.Generator().manual_seed(4)
    n_rot = 22
    for b, neck in enumerate((1.2, -1.2)):                 # necks turned past both ends of the contour LUT
        rot = rodrigues(torch.randn(n_rot, 3, generator=gen, dtype=torch.float64) * 0.4).float()
        rot[12] = rodrigues(torch.tensor([0.0, neck, 0.0])).float()
        betas = torch.randn(10, generator=gen)
        transl = torch.randn(3, generator=gen) * 0.1
        kp, jac = kp_lm_oracle.keypoint_jacobian(model, betas, rot, transl)
        P = 3 * n_rot + 10 + 3
        assert jac.shape == (3 * 123, P) and kp.shape == (123, 3)
        base = keypoints_at(model, betas, rot, transl, torch.zeros(1, P, dtype=torch.float64))[0].numpy()
        assert np.abs(kp - base).max() <= 1e-9 * np.abs(base).max()
        h = 1e-5
        fd = []
        for half in (range(0, P // 2), range(P // 2, P)):
            e = torch.zeros(2 * len(half), P, dtype=torch.float64)
            for i, c in enumerate(half):
                e[2 * i, c], e[2 * i + 1, c] = h, -h
            y = keypoints_at(model, betas, rot, transl, e).reshape(len(half), 2, -1).numpy()
            fd.append(((y[:, 0] - y[:, 1]) / (2 * h)).T)
        fd = np.concatenate(fd, 1)
        for name, cols in (('rot', slice(0, 3 * n_rot)), ('betas', slice(3 * n_rot, 3 * n_rot + 10)),
                           ('transl', slice(3 * n_rot + 10, P))):
            err = np.abs(jac[:, cols] - fd[:, cols]).max()
            assert err <= 1e-6 * np.abs(fd[:, cols]).max(), (b, name, err)


def test_oracle_step_fits_rotations_with_non_increasing_loss():
    """Keypoints k = R(theta) p_k + beta_0 q_k + t for 2 rotations (chained) and a scale-like beta: zero residual at
    the generating parameters, nonlinear through the rotations."""
    rng = np.random.default_rng(3)
    K = 12
    p = rng.normal(size=(K, 3))
    q = rng.normal(size=(K, 3)) * 0.2
    R1, R2 = rodrigues(rng.normal(size=3) * 0.8).numpy(), rodrigues(rng.normal(size=3) * 0.8).numpy()
    bstar, tstar = np.array([0.7]), rng.normal(size=3)
    half = K // 2

    def evaluate(rot, beta, t):
        kp = np.zeros((K, 3))
        kp[:half] = p[:half] @ rot[0].T
        kp[half:] = p[half:] @ (rot[0] @ rot[1]).T
        kp += beta[0] * q + t
        jac = np.zeros((3 * K, 10))
        for k in range(K):
            x = kp[k] - beta[0] * q[k] - t                      # rotated point
            for a in range(3):
                w = rot[0][:, a]
                jac[3 * k:3 * k + 3, a] = np.cross(w, x)
                if k >= half:
                    w2 = (rot[0] @ rot[1])[:, a]
                    jac[3 * k:3 * k + 3, 3 + a] = np.cross(w2, x)
            jac[3 * k:3 * k + 3, 6] = q[k]
            jac[3 * k:3 * k + 3, 7:] = np.eye(3)
        return kp, jac

    target, _ = evaluate(np.stack([R1, R2]), bstar, tstar)
    w = np.ones(K)
    w[2] = 0.0                                                   # a dropped keypoint: its rows are never read
    trial = {'rot': np.stack([np.eye(3), np.eye(3)]), 'betas': np.zeros(1), 'transl': np.zeros(3)}
    state, losses = {}, []
    for it in range(31):
        kp, jac = evaluate(trial['rot'], trial['betas'], trial['transl'])
        jac[6:9] = np.nan
        state, trial, _ = kp_lm_oracle.lm_keypoints_step(state, target, w, 10.0, 3.0, it == 0, trial, kp, jac,
                                                         dtype=np.float64)
        losses.append(float(state['loss']))
    assert all(b <= a for a, b in zip(losses, losses[1:])), losses
    assert losses[-1] < 1e-12, losses
    assert np.abs(state['betas'] - bstar).max() < 1e-6 and np.abs(state['transl'] - tstar).max() < 1e-6
    for j in range(2):
        assert np.abs(state['rot'][j] @ state['rot'][j].T - np.eye(3)).max() < 1e-12


def test_unknown_method_raises():
    from shapy_b200.fit import fit_body_to_keypoints
    import pytest
    with pytest.raises(ValueError):
        fit_body_to_keypoints(None, None, method='gauss-newton')
