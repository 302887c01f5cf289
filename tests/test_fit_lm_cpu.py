"""CPU: the NumPy restatement of the Levenberg-Marquardt fit (oracle/lm_oracle.py) solves a small nonlinear
least-squares problem, and its measurement Jacobian matches float64 central differences where the measurements are
smooth (mass and height)."""
import numpy as np
import pytest
import torch

from oracle import lm_oracle, measure_oracle
from shapy_b200 import synth


def test_lm_oracle_solves_linear_plus_quadratic_residuals():
    """m(beta) = t + A d + 0.3 (d . Q_k d), d = beta - beta*: zero residual at beta*, curved around it."""
    rng = np.random.default_rng(7)
    nb = 4
    A = rng.normal(size=(5, nb))
    Q = rng.normal(size=(5, nb, nb)) * 0.3
    bstar = rng.normal(size=nb)
    t = rng.normal(size=5) + 3.0
    w = np.array([1.0, 2.0, 0.5, 1.0, 3.0])

    def evaluate(beta):
        d = beta - bstar
        m = t + A @ d + np.einsum('i,kij,j->k', d, Q, d)
        J = A + np.einsum('kij,j->ki', Q + Q.transpose(0, 2, 1), d)
        return m, J

    trial = np.zeros(nb)
    state = {}
    losses = []
    for it in range(21):
        m, J = evaluate(trial)
        state, trial, _ = lm_oracle.lm_step(state, t, w, 0.0, 10.0, 3.0, it == 0, trial, m, J, dtype=np.float64)
        losses.append(float(state['loss']))
    assert all(b <= a for a, b in zip(losses, losses[1:])), losses
    assert losses[-1] < 1e-10, losses
    assert np.abs(state['betas'] - bstar).max() < 1e-5


def test_lm_oracle_step_semantics():
    """Reject keeps the state and raises lambda; a dropped term's NaN does not reach the step; a non-finite start
    reports NaN and keeps its betas."""
    rng = np.random.default_rng(3)
    nb = 3
    J = rng.normal(size=(5, nb)).astype(np.float32)
    t = np.ones(5, np.float32)
    w = np.array([1, 1, 1, 0, 1], np.float32)
    m = np.array([1.5, 0.5, 1.2, np.nan, 0.9], np.float32)
    Jn = J.copy()
    Jn[3] = np.nan
    s, trial, acc = lm_oracle.lm_step({}, t, w, 0.0, 10.0, 3.0, True, np.zeros(nb, np.float32), m, Jn)
    assert acc and np.isfinite(s['loss']) and np.isfinite(trial).all() and s['lambda'] > 0
    worse = m + np.float32(5.0)
    s2, trial2, acc2 = lm_oracle.lm_step(s, t, w, 0.0, 10.0, 3.0, False, trial, worse, Jn)
    assert not acc2 and s2['lambda'] == np.float32(s['lambda'] * np.float32(10.0)) and s2['loss'] == s['loss']
    bad = m.copy()
    bad[0] = np.nan
    s3, trial3, _ = lm_oracle.lm_step({}, t, w, 0.0, 10.0, 3.0, True, np.full(nb, 0.5, np.float32), bad, Jn)
    assert np.isnan(s3['loss']) and np.array_equal(trial3, np.full(nb, 0.5, np.float32))


def test_jacobian_betas_vs_central_differences():
    d = synth.make_smplx()
    vt = d['v_template'].double().numpy()
    S = d['shapedirs'].double().numpy()
    faces = d['faces_tensor'].numpy()
    lm = synth.load_landmarks()
    beta = (torch.randn(10, generator=torch.Generator().manual_seed(9)) * 0.5).double().numpy()
    v = (vt + S @ beta).astype(np.float32)
    J = lm_oracle.jacobian_betas(v, faces, S, lm)
    assert J.shape == (5, 10)

    def mass_height(b):
        t = (vt + S @ b)[faces]
        x, y, z = t[..., 0], t[..., 1], t[..., 2]
        vol = (-x[:, 2] * y[:, 1] * z[:, 0] + x[:, 1] * y[:, 2] * z[:, 0] + x[:, 2] * y[:, 0] * z[:, 1]
               - x[:, 0] * y[:, 2] * z[:, 1] - x[:, 1] * y[:, 0] * z[:, 2] + x[:, 0] * y[:, 1] * z[:, 2])
        hy = [(t[lm[k]['face_idx'], :, 1] * np.asarray(lm[k]['bc'])).sum() for k in ('head_top', 'left_heel')]
        return np.array([abs(vol.sum()) / 6 * measure_oracle.DENSITY, abs(hy[0] - hy[1])])

    fd = np.stack([(mass_height(beta + 1e-4 * e) - mass_height(beta - 1e-4 * e)) / 2e-4 for e in np.eye(10)], 1)
    for k in range(2):
        assert np.abs(J[k] - fd[k]).max() <= 1e-3 * np.abs(fd[k]).max(), (k, J[k], fd[k])


def test_unknown_method_raises():
    from shapy_b200.fit import fit_betas_to_measurements
    with pytest.raises(ValueError):
        fit_betas_to_measurements(None, None, {'height': 1.8}, method='lbfgs')
