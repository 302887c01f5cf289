"""CPU: the float64 restatement of the stacked keypoint + measurement LM step (tests/kp_lm_oracle.py with `meas`): it
reduces to the keypoint step without measurement rows, its step solves the damped normal equations of the stacked weighted
residual, its accept / reject / lambda sequence, and it fits a small nonlinear problem with a non-increasing loss."""
import math

import numpy as np
import pytest

import kp_lm_oracle

K, NB, N_ROT = 10, 2, 2
P = 3 * N_ROT + NB + 3


def _rodrigues(aa):
    return kp_lm_oracle.exp_gram_schmidt(np.eye(3), aa)


def _problem(seed):
    """Keypoints k = R_0 p_k (first half) or R_0 R_1 p_k (second half) + q_k . beta + t, and five measurements
    m(beta) = a + C beta + 0.2 (D beta)^2, all with exact Jacobians; zero residual at the generating parameters."""
    rng = np.random.default_rng(seed)
    p = rng.normal(size=(K, 3))
    q = rng.normal(size=(K, 3, NB)) * 0.2
    a, C, D = rng.uniform(0.5, 1.5, 5), rng.normal(size=(5, NB)) * 0.3, rng.normal(size=(5, NB)) * 0.3
    half = K // 2

    def evaluate(rot, beta, t):
        beta = np.asarray(beta, np.float64)
        R01 = rot[0] @ rot[1]
        kp = np.zeros((K, 3))
        kp[:half] = p[:half] @ rot[0].T
        kp[half:] = p[half:] @ R01.T
        rotated = kp.copy()
        kp += q @ beta + t
        jac = np.zeros((3 * K, P))
        for k in range(K):
            for c in range(3):
                jac[3 * k:3 * k + 3, c] = np.cross(rot[0][:, c], rotated[k])
                if k >= half:
                    jac[3 * k:3 * k + 3, 3 + c] = np.cross(R01[:, c], rotated[k])
            jac[3 * k:3 * k + 3, 6:6 + NB] = q[k]
            jac[3 * k:3 * k + 3, 6 + NB:] = np.eye(3)
        db = D @ beta
        meas = a + C @ beta + 0.2 * db ** 2
        mjac = C + 0.4 * db[:, None] * D
        return kp, jac, meas, mjac

    truth = {'rot': np.stack([_rodrigues(rng.normal(size=3) * 0.6), _rodrigues(rng.normal(size=3) * 0.6)]),
             'betas': rng.normal(size=NB), 'transl': rng.normal(size=3)}
    return evaluate, truth, rng


def _start():
    return {'rot': np.stack([np.eye(3), np.eye(3)]), 'betas': np.zeros(NB), 'transl': np.zeros(3)}


def _f32(d):
    return {k: np.asarray(v, np.float32) for k, v in d.items()}


def test_reduces_to_keypoint_step_without_measurement_rows():
    """Every measurement weight 0 (with NaN measurements and rows, never read) and rho = 0: the same state, lambda,
    count and next trial as kp_lm_oracle.lm_keypoints_step, bit for bit, over a run of steps."""
    evaluate, truth, rng = _problem(5)
    target = evaluate(truth['rot'], truth['betas'], truth['transl'])[0] + rng.normal(size=(K, 3)) * 0.01
    w = rng.uniform(0.5, 1.5, K).astype(np.float32)
    w[3] = 0.0
    mt, mw = np.ones(5, np.float32), np.zeros(5, np.float32)
    trial_a = trial_b = _f32(_start())
    sa, sb = {}, {}
    for it in range(8):
        kp, jac, _, _ = [np.asarray(x, np.float32) for x in evaluate(trial_a['rot'], trial_a['betas'], trial_a['transl'])]
        nan5, nanj = np.full(5, np.nan, np.float32), np.full((5, NB), np.nan, np.float32)
        sa, trial_a, acc_a = kp_lm_oracle.lm_keypoints_step(sa, target, w, 10.0, 3.0, it == 0, trial_a, kp, jac)
        sb, trial_b, acc_b = kp_lm_oracle.lm_keypoints_step(sb, target, w, 10.0, 3.0, it == 0, trial_b, kp, jac,
                                                            meas=(mt, mw), trial_meas=(nan5, nanj), betas_weight=0.0)
        assert acc_a == acc_b
        for k in ('rot', 'betas', 'transl', 'keypoints', 'jac', 'lambda', 'accepted'):
            assert np.array_equal(sa[k], sb[k]), (it, k)
        assert np.array_equal(sa['loss'], sb['loss'], equal_nan=True)
        for k in ('rot', 'betas', 'transl'):
            assert np.array_equal(trial_a[k], trial_b[k]), (it, k)


@pytest.mark.parametrize('rho', [0.0, 0.05])
def test_delta_solves_stacked_normal_equations(rho):
    """The step against A and g built densely from the stacked weighted residual [sqrt(w) (kp - t); sqrt(w_m) (m - t_m);
    sqrt(rho) beta]: (A + lambda I) delta = -g, with rho I inside A through the regulariser rows."""
    evaluate, truth, rng = _problem(7)
    target = evaluate(truth['rot'], truth['betas'], truth['transl'])[0] + rng.normal(size=(K, 3)) * 0.02
    mt = evaluate(truth['rot'], truth['betas'], truth['transl'])[2] + rng.normal(size=5) * 0.01
    w = rng.uniform(0.5, 1.5, K)
    w[1] = 0.0
    mw = np.array([3.0, 0.0, 20.0, 10.0, 5.0])
    trial = {'rot': np.stack([_rodrigues(rng.normal(size=3) * 0.3) for _ in range(2)]),
             'betas': rng.normal(size=NB) * 0.5, 'transl': rng.normal(size=3) * 0.1}
    kp, jac, meas, mjac = evaluate(trial['rot'], trial['betas'], trial['transl'])
    meas[1], mjac[1] = np.nan, np.nan                            # dropped: never read
    new, _, acc, delta = kp_lm_oracle.lm_keypoints_step(
        {}, target, w, 10.0, 3.0, True, trial, kp, jac, meas=(mt, mw), trial_meas=(meas, mjac), betas_weight=rho,
        dtype=np.float64, return_delta=True)
    assert acc
    o = 3 * N_ROT
    rows, res = [], []
    for k in range(K):
        for c in range(3):
            rows.append(math.sqrt(w[k]) * jac[3 * k + c])
            res.append(math.sqrt(w[k]) * (kp[k, c] - target[k, c]))
    for k in range(5):
        if mw[k] > 0:
            row = np.zeros(P)
            row[o:o + NB] = math.sqrt(mw[k]) * mjac[k]
            rows.append(row)
            res.append(math.sqrt(mw[k]) * (meas[k] - mt[k]))
    rho32 = float(np.float32(rho))
    for i in range(NB):
        row = np.zeros(P)
        row[o + i] = math.sqrt(rho32)
        rows.append(row)
        res.append(math.sqrt(rho32) * trial['betas'][i])
    J, r = np.array(rows), np.array(res)
    A, g = J.T @ J, J.T @ r
    lam = float(new['lambda'])
    diag = np.diag(A) - rho32 * (np.arange(P) >= o) * (np.arange(P) < o + NB)   # the first lambda leaves rho out
    assert lam == pytest.approx(1e-3 * max(diag.max(), 1e-6), rel=1e-6)
    want = np.linalg.solve(A + lam * np.eye(P), -g)
    assert np.abs(delta - want).max() <= 1e-8 * np.abs(want).max(), (delta, want)
    assert new['loss'] == pytest.approx(float(r @ r), rel=1e-12)


def test_accept_reject_and_lambda_sequence():
    """A constructed series of trials: first (lambda from the diagonal), a better trial (accepted, lambda / 3), a worse
    one (rejected, lambda * 10), a weighted NaN measurement (rejected), a NaN dropped measurement with a better trial
    (accepted), and lambda clamped at 1e9; a non-finite start reports NaN and never moves."""
    evaluate, truth, rng = _problem(9)
    tgt_kp, _, tgt_m, _ = evaluate(truth['rot'], truth['betas'], truth['transl'])
    w, mw = np.ones(K, np.float32), np.array([1.0, 100.0, 2000.0, 1000.0, 1000.0], np.float32)
    rho = 0.01

    def point(scale):
        return _f32({'rot': np.stack([truth['rot'][j] @ _rodrigues(np.full(3, scale)) for j in range(2)]),
                     'betas': truth['betas'] + scale, 'transl': truth['transl'] + scale})

    def ev(x):
        return [np.asarray(v, np.float32) for v in evaluate(x['rot'].astype(np.float64), x['betas'], x['transl'])]

    def step(state, x, first, edit=None):
        kp, jac, m, mj = ev(x)
        if edit:
            edit(m, mj)
        return kp_lm_oracle.lm_keypoints_step(state, tgt_kp, w, 10.0, 3.0, first, x, kp, jac, meas=(tgt_m, mw),
                                              trial_meas=(m, mj), betas_weight=rho)

    s, _, acc = step({}, point(0.2), True)
    assert acc and s['accepted'] == 0
    lam0 = s['lambda']
    seq = [(point(0.1), None, True), (point(0.3), None, False),
           (point(0.05), lambda m, mj: m.__setitem__(2, np.nan), False),
           (point(0.05), lambda m, mj: (m.__setitem__(2, np.nan), mw.__setitem__(2, 0.0)), True)]
    lam, count = lam0, 0
    for x, edit, want in seq:
        prev = s['loss']
        s, _, acc = step(s, x, False, edit)
        assert acc == want
        lam = np.float32(lam / np.float32(3.0)) if want else np.float32(lam * np.float32(10.0))
        count += int(want)
        assert s['lambda'] == lam and s['accepted'] == count
        assert (s['loss'] < prev) if want else (s['loss'] == prev)
    mw[2] = 2000.0
    s['lambda'] = np.float32(5e8)
    s, _, acc = step(s, point(1.0), False)
    assert not acc and s['lambda'] == np.float32(1e9)
    # a non-finite start: NaN loss, the next trial is the state
    x = point(0.2)
    bad, nxt, acc = step({}, x, True, lambda m, mj: m.__setitem__(0, np.nan))
    assert acc and math.isnan(float(bad['loss']))
    for k in ('rot', 'betas', 'transl'):
        assert np.array_equal(nxt[k], x[k])


def test_fits_keypoints_and_measurements_with_non_increasing_loss():
    evaluate, truth, _ = _problem(11)
    tgt_kp, _, tgt_m, _ = evaluate(truth['rot'], truth['betas'], truth['transl'])
    w, mw = np.ones(K), np.array([1.0, 100.0, 2000.0, 1000.0, 1000.0])
    trial, state, losses = _start(), {}, []
    for it in range(40):
        kp, jac, m, mj = evaluate(trial['rot'], trial['betas'], trial['transl'])
        state, trial, _ = kp_lm_oracle.lm_keypoints_step(state, tgt_kp, w, 10.0, 3.0, it == 0, trial, kp, jac,
                                                         meas=(tgt_m, mw), trial_meas=(m, mj), dtype=np.float64)
        losses.append(float(state['loss']))
    assert all(b <= a for a, b in zip(losses, losses[1:])), losses
    assert losses[-1] < 1e-12, losses
    assert np.abs(state['betas'] - truth['betas']).max() < 1e-6
