"""CPU: the float64 restatement of the sequence 2D keypoint LM step (tests/kp2d_sequence_lm_oracle.py) pinned to
central differences of the smoothness loss, its block sweep to a dense solve of the whole normal matrix, a sequence of
one frame to the perspective oracle, zero smoothness weights to a dense grouped perspective step, and run as a plain
fp64 LM on a short synthetic sequence."""
import math

import numpy as np
import pytest

import kp2d_lm_oracle as o2
import kp2d_sequence_lm_oracle as osq
import kp2dg_lm_oracle as og
from lm_harness import expm, toy_problem

INTR = np.array([1000.0, 500.0, 480.0])


def _rots(rng, n=2, s=0.8):
    return np.stack([expm(rng.normal(size=3) * s) for _ in range(n)])


def test_smoothness_rows_vs_central_differences():
    """2 J^T W r of the pair's rows is the central-difference gradient of smooth_loss at random rotations, on all four
    blocks [delta_0 | tau_0 | delta_1 | tau_1]; J^T W J gives frame_system's diagonal blocks and coupling's C."""
    rng = np.random.default_rng(5)
    r0, r1 = _rots(rng), _rots(rng)
    t0, t1 = rng.normal(size=3), rng.normal(size=3)
    srw, stw = 3.0, 7.0
    w, r, J = osq.smooth_rows(r0, r1, t0, t1, srw, stw)
    n1 = 9

    def L(th):
        a = np.stack([r0[j] @ expm(th[3 * j:3 * j + 3]) for j in range(2)])
        b = np.stack([r1[j] @ expm(th[n1 + 3 * j:n1 + 3 * j + 3]) for j in range(2)])
        return osq.smooth_loss(a, b, t0 + th[6:9], t1 + th[n1 + 6:], srw, stw)

    h = 1e-6
    fd = np.zeros(2 * n1)
    for i in range(2 * n1):
        e = np.zeros(2 * n1)
        e[i] = h
        fd[i] = (L(e) - L(-e)) / (2 * h)
    g = J.T @ (w * r)
    assert np.abs(2 * g - fd).max() <= 1e-7 * np.abs(fd).max(), (2 * g, fd)
    assert math.isclose(osq.smooth_loss(r0, r1, t0, t1, srw, stw), float(np.sum(w * r * r)), rel_tol=1e-12)
    H = J.T @ (w[:, None] * J)
    assert np.allclose(H[n1:, :n1], osq.coupling(r0, r1, srw, stw), rtol=0, atol=1e-12)
    # the diagonal blocks and gradients of frame_system's smoothness rows: frame 0 with neighbour 1, and frame 1 with 0
    kp, jac = np.zeros((1, 3)), np.zeros((3, 10))
    for rot, tr, nb_, blk in ((r0, t0, (r1, t1), slice(0, n1)), (r1, t1, (r0, t0), slice(n1, 2 * n1))):
        A, gf = osq.frame_system(np.zeros((1, 2)), np.zeros(1), INTR, kp, jac, rot, tr, [nb_], srw=srw, stw=stw)
        assert np.allclose(A[:n1, :n1], H[blk, blk], rtol=0, atol=1e-12)
        assert np.allclose(gf[:n1], g[blk], rtol=0, atol=1e-12)


def _sequence(seed, T, sigma_noise=5.0):
    """T frames of the toy body (two chained rotations, one betas) turning and walking in front of the camera, with
    noisy targets; returns (evaluate, frames, state-like per-frame (rot, transl), beta)."""
    evaluate, rng = toy_problem(seed)
    beta = np.array([0.3])
    base = _rots(rng, s=0.5)
    frames, rots, trs = [], [], []
    for t in range(T):
        rot = np.stack([base[j] @ expm(rng.normal(size=3) * 0.1 + 0.05 * t) for j in range(2)])
        tr = np.array([0.1 * t - 0.5, -0.2, 5.0 + 0.05 * t])
        kp, _ = evaluate(rot, beta)
        tg = o2.project(kp, tr, INTR) + rng.normal(size=(12, 2)) * sigma_noise
        w = rng.uniform(0.5, 1.5, 12)
        w[3], tg[3] = 0.0, np.nan
        anchor = np.stack([r @ expm(rng.normal(size=3) * 0.2) for r in rot])
        frames.append({'targets': tg, 'weights': w, 'intr': INTR, 'anchor': anchor})
        rots.append(rot)
        trs.append(tr)
    return evaluate, frames, rots, trs, beta


def _state(evaluate, rots, trs, beta):
    kps, jacs = zip(*[evaluate(r, beta) for r in rots])
    return {'rot': list(rots), 'transl': list(trs), 'keypoints': list(kps), 'jac': list(jacs), 'betas': beta}


@pytest.mark.parametrize('T', [1, 2, 3, 17])
def test_block_sweep_equals_a_dense_solve(T):
    evaluate, frames, rots, trs, beta = _sequence(20 + T, T)
    st = _state(evaluate, rots, trs, beta)
    kw = dict(sigma=30.0, pose_w=2e3, betas_w=1e3, srw=5e3, stw=2e4)
    lam = 0.7
    M, rhs = osq.dense_system(frames, st, lam, **kw)
    want = np.linalg.solve(M, rhs)
    sys_, C = osq._blocks(frames, st, lam, kw['sigma'], kw['pose_w'], kw['srw'], kw['stw'])
    n1 = 9
    sym = lambda A: np.tril(A) + np.tril(A, -1).T  # noqa: E731
    D = [sym(A[:n1, :n1]) for A, _ in sys_]
    B = [A[n1:, :n1].T for A, _ in sys_]
    E = sum(sym(A[n1:, n1:]) for A, _ in sys_) + (kw['betas_w'] + lam) * np.eye(1)
    rb = -sum(g[n1:] for _, g in sys_) - kw['betas_w'] * beta
    x, db, ok = osq.sweep(D, C, B, E, [-g[:n1] for _, g in sys_], rb)
    assert ok
    got = np.concatenate(x + [db])
    assert np.abs(got - want).max() <= 1e-10 * max(1.0, np.abs(want).max()), np.abs(got - want).max()
    # the couplings are the dense matrix's blocks below the diagonal, and they are not symmetric
    for t in range(T - 1):
        assert np.array_equal(M[(t + 1) * n1:(t + 2) * n1, t * n1:(t + 1) * n1], C[t])
    if T > 1:
        assert np.abs(C[0] - C[0].T).max() > 1e-3


def _step_args(evaluate, frames, rots, trs, beta, rng):
    """A state at (rots, trs, beta) with its loss, and a trial nearby."""
    st = _state(evaluate, rots, trs, beta)
    trial = {'rot': [np.stack([r @ expm(rng.normal(size=3) * 0.05) for r in rot]) for rot in rots],
             'transl': [t + rng.normal(size=3) * 0.02 for t in trs], 'betas': beta + 0.05}
    for t, fr in enumerate(frames):
        fr['trial_kp'], fr['trial_jac'] = evaluate(trial['rot'][t], trial['betas'])
    return st, trial


@pytest.mark.parametrize('first', [False, True])
@pytest.mark.parametrize('terms', [(math.inf, 0.0, 0.0), (30.0, 2e3, 1e3)])
def test_one_frame_is_the_perspective_step(first, terms):
    sigma, pw, bw = terms
    evaluate, frames, rots, trs, beta = _sequence(31, 1)
    rng = np.random.default_rng(32)
    st, trial = _step_args(evaluate, frames, rots, trs, beta, rng)
    fr = frames[0]
    lcur = np.float32(o2.loss(fr['targets'], fr['weights'], st['keypoints'][0], trs[0], sigma, rots[0], fr['anchor'],
                              pw, beta, bw, intr=INTR) * (0.5 if first else 1.01))
    s1 = dict(st, loss=lcur, **{'lambda': np.float32(0.02)}, accepted=0)
    new, nxt, acc = osq.lm_sequence_step(s1, frames, 10.0, 3.0, first, trial, sigma, pw, bw, 1e4, 1e4)
    s2 = {'rot': rots[0], 'betas': beta, 'transl': trs[0], 'keypoints': st['keypoints'][0], 'jac': st['jac'][0],
          'loss': lcur, 'lambda': np.float32(0.02), 'accepted': 0}
    tr2 = {'rot': trial['rot'][0], 'betas': trial['betas'], 'transl': trial['transl'][0]}
    new2, nxt2, acc2 = o2.lm_keypoints_2d_step(s2, fr['targets'], fr['weights'], 10.0, 3.0, first, tr2, fr['trial_kp'],
                                               fr['trial_jac'], sigma, fr['anchor'], pw, bw, intr=INTR)
    assert acc == acc2 and (acc or not first)
    assert new['loss'] == new2['loss'] and new['lambda'] == new2['lambda'] and new['accepted'] == new2['accepted']
    # the step to fp32 rounding of the same fp64 values (the sweep and the full solve agree to ~1e-12)
    for a, b in ((nxt['rot'][0], nxt2['rot']), (nxt['transl'][0], nxt2['transl']), (nxt['betas'], nxt2['betas'])):
        assert np.abs(np.asarray(a, np.float64) - b).max() <= 1e-6 * max(1.0, np.abs(b).max())
    new64, nxt64, _ = osq.lm_sequence_step(s1, frames, 10.0, 3.0, first, trial, sigma, pw, bw, dtype=np.float64)
    new64b, nxt64b, _ = o2.lm_keypoints_2d_step(s2, fr['targets'], fr['weights'], 10.0, 3.0, first, tr2,
                                                fr['trial_kp'], fr['trial_jac'], sigma, fr['anchor'], pw, bw, intr=INTR,
                                                dtype=np.float64)
    for a, b in ((nxt64['rot'][0], nxt64b['rot']), (nxt64['transl'][0], nxt64b['transl']),
                 (nxt64['betas'], nxt64b['betas'])):
        assert np.abs(a - b).max() <= 1e-12 * max(1.0, np.abs(b).max())


def test_zero_smoothness_is_the_dense_grouped_perspective_step():
    """With both smoothness weights 0 the step is the grouped step's block-arrow system under the perspective rows:
    each frame's [delta | tau] block only meets beta.  Built here independently: each frame's perspective normal
    equations reordered to [delta | tau | beta], stacked into one dense matrix and solved."""
    T = 5
    evaluate, frames, rots, trs, beta = _sequence(41, T)
    rng = np.random.default_rng(42)
    st, trial = _step_args(evaluate, frames, rots, trs, beta, rng)
    sigma, pw, bw = 30.0, 2e3, 1e3
    s1 = dict(st, loss=np.float32(1e30), **{'lambda': np.float32(0.05)}, accepted=0)
    new, nxt, acc = osq.lm_sequence_step(s1, frames, 10.0, 3.0, False, trial, sigma, pw, bw, dtype=np.float64)
    assert acc
    lam = float(new['lambda'])
    n1, nb = 9, 1
    N = T * n1 + nb
    M, rhs = np.zeros((N, N)), np.zeros(N)
    for t, fr in enumerate(frames):
        A, g, _ = o2.normal_equations(fr['targets'], fr['weights'], new['keypoints'][t], new['jac'][t],
                                      new['transl'][t], sigma, new['rot'][t], fr['anchor'], pw, intr=INTR)
        perm = og.reorder(2, nb)
        A, g = A[perm][:, perm], g[perm]
        a = slice(t * n1, (t + 1) * n1)
        M[a, a] = A[:n1, :n1] + lam * np.eye(n1)
        M[a, T * n1:] = A[:n1, n1:]
        M[T * n1:, a] = A[n1:, :n1]
        M[T * n1:, T * n1:] += A[n1:, n1:]
        rhs[a], rhs[T * n1:] = -g[:n1], rhs[T * n1:] - g[n1:]
    M[T * n1:, T * n1:] += (bw + lam) * np.eye(nb)
    rhs[T * n1:] -= bw * new['betas']
    d = np.linalg.solve(M, rhs)
    for t in range(T):
        assert np.abs(nxt['transl'][t] - (new['transl'][t] + d[t * n1 + 6:t * n1 + 9])).max() <= 1e-10
    assert np.abs(nxt['betas'] - (new['betas'] + d[T * n1:])).max() <= 1e-10
    # and the loss is the sum of the frames' perspective losses + the betas prior, with no smoothness term
    L = sum(o2.loss(fr['targets'], fr['weights'], fr['trial_kp'], trial['transl'][t], sigma, trial['rot'][t],
                    fr['anchor'], pw, intr=INTR) for t, fr in enumerate(frames))
    assert math.isclose(float(new['loss']), L + bw * float(np.sum(trial['betas'] ** 2)), rel_tol=1e-12)


@pytest.mark.parametrize('smooth', [(0.0, 0.0), (1e4, 1e5)])
def test_fp64_lm_loss_never_rises_on_a_short_sequence(smooth):
    T = 6
    evaluate, frames, rots, trs, beta = _sequence(50, T, sigma_noise=0.5)
    rng = np.random.default_rng(51)
    trial = {'rot': [np.stack([r @ expm(rng.normal(size=3) * 0.15) for r in rot]) for rot in rots],
             'transl': [t + np.array([0.05, 0.05, 0.4]) * rng.normal(size=3) for t in trs], 'betas': np.zeros(1)}
    state, losses = {}, []
    for it in range(40):
        for t, fr in enumerate(frames):
            fr['trial_kp'], fr['trial_jac'] = evaluate(trial['rot'][t], trial['betas'])
        state, trial, _ = osq.lm_sequence_step(state, frames, 10.0, 3.0, it == 0, trial, 30.0, 1e2, 1e-2, *smooth,
                                               dtype=np.float64)
        losses.append(float(state['loss']))
    assert all(b <= a for a, b in zip(losses, losses[1:])), losses
    assert losses[-1] < 0.5 * losses[0], losses
    assert abs(float(state['betas'][0]) - 0.3) < 0.05
