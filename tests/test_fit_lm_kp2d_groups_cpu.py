"""CPU: the float64 restatement of the grouped 2D keypoint LM step (tests/kp2dg_lm_oracle.py) on the toy problem of
tests/test_fit_lm_kp2d_cpu.py with one betas shared by several views: the Schur step against a dense solve of the
explicitly stacked block-arrow system, its normal matrix against J^T W J of the stacked Jacobian, groups of one against
the 2D oracles, NaN handling, an fp64 LM loop; and the host logic of fit_body_to_keypoints_2d(groups=)."""
import math

import numpy as np
import pytest
import torch

import kp2d_lm_oracle as o2
import kp2dg_lm_oracle as og
from oracle.lm_oracle import meas_loss
from lm_harness import expm, toy_problem

K = 12


def _views(M, seed, sigma=math.inf, pose_w=0.0, noise=0.05):
    """M views of one body of toy_problem (shared betas bstar, per-view rotations and camera), targets from bstar, a
    state and a trial near them."""
    evaluate, rng = toy_problem(seed, K)
    bstar = np.array([0.5])
    images, state, trial = [], {'rot': [], 'camera': [], 'keypoints': [], 'jac': []}, {'rot': [], 'camera': []}
    beta_s, beta_t = bstar + 0.2, bstar + 0.1
    for _ in range(M):
        R = np.stack([expm(rng.normal(size=3) * 0.6) for _ in range(2)])
        cam = np.array([0.5 + 0.2 * rng.normal(), 0.1 * rng.normal(), 0.1 * rng.normal()])
        kp, _ = evaluate(R, bstar)
        tg = o2.project(kp, cam) + noise * rng.normal(size=(K, 2))
        Rs = np.stack([r @ expm(rng.normal(size=3) * 0.1) for r in R])
        Rt = np.stack([r @ expm(rng.normal(size=3) * 0.05) for r in R])
        cs, ct = cam + 0.05 * rng.normal(size=3), cam + 0.02 * rng.normal(size=3)
        ks, js = evaluate(Rs, beta_s)
        kt, jt = evaluate(Rt, beta_t)
        images.append({'targets': tg, 'weights': rng.uniform(0.5, 1.5, K), 'anchor': R, 'trial_kp': kt,
                       'trial_jac': jt})
        for k, v in (('rot', Rs), ('camera', cs), ('keypoints', ks), ('jac', js)):
            state[k].append(v)
        trial['rot'].append(Rt)
        trial['camera'].append(ct)
    state['betas'] = beta_s
    trial['betas'] = beta_t
    return evaluate, images, state, trial, bstar


def _group_state(images, state, sigma, pose_w, betas_w, meas=None):
    """The state's own loss, so that a later step compares against it."""
    L = 0.0
    for i, im in enumerate(images):
        L += o2.loss(im['targets'], im['weights'], state['keypoints'][i], state['camera'][i], sigma, state['rot'][i],
                     im['anchor'], pose_w)
    if meas is not None:
        L += meas_loss(meas['targets'], meas['weights'], state['meas'])
    if betas_w > 0:
        L += float(np.float32(betas_w)) * float(np.sum(np.asarray(state['betas']) ** 2))
    return np.float64(L)


@pytest.mark.parametrize('M', [1, 2, 5])
@pytest.mark.parametrize('sigma,pose_w,betas_w', [(math.inf, 0.0, 0.0), (0.3, 0.5, 0.2)])
def test_schur_step_equals_dense_block_arrow_solve(M, sigma, pose_w, betas_w):
    _, images, state, trial, _ = _views(M, 3 + M)
    state.update(loss=_group_state(images, state, sigma, pose_w, betas_w), **{'lambda': 0.05, 'accepted': 0})
    new, _, _, blocks, db = og.lm_groups_step(state, images, 10.0, 3.0, False, trial, sigma, pose_w, betas_w,
                                              dtype=np.float64)
    lam = float(new['lambda'])
    n1, nb = 9, 1
    N = M * n1 + nb
    Afull, gfull = np.zeros((N, N)), np.zeros(N)
    perm = og.reorder(2, nb)
    for i, im in enumerate(images):
        A, g, _ = o2.normal_equations(im['targets'], im['weights'], new['keypoints'][i], new['jac'][i],
                                      new['camera'][i], sigma, new['rot'][i], im['anchor'], pose_w)
        A, g = A[perm][:, perm], g[perm]
        r = slice(i * n1, (i + 1) * n1)
        Afull[r, r] = A[:n1, :n1] + lam * np.eye(n1)
        Afull[r, M * n1:] = A[:n1, n1:]
        Afull[M * n1:, r] = A[n1:, :n1]
        Afull[M * n1:, M * n1:] += A[n1:, n1:]
        gfull[r] = g[:n1]
        gfull[M * n1:] += g[n1:]
    gfull[M * n1:] += float(np.float32(betas_w)) * np.asarray(new['betas'])
    Afull[M * n1:, M * n1:] += (float(np.float32(betas_w)) + lam) * np.eye(nb)
    want = np.linalg.solve(Afull, -gfull)
    got = np.concatenate([-b[3] - b[2] @ db for b in blocks] + [db])
    assert np.abs(got - want).max() <= 1e-10 * np.abs(want).max(), (got, want)


def test_normal_matrix_equals_stacked_jtwj():
    """sigma = inf, no priors: the block-arrow matrix of the per-image normal equations is J^T W J of the stacked
    Jacobian, each image's rows in its own [delta | c] columns and the shared betas column."""
    M = 3
    _, images, state, _, _ = _views(M, 11)
    n1, nb = 9, 1
    N = M * n1 + nb
    perm = og.reorder(2, nb)
    Ablk, gblk = np.zeros((N, N)), np.zeros(N)
    Js, Ws, rs = [], [], []
    for i, im in enumerate(images):
        A, g, _ = o2.normal_equations(im['targets'], im['weights'], state['keypoints'][i], state['jac'][i],
                                      state['camera'][i])
        A, g = A[perm][:, perm], g[perm]
        idx = list(range(i * n1, (i + 1) * n1)) + list(range(M * n1, N))
        Ablk[np.ix_(idx, idx)] += A
        gblk[idx] += g
        J2 = o2.jacobian_2d(state['keypoints'][i], state['jac'][i], state['camera'][i])[:, perm]
        Jrow = np.zeros((2 * K, N))
        Jrow[:, idx] = J2
        Js.append(Jrow)
        Ws.append(np.repeat(im['weights'], 2))
        rs.append((o2.project(state['keypoints'][i], state['camera'][i]) - im['targets']).reshape(-1))
    J, W, r = np.concatenate(Js), np.concatenate(Ws), np.concatenate(rs)
    assert np.allclose(Ablk, J.T @ (W[:, None] * J), rtol=1e-12, atol=1e-12)
    assert np.allclose(gblk, J.T @ (W * r), rtol=1e-12, atol=1e-12)


def _single(images, state, trial, i=0):
    s = {k: state[k][i] for k in ('rot', 'camera', 'keypoints', 'jac')}
    s['betas'] = state['betas']
    t = {'rot': trial['rot'][i], 'camera': trial['camera'][i], 'betas': trial['betas']}
    return s, t


@pytest.mark.parametrize('first', [True, False])
@pytest.mark.parametrize('with_meas', [False, True])
@pytest.mark.parametrize('sigma,pose_w,betas_w', [(math.inf, 0.0, 0.0), (0.3, 0.5, 0.2)])
def test_groups_of_one_equal_the_2d_oracles(first, with_meas, sigma, pose_w, betas_w):
    _, images, state, trial, _ = _views(1, 21)
    rng = np.random.default_rng(5)
    meas = None
    if with_meas:
        meas = {'targets': rng.uniform(1, 2, 5), 'weights': np.array([1.0, 100.0, 0.0, 10.0, 10.0]),
                'trial_meas': rng.uniform(1, 2, 5), 'trial_meas_jac': rng.normal(size=(5, 1))}
        meas['trial_meas'][2], meas['trial_meas_jac'][2] = np.nan, np.nan        # dropped: never read
        state.update(meas=rng.uniform(1, 2, 5).astype(np.float32), meas_jac=rng.normal(size=(5, 1)).astype(np.float32))
    if not first:
        state.update(loss=np.float32(_group_state(images, state, sigma, pose_w, betas_w, meas)),
                     **{'lambda': np.float32(0.05), 'accepted': 0})
    new, nxt, acc, _, _ = og.lm_groups_step(state, images, 10.0, 3.0, first, trial, sigma, pose_w, betas_w, meas)
    s, t = _single(images, state, trial)
    for k in ('loss', 'lambda', 'accepted', 'meas', 'meas_jac'):
        if k in state:
            s[k] = state[k]
    im = images[0]
    mkw = {} if meas is None else dict(meas=(meas['targets'], meas['weights']),
                                       trial_meas=(meas['trial_meas'], meas['trial_meas_jac']))
    want, wnxt, wacc = o2.lm_keypoints_2d_step(s, im['targets'], im['weights'], 10.0, 3.0, first, t, im['trial_kp'],
                                               im['trial_jac'], sigma, im['anchor'], pose_w, betas_w, **mkw)
    assert acc == wacc
    for k in ('loss', 'lambda', 'accepted'):
        assert np.array_equal(new[k], want[k], equal_nan=True), (k, new[k], want[k])
    for k in ('rot', 'camera'):
        assert np.abs(np.asarray(nxt[k][0], np.float64) - wnxt[k]).max() <= 1e-6 * max(1.0, np.abs(wnxt[k]).max())
    assert np.abs(nxt['betas'] - wnxt['betas']).max() <= 1e-6 * max(1.0, np.abs(wnxt['betas']).max())
    # in float64 the two eliminations agree to rounding
    new64, nxt64, _, _, _ = og.lm_groups_step(state, images, 10.0, 3.0, first, trial, sigma, pose_w, betas_w, meas,
                                              dtype=np.float64)
    _, w64, _ = o2.lm_keypoints_2d_step(s, im['targets'], im['weights'], 10.0, 3.0, first, t, im['trial_kp'],
                                        im['trial_jac'], sigma, im['anchor'], pose_w, betas_w, dtype=np.float64, **mkw)
    for k in ('rot', 'camera'):
        assert np.abs(nxt64[k][0] - w64[k]).max() <= 1e-10 * max(1.0, np.abs(w64[k]).max()), k
    assert np.abs(nxt64['betas'] - w64['betas']).max() <= 1e-10 * max(1.0, np.abs(w64['betas']).max())


def test_dropped_nan_changes_nothing_and_a_weighted_nan_rejects_the_group():
    _, images, state, trial, _ = _views(3, 31)
    state.update(loss=np.float32(_group_state(images, state, math.inf, 0.0, 0.0) * 1.5),
                 **{'lambda': np.float32(0.05), 'accepted': 0})
    ref = og.lm_groups_step(state, images, 10.0, 3.0, False, trial)
    assert ref[2]                                          # the trial is better than the inflated state loss
    # a dropped keypoint with NaN target, keypoints and rows in state and trial
    imgs = [dict(im) for im in images]
    st = {k: (list(v) if isinstance(v, list) else v) for k, v in state.items()}
    for i, im in enumerate(imgs):
        im['weights'] = im['weights'].copy()
        im['targets'], im['trial_kp'], im['trial_jac'] = im['targets'].copy(), im['trial_kp'].copy(), \
            im['trial_jac'].copy()
        im['weights'][4] = 0.0
        im['targets'][4] = im['trial_kp'][4] = np.nan
        im['trial_jac'][12:15] = np.nan
        st['keypoints'][i], st['jac'][i] = st['keypoints'][i].copy(), st['jac'][i].copy()
        st['keypoints'][i][4], st['jac'][i][12:15] = np.nan, np.nan
    clean = [dict(im, weights=im['weights'].copy()) for im in images]
    for im in clean:
        im['weights'][4] = 0.0
    a = og.lm_groups_step(state, clean, 10.0, 3.0, False, trial)
    b = og.lm_groups_step(st, imgs, 10.0, 3.0, False, trial)
    for k in ('loss', 'lambda', 'accepted'):
        assert np.array_equal(a[0][k], b[0][k]), k
    for k in ('rot', 'camera'):
        assert all(np.array_equal(x, y) for x, y in zip(a[1][k], b[1][k])), k
    assert np.array_equal(a[1]['betas'], b[1]['betas'])
    # a weighted NaN in one image's trial keypoints: the group's trial loss is NaN, the whole group is rejected
    bad = [dict(im) for im in images]
    bad[1] = dict(bad[1], trial_kp=bad[1]['trial_kp'].copy())
    bad[1]['trial_kp'][2] = np.nan
    new, nxt, acc, _, _ = og.lm_groups_step(state, bad, 10.0, 3.0, False, trial)
    assert not acc and new['loss'] == state['loss'] and new['lambda'] == np.float32(0.5)
    for i in range(3):
        assert np.array_equal(new['rot'][i], state['rot'][i]) and np.array_equal(new['camera'][i], state['camera'][i])
    assert np.array_equal(new['betas'], state['betas'])


@pytest.mark.parametrize('sigma', [math.inf, 0.5])
def test_fp64_lm_keeps_the_group_loss_non_increasing_and_recovers_the_shared_betas(sigma):
    M = 4
    evaluate, images, state, trial, bstar = _views(M, 41, noise=0.0)
    trial = {'rot': [r.copy() for r in state['rot']], 'camera': [c.copy() for c in state['camera']],
             'betas': np.zeros(1)}
    st, losses = {}, []
    for it in range(60):
        for i, im in enumerate(images):
            im['trial_kp'], im['trial_jac'] = evaluate(trial['rot'][i], trial['betas'])
        st, trial, _, _, _ = og.lm_groups_step(st, images, 10.0, 3.0, it == 0, trial, sigma, dtype=np.float64)
        losses.append(float(st['loss']))
    assert all(b <= a for a, b in zip(losses, losses[1:])), losses
    assert losses[-1] < 1e-16, losses
    assert abs(float(st['betas'][0]) - float(bstar[0])) < 1e-7


# ------------------------------------------------------------------------------------------------ host logic
def test_group_plan_sorts_stably_and_builds_offsets():
    from shapy_b200.fit import group_plan
    order, off = group_plan(torch.tensor([2, 0, 1, 0, 2, 2]), 6)
    assert order.tolist() == [1, 3, 2, 0, 4, 5] and off.tolist() == [0, 2, 3, 6] and off.dtype == torch.int32
    order, off = group_plan(np.arange(5)[::-1].copy(), 5)
    assert order.tolist() == [4, 3, 2, 1, 0] and off.tolist() == [0, 1, 2, 3, 4, 5]
    order, off = group_plan(torch.zeros(0, dtype=torch.int64), 0)
    assert order.numel() == 0 and off.tolist() == [0]


@pytest.mark.parametrize('bad', [[0, 2, 2], [1, 1, 1], [0, -1, 1], [0.0, 1.0, 1.0], [0, 1], [[0, 1, 1]],
                                 [True, False, True]])
def test_group_plan_rejects_bad_labels(bad):
    from shapy_b200.fit import group_plan
    with pytest.raises(ValueError):
        group_plan(torch.tensor(bad), 3)


def test_group_sum_is_in_image_order_and_the_permutation_round_trips():
    from shapy_b200.fit import _group_sum, group_plan
    labels = torch.tensor([1, 0, 1, 2, 1, 0])
    x = torch.tensor([1e8, 1.0, -1e8, 3.0, 1.0, 2.0], dtype=torch.float32)
    order, off = group_plan(labels, 6)
    xs = x[order]
    got = _group_sum(xs[:, None], off)[:, 0]
    want = []
    for g in range(3):
        acc = None
        for v in x[labels == g]:                   # the caller's order within the group, left to right in fp32
            acc = v.clone() if acc is None else acc + v
        want.append(acc)
    assert torch.equal(got, torch.stack(want))
    assert float(got[1]) == 1.0                    # (1e8 - 1e8) + 1, not 1e8 + (-1e8 + 1)
    inv = torch.argsort(order)
    assert torch.equal(xs[inv], x)
