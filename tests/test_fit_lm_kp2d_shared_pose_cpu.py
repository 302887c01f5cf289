"""CPU: the float64 restatement of the shared-pose 2D keypoint LM step (tests/kp2d_shared_pose_lm_oracle.py) on the toy
problem of tests/test_fit_lm_kp2d_cpu.py (two chained rotations, one betas), seen by several views that share the body
rotation R_1 and the betas and each have their own global rotation R_0 and camera: the Schur step against a dense solve
of the explicitly stacked system, its normal matrix against J^T W J of the stacked Jacobian, groups of one against the
2D oracles, n_rot = 1 against the grouped oracle, NaN handling, an fp64 LM loop; and the host start rule."""
import math

import numpy as np
import pytest
import torch

import kp2d_lm_oracle as o2
import kp2d_shared_pose_lm_oracle as osp
import kp2dg_lm_oracle as og
from oracle.lm_oracle import meas_loss
from lm_harness import expm, toy_problem

K = 12


def _views(M, seed, noise=0.05):
    """M views of one posed body of toy_problem: shared R_1* and betas*, per-view R_0 and camera; targets from them, and
    a state and a trial near them whose body rotation is one per group, as the device keeps it."""
    evaluate, rng = toy_problem(seed, K)
    bstar = np.array([0.5])
    R1 = expm(rng.normal(size=3) * 0.6)
    R1s, R1t = R1 @ expm(rng.normal(size=3) * 0.1), R1 @ expm(rng.normal(size=3) * 0.05)
    images, state, trial = [], {'rot': [], 'camera': [], 'keypoints': [], 'jac': []}, {'rot': [], 'camera': []}
    beta_s, beta_t = bstar + 0.2, bstar + 0.1
    for _ in range(M):
        R0 = expm(rng.normal(size=3) * 0.6)
        cam = np.array([0.5 + 0.2 * rng.normal(), 0.1 * rng.normal(), 0.1 * rng.normal()])
        kp, _ = evaluate(np.stack([R0, R1]), bstar)
        tg = o2.project(kp, cam) + noise * rng.normal(size=(K, 2))
        Rs = np.stack([R0 @ expm(rng.normal(size=3) * 0.1), R1s])
        Rt = np.stack([R0 @ expm(rng.normal(size=3) * 0.05), R1t])
        cs, ct = cam + 0.05 * rng.normal(size=3), cam + 0.02 * rng.normal(size=3)
        ks, js = evaluate(Rs, beta_s)
        kt, jt = evaluate(Rt, beta_t)
        images.append({'targets': tg, 'weights': rng.uniform(0.5, 1.5, K), 'trial_kp': kt, 'trial_jac': jt})
        for k, v in (('rot', Rs), ('camera', cs), ('keypoints', ks), ('jac', js)):
            state[k].append(v)
        trial['rot'].append(Rt)
        trial['camera'].append(ct)
    state['betas'] = beta_s
    trial['betas'] = beta_t
    anchor = np.stack([np.eye(3), R1 @ expm(rng.normal(size=3) * 0.05)])
    return evaluate, images, state, trial, anchor, (R1, bstar)


def _group_state(images, state, anchor, sigma, pose_w, betas_w, meas=None):
    """The state's own loss, so that a later step compares against it."""
    L = 0.0
    for i, im in enumerate(images):
        L += o2.loss(im['targets'], im['weights'], state['keypoints'][i], state['camera'][i], sigma)
    L += o2.prior_loss(state['rot'][0][1:], anchor[1:], pose_w) if pose_w > 0 else 0.0
    if meas is not None:
        L += meas_loss(meas['targets'], meas['weights'], state['meas'])
    if betas_w > 0:
        L += float(np.float32(betas_w)) * float(np.sum(np.asarray(state['betas']) ** 2))
    return np.float64(L)


def _meas(rng, state):
    meas = {'targets': rng.uniform(1, 2, 5), 'weights': np.array([1.0, 100.0, 0.0, 10.0, 10.0]),
            'trial_meas': rng.uniform(1, 2, 5), 'trial_meas_jac': rng.normal(size=(5, 1))}
    meas['trial_meas'][2], meas['trial_meas_jac'][2] = np.nan, np.nan        # dropped: never read
    state.update(meas=rng.uniform(1, 2, 5).astype(np.float32), meas_jac=rng.normal(size=(5, 1)).astype(np.float32))
    state['meas_jac'][2] = np.nan
    return meas


def _stacked(images, new, M, lam=None, sigma=math.inf):
    """The group's stacked normal equations at the state from the per-image ones, columns [each image's delta_0, c |
    delta_1, beta], keypoint rows only; with lam the image blocks are damped by it."""
    n1, ns = 6, 4
    N = M * n1 + ns
    A, g = np.zeros((N, N)), np.zeros(N)
    perm = osp.order(2, 1)
    for i, im in enumerate(images):
        Ai, gi, _ = o2.normal_equations(im['targets'], im['weights'], new['keypoints'][i], new['jac'][i],
                                        new['camera'][i], sigma)
        Ai, gi = Ai[perm][:, perm], gi[perm]
        idx = list(range(i * n1, (i + 1) * n1)) + list(range(M * n1, N))
        A[np.ix_(idx, idx)] += Ai
        g[idx] += gi
        if lam is not None:
            A[i * n1:(i + 1) * n1, i * n1:(i + 1) * n1] += lam * np.eye(n1)
    return A, g


@pytest.mark.parametrize('M', [1, 2, 3, 4, 5])
@pytest.mark.parametrize('sigma', [math.inf, 0.3])
@pytest.mark.parametrize('pose_w,betas_w', [(0.0, 0.0), (0.5, 0.2)])
@pytest.mark.parametrize('with_meas', [False, True])
def test_schur_step_equals_dense_stacked_solve(M, sigma, pose_w, betas_w, with_meas):
    _, images, state, trial, anchor, _ = _views(M, 3 + M)
    meas = _meas(np.random.default_rng(M), state) if with_meas else None
    state.update(loss=_group_state(images, state, anchor, sigma, pose_w, betas_w, meas),
                 **{'lambda': 0.05, 'accepted': 0})
    new, _, _, blocks, ds = osp.shared_pose_step(state, images, 10.0, 3.0, False, trial, anchor, sigma, pose_w,
                                                 betas_w, meas, dtype=np.float64)
    lam = float(new['lambda'])
    A, g = _stacked(images, new, M, lam, sigma)
    sh = slice(M * 6, M * 6 + 4)
    # the prior of the shared R_1 (columns 0..2 of the shared block), its measurement rows and prior on beta (column 3)
    if pose_w > 0:
        R, hw = new['rot'][0][1], 0.5 * float(np.float32(pose_w))
        D = np.stack([o2.rot_tangent(R, a) for a in range(3)], 1)
        A[M * 6:M * 6 + 3, M * 6:M * 6 + 3] += hw * D.T @ D
        g[M * 6:M * 6 + 3] += hw * D.T @ (R - anchor[1]).reshape(9)
    if with_meas:
        u = np.where(meas['weights'] > 0, meas['weights'], 0.0)
        Jm = np.where(u[:, None] > 0, np.asarray(new['meas_jac'], np.float64), 0.0)
        r = np.where(u > 0, np.asarray(new['meas'], np.float64) - meas['targets'], 0.0)
        A[M * 6 + 3, M * 6 + 3] += float(Jm[:, 0] @ (u * Jm[:, 0]))
        g[M * 6 + 3] += float(Jm[:, 0] @ (u * r))
    bw = float(np.float32(betas_w))
    g[M * 6 + 3] += bw * float(new['betas'][0])
    A[sh, sh] += lam * np.eye(4)
    A[M * 6 + 3, M * 6 + 3] += bw
    want = np.linalg.solve(A, -g)
    got = np.concatenate([-b[3] - b[2] @ ds for b in blocks] + [ds])
    assert np.abs(got - want).max() <= 1e-10 * np.abs(want).max(), (got, want)


def test_normal_matrix_equals_stacked_jtwj():
    """sigma = inf, no priors: the stacked normal matrix is J^T W J of the stacked Jacobian, each image's rows in its
    own [delta_0 | c] columns and the shared [delta_1 | beta] columns."""
    M = 3
    _, images, state, _, _, _ = _views(M, 11)
    A, g = _stacked(images, state, M)
    N = M * 6 + 4
    perm = osp.order(2, 1)
    Js, Ws, rs = [], [], []
    for i, im in enumerate(images):
        J2 = o2.jacobian_2d(state['keypoints'][i], state['jac'][i], state['camera'][i])[:, perm]
        Jrow = np.zeros((2 * K, N))
        Jrow[:, list(range(i * 6, (i + 1) * 6)) + list(range(M * 6, N))] = J2
        Js.append(Jrow)
        Ws.append(np.repeat(im['weights'], 2))
        rs.append((o2.project(state['keypoints'][i], state['camera'][i]) - im['targets']).reshape(-1))
    J, W, r = np.concatenate(Js), np.concatenate(Ws), np.concatenate(rs)
    assert np.allclose(A, J.T @ (W[:, None] * J), rtol=1e-12, atol=1e-12)
    assert np.allclose(g, J.T @ (W * r), rtol=1e-12, atol=1e-12)
    # the shared rotation's columns of each image are its own R_1 columns of the 2D Jacobian
    J2 = o2.jacobian_2d(state['keypoints'][0], state['jac'][0], state['camera'][0])
    assert np.array_equal(J[:2 * K, M * 6:M * 6 + 3], J2[:, 3:6])


@pytest.mark.parametrize('first', [True, False])
@pytest.mark.parametrize('with_meas', [False, True])
@pytest.mark.parametrize('sigma,pose_w,betas_w', [(math.inf, 0.0, 0.0), (0.3, 0.5, 0.2)])
def test_groups_of_one_equal_the_2d_oracles(first, with_meas, sigma, pose_w, betas_w):
    _, images, state, trial, anchor, _ = _views(1, 21)
    meas = _meas(np.random.default_rng(5), state) if with_meas else None
    if not first:
        state.update(loss=np.float32(_group_state(images, state, anchor, sigma, pose_w, betas_w, meas)),
                     **{'lambda': np.float32(0.05), 'accepted': 0})
    im = images[0]
    s = {k: state[k][0] for k in ('rot', 'camera', 'keypoints', 'jac')}
    for k in ('betas', 'loss', 'lambda', 'accepted', 'meas', 'meas_jac'):
        if k in state:
            s[k] = state[k]
    t = {'rot': trial['rot'][0], 'camera': trial['camera'][0], 'betas': trial['betas']}

    def two_d(dtype):
        mkw = {} if meas is None else dict(meas=(meas['targets'], meas['weights']),
                                           trial_meas=(meas['trial_meas'], meas['trial_meas_jac']))
        return o2.lm_keypoints_2d_step(s, im['targets'], im['weights'], 10.0, 3.0, first, t, im['trial_kp'],
                                       im['trial_jac'], sigma, anchor, pose_w, betas_w, dtype=dtype, **mkw)
    new, nxt, acc, _, _ = osp.shared_pose_step(state, images, 10.0, 3.0, first, trial, anchor, sigma, pose_w, betas_w,
                                               meas)
    want, wnxt, wacc = two_d(np.float32)
    assert acc == wacc
    for k in ('loss', 'lambda', 'accepted'):
        assert np.array_equal(new[k], want[k], equal_nan=True), (k, new[k], want[k])
    for k in ('rot', 'camera'):
        assert np.abs(np.asarray(nxt[k][0], np.float64) - wnxt[k]).max() <= 1e-6 * max(1.0, np.abs(wnxt[k]).max())
    assert np.abs(nxt['betas'] - wnxt['betas']).max() <= 1e-6 * max(1.0, np.abs(wnxt['betas']).max())
    # in float64 the two eliminations agree to rounding
    _, nxt64, _, _, _ = osp.shared_pose_step(state, images, 10.0, 3.0, first, trial, anchor, sigma, pose_w, betas_w,
                                             meas, dtype=np.float64)
    _, w64, _ = two_d(np.float64)
    for k in ('rot', 'camera'):
        assert np.abs(nxt64[k][0] - w64[k]).max() <= 1e-10 * max(1.0, np.abs(w64[k]).max()), k
    assert np.abs(nxt64['betas'] - w64['betas']).max() <= 1e-10 * max(1.0, np.abs(w64['betas']).max())


def _one_rotation(seed):
    """A toy problem with one rotation: kp = R p + beta q + t, (3K, 7) Jacobian with the transl columns last."""
    rng = np.random.default_rng(seed)
    p, q, t = rng.normal(size=(K, 3)), rng.normal(size=(K, 3)) * 0.2, rng.normal(size=3) * 0.1

    def evaluate(rot, beta):
        kp = p @ rot[0].T + beta[0] * q + t
        jac = np.zeros((3 * K, 7))
        for k in range(K):
            for a in range(3):
                jac[3 * k:3 * k + 3, a] = np.cross(rot[0][:, a], kp[k] - beta[0] * q[k] - t)
            jac[3 * k:3 * k + 3, 3] = q[k]
            jac[3 * k:3 * k + 3, 4:] = np.eye(3)
        return kp, jac
    return evaluate, rng


@pytest.mark.parametrize('first', [True, False])
@pytest.mark.parametrize('with_meas', [False, True])
def test_one_rotation_equals_the_grouped_oracle(first, with_meas):
    """n_rot = 1: nothing is shared but beta, and every output is the grouped step's, bit for bit."""
    evaluate, rng = _one_rotation(9)
    M = 3
    images, state, trial = [], {'rot': [], 'camera': [], 'keypoints': [], 'jac': []}, {'rot': [], 'camera': []}
    for _ in range(M):
        R = expm(rng.normal(size=3) * 0.6)[None]
        cam = np.array([0.5, 0.0, 0.0]) + 0.1 * rng.normal(size=3)
        kp, _ = evaluate(R, np.array([0.5]))
        Rs, Rt = R @ expm(rng.normal(size=3) * 0.1), R @ expm(rng.normal(size=3) * 0.05)
        ks, js = evaluate(Rs, np.array([0.7]))
        kt, jt = evaluate(Rt, np.array([0.6]))
        images.append({'targets': o2.project(kp, cam) + 0.02 * rng.normal(size=(K, 2)),
                       'weights': rng.uniform(0.5, 1.5, K), 'trial_kp': kt, 'trial_jac': jt, 'anchor': R})
        for k, v in (('rot', Rs), ('camera', cam + 0.05), ('keypoints', ks), ('jac', js)):
            state[k].append(v)
        trial['rot'].append(Rt)
        trial['camera'].append(cam + 0.02)
    state['betas'], trial['betas'] = np.array([0.7]), np.array([0.6])
    meas = _meas(rng, state) if with_meas else None
    if not first:
        state.update(loss=np.float32(1e3), **{'lambda': np.float32(0.05), 'accepted': 2})
    a = osp.shared_pose_step(state, images, 10.0, 3.0, first, trial, np.eye(3)[None], 0.3, 0.5, 0.2, meas)
    b = og.lm_groups_step(state, images, 10.0, 3.0, first, trial, 0.3, 0.5, 0.2, meas)
    for k in ('loss', 'lambda', 'accepted', 'betas'):
        assert np.array_equal(a[0][k], b[0][k]), k
    assert a[2] == b[2]
    for k in ('rot', 'camera'):
        assert all(np.array_equal(x, y) for x, y in zip(a[1][k], b[1][k])), k
    assert np.array_equal(a[1]['betas'], b[1]['betas'])


def test_dropped_nan_changes_nothing_and_a_weighted_nan_rejects_the_group():
    _, images, state, trial, anchor, _ = _views(3, 31)
    args = (math.inf, 0.5, 0.1)
    state.update(loss=np.float32(_group_state(images, state, anchor, *args) * 1.5),
                 **{'lambda': np.float32(0.05), 'accepted': 0})
    ref = osp.shared_pose_step(state, images, 10.0, 3.0, False, trial, anchor, *args)
    assert ref[2]                                          # the trial is better than the inflated state loss
    imgs = [dict(im) for im in images]
    st = {k: (list(v) if isinstance(v, list) else v) for k, v in state.items()}
    for i, im in enumerate(imgs):                          # a dropped keypoint, NaN everywhere it could be read
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
    a = osp.shared_pose_step(state, clean, 10.0, 3.0, False, trial, anchor, *args)
    b = osp.shared_pose_step(st, imgs, 10.0, 3.0, False, trial, anchor, *args)
    for k in ('loss', 'lambda', 'accepted'):
        assert np.array_equal(a[0][k], b[0][k]), k
    for k in ('rot', 'camera'):
        assert all(np.array_equal(x, y) for x, y in zip(a[1][k], b[1][k])), k
    assert np.array_equal(a[1]['betas'], b[1]['betas'])
    # the anchor's joint 0 is never read
    anc = anchor.copy()
    anc[0] = np.nan
    c = osp.shared_pose_step(state, images, 10.0, 3.0, False, trial, anc, *args)
    assert np.array_equal(c[0]['loss'], ref[0]['loss']) and np.array_equal(c[1]['betas'], ref[1]['betas'])
    # a weighted NaN in one image's trial keypoints: the group's trial loss is NaN, the whole group is rejected
    bad = [dict(im) for im in images]
    bad[1] = dict(bad[1], trial_kp=bad[1]['trial_kp'].copy())
    bad[1]['trial_kp'][2] = np.nan
    new, nxt, acc, _, _ = osp.shared_pose_step(state, bad, 10.0, 3.0, False, trial, anchor, *args)
    assert not acc and new['loss'] == state['loss'] and new['lambda'] == np.float32(0.5)
    for i in range(3):
        assert np.array_equal(new['rot'][i], state['rot'][i]) and np.array_equal(new['camera'][i], state['camera'][i])
    assert np.array_equal(new['betas'], state['betas'])


@pytest.mark.parametrize('sigma', [math.inf, 0.5])
def test_fp64_lm_keeps_the_group_loss_non_increasing_and_recovers_the_shared_pose(sigma):
    M = 4
    evaluate, images, state, _, anchor, (R1, bstar) = _views(M, 41, noise=0.0)
    trial = {'rot': [r.copy() for r in state['rot']], 'camera': [c.copy() for c in state['camera']],
             'betas': np.zeros(1)}
    st, losses = {}, []
    for it in range(60):
        for i, im in enumerate(images):
            im['trial_kp'], im['trial_jac'] = evaluate(trial['rot'][i], trial['betas'])
        st, trial, _, _, _ = osp.shared_pose_step(st, images, 10.0, 3.0, it == 0, trial, anchor, sigma,
                                                  dtype=np.float64)
        losses.append(float(st['loss']))
        assert all(np.array_equal(r[1], trial['rot'][0][1]) for r in trial['rot'])       # one body rotation
    assert all(b <= a for a, b in zip(losses, losses[1:])), losses
    assert losses[-1] < 1e-16, losses
    assert abs(float(st['betas'][0]) - float(bstar[0])) < 1e-7
    assert np.abs(st['rot'][0][1] - R1).max() < 1e-7


# ------------------------------------------------------------------------------------------------ host logic
def test_shared_start_is_the_chordal_mean_made_a_rotation_by_gram_schmidt():
    """_shared_body_raw: the image-order mean of each group's body rotations, as the 6D decoder's input (its first two
    columns); decoded, the Gram-Schmidt of that mean.  Identical rotations give themselves back."""
    from shapy_b200.fit import _group_sum, _shared_body_raw, group_plan
    rng = np.random.default_rng(3)
    base = np.stack([expm(rng.normal(size=3)) for _ in range(21)])
    views = [np.stack([r @ expm(rng.normal(size=3) * 0.2) for r in base]) for _ in range(3)]
    rot = torch.tensor(np.stack([np.concatenate([expm(rng.normal(size=3))[None], v]) for v in views] +
                                [np.concatenate([np.eye(3)[None], base])]), dtype=torch.float32)  # (4, 22, 3, 3)
    order, off = group_plan(torch.tensor([0, 0, 0, 1]), 4)
    cnt = (off[1:] - off[:-1]).float()
    raw = _shared_body_raw(rot[order], off, cnt)
    assert raw.shape == (2, 126)
    mean = _group_sum(rot[order][:, 1:], off) / cnt[:, None, None, None]
    assert torch.equal(raw, mean[..., :2].reshape(2, 126))
    want = (views[0].astype(np.float32) + views[1].astype(np.float32)) + views[2].astype(np.float32)
    assert np.allclose(raw[0].view(21, 3, 2).numpy(), (want / np.float32(3))[..., :2], rtol=0, atol=1e-6)
    R = np.stack([osp.gram_schmidt(m) for m in raw[0].view(21, 3, 2).double().numpy()])
    assert np.allclose(np.einsum('jab,jac->jbc', R, R), np.eye(3), atol=1e-12)
    want_R = np.stack([osp.gram_schmidt(m) for m in np.mean(np.stack(views), 0)])     # the chordal mean's projection
    assert np.abs(R - want_R).max() < 1e-5
    assert np.allclose(raw[1].view(21, 3, 2).numpy(), base.astype(np.float32)[..., :2])


def test_share_pose_needs_groups():
    from shapy_b200.fit import fit_body_to_keypoints_2d
    with pytest.raises(ValueError, match='share_pose needs groups'):
        fit_body_to_keypoints_2d(None, torch.zeros(2, 3, 2), share_pose=True)
