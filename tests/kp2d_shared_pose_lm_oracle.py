"""NumPy float64 restatement of the shared-pose 2D keypoint Levenberg-Marquardt step (test infrastructure), on top of
tests/kp2dg_lm_oracle.py: the images of one group are views of one posed body, so they share the betas and the body
rotations of joints 1 .. n_rot - 1; each keeps its global rotation and camera.  The step is the Schur complement of the
group's normal matrix with the image blocks [delta_0 | c] eliminated and the shared block [delta_1 .. | beta] solved.

  order               the column order [delta_0 | c | delta_1 .. | beta], as indices into [delta | beta | c]
  image_scratch       launch 1 for one image: the bracket of its trial keypoint term (no prior) and, on the first step,
                      the max of its keypoint-row diagonal over [delta_0 | c] and its shared-column entries
  decide              the group's decision: kp2dg_lm_oracle.decide with the group's pose prior added once, after the
                      keypoint brackets, from the group's trial rotations and its anchor
  image_block         launch 2 for one image: its keypoint rows in that order, the leading 6 x 6 block damped by lambda
                      and factored alone; (S_i, s_i, X_i, x_i, ok_i)
  shared_pose_step    shapy_fit_lm_keypoints_2d_shared_pose_step (and _measurements_step, with `meas`) for one group:
                      the same fp64 operations in the same order; as in kp2d_lm_oracle, softplus' exp / log1p may
                      differ from the device's in the last bit
  gram_schmidt        the 6D decoder's Gram-Schmidt of a 3 x 3 matrix's first two columns
"""
import math

import numpy as np

import kp2d_lm_oracle as o2
import kp2dg_lm_oracle as og
from oracle.lm_oracle import cholesky_solve, exp_gram_schmidt, lm_add_next, lm_diag_max, meas_rows

N1 = 6                                                  # the image block [delta_0 | c]


def order(n_rot, nb):
    o = 3 * n_rot
    return np.array([0, 1, 2, o + nb, o + nb + 1, o + nb + 2] + list(range(3, o)) + list(range(o, o + nb)))


def image_scratch(targets, weights, trial_kp, trial_jac, trial, first, sigma=math.inf, dtype=np.float32):
    """(bracket, dmax over the [delta_0 | c] diagonal from DIAG_FLOOR, the shared-column diagonal) of one image."""
    lt = o2.loss(targets, weights, trial_kp, trial['camera'], sigma)
    if not first:
        return lt, None, None
    f = dtype
    _, _, dg = o2.normal_equations(targets, weights, np.asarray(trial_kp, f), np.asarray(trial_jac, f),
                                   np.asarray(trial['camera'], f), sigma)
    dg = dg[order(np.asarray(trial['rot']).shape[0], len(trial['betas']))]
    return lt, lm_diag_max(dg[:N1]), dg[N1:].copy()


def decide(scratch, first, lcur, lam, lambda_up, lambda_down, trial_rot, anchor, pose_w, trial_betas, betas_w=0.0,
           meas_terms=None, dtype=np.float32):
    """kp2dg_lm_oracle.decide with the prior of the group's trial rotations trial_rot (n_rot, 3, 3) added once."""
    sc = [list(s) for s in scratch]
    if pose_w > 0.0:    # the device adds the brackets left to right, then the prior; og.decide adds only the brackets,
        L = sc[0][0]    # so their sum with the prior goes first and exact zeros follow (x + 0.0 is x)
        for s in sc[1:]:
            L += s[0]
        sc = [[L + o2.prior_loss(np.asarray(trial_rot, np.float64)[1:], np.asarray(anchor, np.float64)[1:], pose_w),
               *sc[0][1:]]] + [[0.0, *s[1:]] for s in sc[1:]]
    return og.decide(sc, first, lcur, lam, lambda_up, lambda_down, trial_betas, betas_w, meas_terms, dtype)


def image_block(targets, weights, kp, jac, camera, n_rot, lam, sigma=math.inf, nb=None):
    """Launch 2 for one image at its state: (S_i (ns, ns) lower, s_i, X_i (6, ns), x_i, ok_i)."""
    A, g, _ = o2.normal_equations(targets, weights, kp, jac, camera, sigma)
    perm = order(n_rot, nb)
    A, g = A[perm][:, perm].copy(), g[perm].copy()
    for j in range(N1):
        A[j, j] += float(lam)
    y, ok = cholesky_solve(A, g, N1)
    W = A[N1:, :N1].copy()                       # the rows of L21, then X^T
    with np.errstate(invalid='ignore', divide='ignore'):
        for j in range(N1 - 1, -1, -1):
            W[:, j] /= A[j, j]
            W[:, :j] -= np.outer(W[:, j], A[j, :j])
    return np.tril(A[N1:, N1:]), -y[N1:], W.T.copy(), -y[:N1], ok


def shared_pose_step(state, images, lambda_up, lambda_down, first, trial, anchor, sigma=math.inf, pose_w=0.0,
                     betas_w=0.0, meas=None, dtype=np.float32):
    """One step for one group.  state: {'rot', 'camera', 'keypoints', 'jac': lists over the images (every image's
    rotation rows 1 .. the group's), 'betas' (nb,), 'loss', 'lambda', 'accepted'} (+ 'meas', 'meas_jac' with meas);
    images: a list of {'targets', 'weights', 'trial_kp', 'trial_jac'}; trial: {'rot', 'camera': lists, 'betas'};
    anchor: the group's (n_rot, 3, 3), joint 0 unread; meas as kp2dg_lm_oracle.lm_groups_step's.  Returns (new state,
    next trial, accepted flag, the images' (S_i, s_i, X_i, x_i, ok_i), the shared delta)."""
    f = dtype
    nb = len(trial['betas'])
    n_rot = np.asarray(trial['rot'][0]).shape[0]
    ob, ns = 3 * (n_rot - 1), 3 * (n_rot - 1) + nb
    scratch = [image_scratch(im['targets'], im['weights'], im['trial_kp'], im['trial_jac'],
                             {'rot': trial['rot'][i], 'camera': trial['camera'][i], 'betas': trial['betas']}, first,
                             sigma, dtype) for i, im in enumerate(images)]
    mt = None if meas is None else (meas['targets'], meas['weights'], meas['trial_meas'])
    lcur = state.get('loss', f(np.nan))
    accept, lnew, lam = decide(scratch, first, lcur, state.get('lambda', 0.0), lambda_up, lambda_down,
                               trial['rot'][0], anchor, pose_w, trial['betas'], betas_w, mt, dtype)
    new = {k: ([np.array(x, copy=True) for x in v] if isinstance(v, list) else
               np.array(v, copy=True) if isinstance(v, np.ndarray) else v) for k, v in state.items()}
    if accept:
        for k in ('rot', 'camera'):
            new[k] = [np.asarray(x, f).copy() for x in trial[k]]
        new['keypoints'] = [np.asarray(im['trial_kp'], f).copy() for im in images]
        new['jac'] = [np.asarray(im['trial_jac'], f).copy() for im in images]
        new['betas'] = np.asarray(trial['betas'], f).copy()
        new['loss'] = lnew
        if meas is not None:
            new['meas'] = np.asarray(meas['trial_meas'], f).copy()
            new['meas_jac'] = np.asarray(meas['trial_meas_jac'], f).copy()
    new['lambda'] = lam
    new['accepted'] = int(state.get('accepted', 0)) + (1 if accept and not first else 0)
    blocks = [image_block(im['targets'], im['weights'], new['keypoints'][i], new['jac'][i], new['camera'][i], n_rot,
                          lam, sigma, nb) for i, im in enumerate(images)]
    S, s = np.zeros((ns, ns)), np.zeros(ns)
    for b in blocks:
        S += b[0]
        s += b[1]
    o2.prior_rows(S, s, new['rot'][0], anchor, pose_w, o=-3)     # joint j >= 1 at the shared columns 3 (j - 1) ..
    if meas is not None:
        meas_rows(S, s, ob, meas['targets'], meas['weights'], new['meas'], new['meas_jac'])
    beta = np.asarray(new['betas'], np.float64)
    if betas_w > 0.0:
        s[ob:] += float(np.float32(betas_w)) * beta
    damp = float(np.float32(betas_w)) + float(lam)
    for j in range(ns):
        S[j, j] += damp if j >= ob else float(lam)
    ds, ok = cholesky_solve(S, s)
    ok = ok and math.isfinite(float(lnew)) and all(b[4] for b in blocks)
    nxt = {'rot': [], 'camera': []}
    body = [exp_gram_schmidt(new['rot'][0][j], ds[3 * (j - 1):3 * j]) for j in range(1, n_rot)]
    for i in range(len(images)):
        X, x = blocks[i][2], blocks[i][3]
        d = np.zeros(N1)
        for j in range(N1):
            v = -x[j]
            for l in range(ns):
                v -= X[j, l] * ds[l]
            d[j] = v
        if ok:
            nxt['rot'].append(np.stack([exp_gram_schmidt(new['rot'][i][0], d[:3])] + body).astype(f))
        else:
            nxt['rot'].append(np.asarray(new['rot'][i], f).copy())
        nxt['camera'].append(lm_add_next(new['camera'][i], d[3:], ok, f))
    nxt['betas'] = lm_add_next(new['betas'], ds[ob:], ok, f)
    return new, nxt, accept, blocks, ds


def gram_schmidt(M):
    """The 6D decoder: b1 = a / |a|, b2 = (b - (b1 . b) b1) / |...|, b3 = b1 x b2 of the first two columns a, b."""
    M = np.asarray(M, np.float64)
    a, b = M[:, 0], M[:, 1]
    b1 = a / max(math.sqrt(a @ a), 1e-12)
    u = b - (b1 @ b) * b1
    b2 = u / max(math.sqrt(u @ u), 1e-12)
    return np.stack([b1, b2, np.cross(b1, b2)], 1)
