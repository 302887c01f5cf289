"""NumPy float64 restatement of the grouped 2D keypoint Levenberg-Marquardt step (test infrastructure), on top of
tests/kp2d_lm_oracle.py and oracle/lm_oracle.py: the images of one group share their betas, each keeps its rotations
and camera, and the step is the Schur complement of the group's block-arrow normal matrix.

  image_scratch    launch 1 for one image: the bracket of its trial loss (keypoint term + pose prior) and, on the first
                   step, the max of its keypoint-row diagonal over [delta | c] and its betas entries
  decide           the group's decision from the images' scratch: (accept, loss after it, lambda), as lm_group_decide
                   (and lm_group_commit, which also records it in the group state)
  image_block      launch 2 for one image: its normal equations with the columns reordered to [delta | c | beta], the
                   leading block damped by lambda and factored alone; (S_i, s_i, X_i, x_i, ok_i)
  lm_groups_step   shapy_fit_lm_keypoints_2d_groups_step (and _measurements_step, with `meas`) for one group: the
                   same fp64 operations in the same order (the kernels are compiled with -fmad=false); as in
                   kp2d_lm_oracle, softplus' exp / log1p may differ from the device's in the last bit
"""
import math

import numpy as np

import kp2d_lm_oracle as o2
from oracle.lm_oracle import (cholesky_solve, lm_accept, lm_add_next, lm_diag_max, lm_lambda, lm_loss,
                              lm_rot_next, lm_sq_norm, meas_loss, meas_rows)


def reorder(n_rot, nb):
    """The column order [delta | c | beta] of the grouped step, as indices into [delta | beta | c]."""
    o = 3 * n_rot
    return np.array(list(range(o)) + [o + nb, o + nb + 1, o + nb + 2] + list(range(o, o + nb)))


def image_scratch(targets, weights, trial_kp, trial_jac, trial, first, sigma=math.inf, anchor=None, pose_w=0.0,
                  dtype=np.float32):
    """(bracket, dmax over the [delta | c] diagonal from DIAG_FLOOR, the betas diagonal) of one image's trial; the
    diagonal of the trial as stored (dtype), which the first step accepts."""
    lt = o2.loss(targets, weights, trial_kp, trial['camera'], sigma, trial['rot'], anchor, pose_w)
    if not first:
        return lt, None, None
    f = dtype
    _, _, dg = o2.normal_equations(targets, weights, np.asarray(trial_kp, f), np.asarray(trial_jac, f),
                                   np.asarray(trial['camera'], f), sigma)
    nb = len(trial['betas'])
    dg = dg[reorder(np.asarray(trial['rot']).shape[0], nb)]
    return lt, lm_diag_max(dg[:len(dg) - nb]), dg[len(dg) - nb:].copy()


def decide(scratch, first, lcur, lam, lambda_up, lambda_down, trial_betas, betas_w=0.0, meas_terms=None,
           dtype=np.float32):
    """scratch: the images' image_scratch in image order; meas_terms (meas_targets, meas_weights, trial_meas) or None.
    Returns (accept, loss after the decision, lambda)."""
    f = dtype
    L = scratch[0][0]
    for s in scratch[1:]:
        L += s[0]
    if meas_terms is not None:
        L += meas_loss(*meas_terms)
    if betas_w > 0.0:
        L += float(np.float32(betas_w)) * lm_sq_norm(trial_betas)
    accept = lm_accept(first, L, lcur)
    dmax = None
    if first:       # the images' brackets, then the betas diagonal summed over the images in image order
        dmax = lm_diag_max([s[1] for s in scratch])
        for l in range(len(scratch[0][2])):
            d = scratch[0][2][l]
            for s in scratch[1:]:
                d += s[2][l]
            dmax = lm_diag_max([d], dmax)
    return accept, lm_loss(accept, L, lcur, f), lm_lambda(first, accept, lam, dmax, lambda_up, lambda_down, f)


def image_block(targets, weights, kp, jac, camera, rot, lam, sigma=math.inf, anchor=None, pose_w=0.0, nb=None):
    """Launch 2 for one image at its state: (S_i (nb, nb) lower, s_i, X_i (n1, nb), x_i, ok_i)."""
    n_rot = np.asarray(rot).shape[0]
    A, g, _ = o2.normal_equations(targets, weights, kp, jac, camera, sigma, rot, anchor, pose_w)
    perm = reorder(n_rot, nb)
    A, g = A[perm][:, perm].copy(), g[perm].copy()
    n1 = 3 * n_rot + 3
    for j in range(n1):
        A[j, j] += float(lam)
    y, ok = cholesky_solve(A, g, n1)           # A now holds L11, L21 and the Schur block
    W = A[n1:, :n1].copy()                       # the rows of L21, then X^T (lm_kp_solve_rows)
    with np.errstate(invalid='ignore', divide='ignore'):
        for j in range(n1 - 1, -1, -1):
            W[:, j] /= A[j, j]
            W[:, :j] -= np.outer(W[:, j], A[j, :j])
    return np.tril(A[n1:, n1:]), -y[n1:], W.T.copy(), -y[:n1], ok


def lm_groups_step(state, images, lambda_up, lambda_down, first, trial, sigma=math.inf, pose_w=0.0, betas_w=0.0,
                   meas=None, dtype=np.float32):
    """One step for one group.  state: {'rot', 'camera', 'keypoints', 'jac': lists over the images, 'betas' (nb,),
    'loss', 'lambda', 'accepted'} (+ 'meas' (5,), 'meas_jac' (5, nb) with meas); images: a list of {'targets',
    'weights', 'anchor', 'trial_kp', 'trial_jac'}; trial: {'rot', 'camera': lists, 'betas' (nb,)}; meas: None or
    {'targets', 'weights', 'trial_meas', 'trial_meas_jac'}.  Returns (new state, next trial, accepted flag, the
    images' (S_i, s_i, X_i, x_i, ok_i) and dbeta).  dtype: the storage precision (float64 gives a plain fp64 LM)."""
    f = dtype
    M = len(images)
    nb = len(trial['betas'])
    scratch = [image_scratch(im['targets'], im['weights'], im['trial_kp'], im['trial_jac'],
                             {'rot': trial['rot'][i], 'camera': trial['camera'][i], 'betas': trial['betas']}, first,
                             sigma, im.get('anchor'), pose_w, dtype) for i, im in enumerate(images)]
    mt = None if meas is None else (meas['targets'], meas['weights'], meas['trial_meas'])
    lcur = state.get('loss', f(np.nan))
    accept, lnew, lam = decide(scratch, first, lcur, state.get('lambda', 0.0), lambda_up, lambda_down,
                               trial['betas'], betas_w, mt, dtype)
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
    blocks = [image_block(im['targets'], im['weights'], new['keypoints'][i], new['jac'][i], new['camera'][i],
                          new['rot'][i], lam, sigma, im.get('anchor'), pose_w, nb) for i, im in enumerate(images)]
    S, s = np.zeros((nb, nb)), np.zeros(nb)
    for b in blocks:
        S += b[0]
        s += b[1]
    if meas is not None:
        meas_rows(S, s, 0, meas['targets'], meas['weights'], new['meas'], new['meas_jac'])
    beta = np.asarray(new['betas'], np.float64)
    if betas_w > 0.0:
        s += float(np.float32(betas_w)) * beta
    damp = float(np.float32(betas_w)) + float(lam)
    for j in range(nb):
        S[j, j] += damp
    db, ok = cholesky_solve(S, s)
    ok = ok and math.isfinite(float(lnew)) and all(b[4] for b in blocks)
    n_rot = np.asarray(new['rot'][0]).shape[0]
    o = 3 * n_rot
    nxt = {'rot': [], 'camera': []}
    for i in range(M):
        X, x = blocks[i][2], blocks[i][3]
        d = np.zeros(o + 3)
        for j in range(o + 3):
            v = -x[j]
            for l in range(nb):
                v -= X[j, l] * db[l]
            d[j] = v
        nxt['rot'].append(lm_rot_next(new['rot'][i], d, ok, f))
        nxt['camera'].append(lm_add_next(new['camera'][i], d[o:], ok, f))
    nxt['betas'] = lm_add_next(new['betas'], db, ok, f)
    return new, nxt, accept, blocks, db
