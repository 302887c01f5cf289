"""NumPy float64 restatement of the grouped 2D keypoint Levenberg-Marquardt step (test infrastructure), on top of
tests/kp2d_lm_oracle.py and tests/kpm_lm_oracle.py: the images of one group share their betas, each keeps its rotations
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
from kp_lm_oracle import DIAG_FLOOR, LAMBDA_INIT, LAMBDA_MAX, LAMBDA_MIN, exp_gram_schmidt
from kpm_lm_oracle import meas_loss


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
    dmax = DIAG_FLOOR
    for j in range(len(dg) - nb):
        dmax = float(np.fmax(dmax, dg[j]))
    return lt, dmax, dg[len(dg) - nb:].copy()


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
        reg = 0.0
        for x in np.asarray(trial_betas, np.float64):
            reg += x * x
        L += float(np.float32(betas_w)) * reg
    accept = bool(first) or (math.isfinite(L) and L < float(lcur))
    lnew = (f(L) if math.isfinite(L) else f(np.nan)) if accept else lcur
    if first:
        dmax = DIAG_FLOOR
        for s in scratch:
            dmax = float(np.fmax(dmax, s[1]))
        for l in range(len(scratch[0][2])):
            d = scratch[0][2][l]
            for s in scratch[1:]:
                d += s[2][l]
            dmax = float(np.fmax(dmax, d))
        lam = f(LAMBDA_INIT * dmax)
    elif accept:
        lam = f(f(lam) / f(lambda_down))
    else:
        lam = f(f(lam) * f(lambda_up))
    return accept, lnew, f(np.fmin(np.fmax(lam, f(LAMBDA_MIN)), f(LAMBDA_MAX)))


def _solve_partial(A, g, n):
    """lm_kp_solve with its leading n columns eliminated: (A with L11, L21 and the Schur block, y, ok)."""
    P = len(g)
    ok = True
    with np.errstate(invalid='ignore', divide='ignore'):
        for j in range(n):
            d = A[j, j]
            ok = ok and d > 0.0 and math.isfinite(d)
            ljj = math.sqrt(d) if d >= 0 else float('nan')
            A[j, j] = ljj
            A[j + 1:, j] /= ljj
            A[j + 1:, j + 1:] -= np.outer(A[j + 1:, j], A[j + 1:, j])
        y = -g
        for j in range(n):
            y[j] = y[j] / A[j, j]
            y[j + 1:] -= A[j + 1:, j] * y[j]
        for j in range(n - 1, -1, -1):
            y[j] = y[j] / A[j, j]
            y[:j] -= A[j, :j] * y[j]
    return A, y, ok


def image_block(targets, weights, kp, jac, camera, rot, lam, sigma=math.inf, anchor=None, pose_w=0.0, nb=None):
    """Launch 2 for one image at its state: (S_i (nb, nb) lower, s_i, X_i (n1, nb), x_i, ok_i)."""
    n_rot = np.asarray(rot).shape[0]
    A, g, _ = o2.normal_equations(targets, weights, kp, jac, camera, sigma, rot, anchor, pose_w)
    perm = reorder(n_rot, nb)
    A, g = A[perm][:, perm].copy(), g[perm].copy()
    n1 = 3 * n_rot + 3
    for j in range(n1):
        A[j, j] += float(lam)
    A, y, ok = _solve_partial(A, g, n1)
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
        Jm = np.asarray(new['meas_jac'], np.float64)
        for m in range(5):
            u = float(meas['weights'][m])
            if not u > 0.0:
                continue
            uj = u * Jm[m]
            S += np.outer(uj, Jm[m])
            s += uj * (float(new['meas'][m]) - float(meas['targets'][m]))
    beta = np.asarray(new['betas'], np.float64)
    if betas_w > 0.0:
        s += float(np.float32(betas_w)) * beta
    damp = float(np.float32(betas_w)) + float(lam)
    for j in range(nb):
        S[j, j] += damp
    db, ok = o2._solve(S, s)
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
        if ok:
            nxt['rot'].append(np.stack([exp_gram_schmidt(new['rot'][i][j], d[3 * j:3 * j + 3])
                                        for j in range(n_rot)]).astype(f))
            nxt['camera'].append(np.array([f(float(new['camera'][i][t]) + d[o + t]) for t in range(3)], f))
        else:
            nxt['rot'].append(np.asarray(new['rot'][i], f).copy())
            nxt['camera'].append(np.asarray(new['camera'][i], f).copy())
    nxt['betas'] = (np.array([f(float(new['betas'][l]) + db[l]) for l in range(nb)], f) if ok
                    else np.asarray(new['betas'], f).copy())
    return new, nxt, accept, blocks, db
