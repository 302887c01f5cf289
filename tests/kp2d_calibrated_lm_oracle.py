"""NumPy float64 restatement of the calibrated 2D keypoint Levenberg-Marquardt step (test infrastructure), on top of
tests/kp2d_lm_oracle.py and oracle/lm_oracle.py.  One body seen by V views, each with intrinsics (f, px, py) and
world-to-camera extrinsics ext (12,) = R row-major, then T.

  camera_points        Y_k = R (kp_k + t) + T in float64
  project              p_k = f (Y_k,x / Y_k,z, Y_k,y / Y_k,z) + (px, py)
  jacobian_calibrated  one view's projected (2K, P) Jacobian: row 2k + c = u . J3_k, u = (f / Y_z) (R[c, :] -
                       (Y_c / Y_z) R[2, :]), J3_k the (3 x P) block of keypoint k with J_t = I (u on the t columns)
  loss                 the kernel's loss in fp64: the keypoint term of each view (kp2d_lm_oracle.keypoint_loss of its
                       camera-frame points, depth rule included) in view order, then the pose prior, the measurement sum
                       and the betas prior
  normal_equations     A and g before damping: the keypoint rows of the views in order, then the pose-prior rows
                       (accumulated on their own, then added), the measurement rows and betas_w beta; and the diagonal
                       of the keypoint rows alone (the first lambda)
  lm_keypoints_2d_calibrated_step
                       shapy_fit_lm_keypoints_2d_calibrated_step for one body: accept / reject, lambda and the loss
                       agree with float32 storage, the next trial to the last bits of the solve and of sin / cos
"""
import math

import numpy as np

import kp2d_lm_oracle as o2
from oracle.lm_oracle import (cholesky_solve, lm_accept, lm_diag_max, lm_kp_next_trial, lm_lambda, lm_loss,
                              lm_sq_norm, meas_loss, meas_rows)


def _ext(ext):
    e = np.asarray(ext, np.float64).reshape(12)
    return e[:9].reshape(3, 3), e[9:]


def camera_points(kp, transl, ext):
    R, T = _ext(ext)
    X = np.asarray(kp, np.float64) + np.asarray(transl, np.float64)
    return np.stack([R[c, 0] * X[:, 0] + R[c, 1] * X[:, 1] + R[c, 2] * X[:, 2] + T[c] for c in range(3)], 1)


def project(kp, transl, intr, ext):
    return o2.project(camera_points(kp, transl, ext), np.zeros(3), intr)


def jacobian_calibrated(kp, jac3, transl, intr, ext):
    """(2K, P), columns [delta | betas | t]."""
    R, _ = _ext(ext)
    f = float(intr[0])
    Y = camera_points(kp, transl, ext)
    J = np.asarray(jac3, np.float64).copy()
    K, P = Y.shape[0], J.shape[1]
    J.reshape(K, 3, P)[:, :, P - 3:] = np.eye(3)
    out = np.zeros((2 * K, P))
    for k in range(K):
        for c in range(2):
            u = (f / Y[k, 2]) * (R[c] - (Y[k, c] / Y[k, 2]) * R[2])
            out[2 * k + c] = u @ J[3 * k:3 * k + 3]
    return out


def loss(views, kp, transl, sigma=math.inf, rot=None, anchor=None, pose_w=0.0, betas=None, betas_w=0.0, meas=None):
    """views: (targets (V, K, 2), weights (V, K), intr (V, 3), ext (V, 12)); meas None or (meas_targets, meas_weights,
    meas)."""
    tg, wt, intr, ext = views
    L = 0.0
    for v in range(len(wt)):
        with np.errstate(invalid='ignore', over='ignore', divide='ignore'):
            Y = camera_points(kp, transl, ext[v])
        L += o2.keypoint_loss(tg[v], wt[v], Y, np.zeros(3), sigma, intr[v])
    if pose_w > 0.0:
        L += o2.prior_loss(np.asarray(rot, np.float64)[1:], np.asarray(anchor, np.float64)[1:], pose_w)
    if meas is not None:
        L += meas_loss(*meas)
    if betas_w > 0.0:
        L += float(np.float32(betas_w)) * lm_sq_norm(betas)
    return L


def normal_equations(views, kp, jac3, transl, sigma=math.inf, rot=None, anchor=None, pose_w=0.0, betas=None,
                     betas_w=0.0, meas=None):
    """(A, g, diag of the keypoint rows) before damping; meas None or (meas_targets, meas_weights, meas, meas_jac)."""
    tg, wt, intr, ext = views
    P = np.asarray(jac3).shape[1]
    A, g = np.zeros((P, P)), np.zeros(P)
    for v in range(len(wt)):
        with np.errstate(divide='ignore', invalid='ignore'):
            J2 = jacobian_calibrated(kp, jac3, transl, intr[v], ext[v])
            p = project(kp, transl, intr[v], ext[v])
        o2.keypoint_rows(A, g, tg[v], wt[v], p, J2, sigma)
    dg = np.diag(A).copy()
    Ap, gp = np.zeros((P, P)), np.zeros(P)
    o2.prior_rows(Ap, gp, rot, anchor, pose_w)
    A += Ap
    g += gp
    nb = len(betas)
    o = P - 3 - nb
    if meas is not None:
        meas_rows(A, g, o, *meas)
    if betas_w > 0.0:
        g[o:o + nb] += float(np.float32(betas_w)) * np.asarray(betas, np.float64)
    return A, g, dg


def lm_keypoints_2d_calibrated_step(state, views, lambda_up, lambda_down, first, trial, trial_kp, trial_jac,
                                    sigma=math.inf, anchor=None, pose_w=0.0, betas_w=0.0, meas=None, trial_meas=None,
                                    dtype=np.float32):
    """One step for one body.  state: {'rot' (n_rot, 3, 3), 'betas', 'transl', 'keypoints' (K, 3) without t, 'jac'
    (3K, P), 'loss', 'lambda', 'accepted'} and with meas also 'meas' (5,), 'meas_jac' (5, NB) (not modified); trial:
    {'rot', 'betas', 'transl'}; meas None or (meas_targets, meas_weights), trial_meas (meas (5,), meas_jac (5, NB)) of
    the trial.  Returns (new state, next trial, accepted flag).  dtype: the storage precision (float32 as on the
    device; float64 gives a plain fp64 LM)."""
    f = dtype
    lt = loss(views, trial_kp, trial['transl'], sigma, trial['rot'], anchor, pose_w, trial['betas'], betas_w,
              None if meas is None else (meas[0], meas[1], trial_meas[0]))
    lcur = state.get('loss', f(np.nan))
    accept = lm_accept(first, lt, lcur)
    new = {k: np.array(v, copy=True) if isinstance(v, np.ndarray) else v for k, v in state.items()}
    lnew = lm_loss(accept, lt, lcur, f)
    if accept:
        new.update({k: np.asarray(trial[k], f).copy() for k in ('rot', 'betas', 'transl')})
        new.update(keypoints=np.asarray(trial_kp, f).copy(), jac=np.asarray(trial_jac, f).copy(), loss=lnew)
        if meas is not None:
            new.update(meas=np.asarray(trial_meas[0], f).copy(), meas_jac=np.asarray(trial_meas[1], f).copy())
    A, g, dg = normal_equations(views, new['keypoints'], new['jac'], new['transl'], sigma, new['rot'], anchor, pose_w,
                                new['betas'], betas_w,
                                None if meas is None else (meas[0], meas[1], new['meas'], new['meas_jac']))
    P = len(g)
    n_rot, nb = new['rot'].shape[0], len(new['betas'])
    o = 3 * n_rot
    lam = lm_lambda(first, accept, state.get('lambda'), lm_diag_max(dg) if first else None, lambda_up, lambda_down, f)
    new['lambda'] = lam
    new['accepted'] = int(state.get('accepted', 0)) + (1 if accept and not first else 0)
    damp = float(np.float32(betas_w)) + float(lam)
    for j in range(P):
        A[j, j] += damp if o <= j < o + nb else float(lam)
    y, ok = cholesky_solve(A, g)
    ok = ok and math.isfinite(float(lnew))
    return new, lm_kp_next_trial(new, y, ok, ('rot', 'betas', 'transl'), f), accept
