"""NumPy float64 restatement of the single-image 2D keypoint Levenberg-Marquardt step (test infrastructure), on top of
tests/kp_lm_oracle.py and oracle/lm_oracle.py.  One camera per body: the weak-perspective camera c = (c0, c1, c2)
(intr None), or a perspective camera with known intrinsics intr = (f, px, py) and the translation t.

  softplus             softplus(c0) and its derivative, with F.softplus' threshold of 20
  project              weak perspective p_k = softplus(c0) (kp_k,xy + (c1, c2)); perspective p_k = f (Y_k,x / Y_k,z,
                       Y_k,y / Y_k,z) + (px, py), Y_k = kp_k + t
  jacobian_2d          the weak-perspective (2K, P) Jacobian from the 3D keypoint Jacobian, columns [... | c0 c1 c2]
  jacobian_persp       the perspective (2K, P) Jacobian: rows 2k + c = (f / Y_z) (J_{3k+c} - (Y_c / Y_z) J_{3k+2}), with
                       J_t = I on the t columns
  rot_tangent          R [e_a]x as 9 row-major entries
  keypoint_loss        the robust keypoint term; for the perspective camera +inf when a weighted keypoint has Y_z <= 0
                       or not finite, or f is not finite and > 0 (the depth rule)
  prior_loss           1/2 w sum_j |R_j - R0_j|_F^2 of the given joints, j order, row-major entries
  loss                 the kernel's loss in fp64, left to right: the keypoint term, the pose prior (one term, or one per
                       joint with joint_w), the measurement sum (formed on its own), the betas and expression
                       regularisers
  keypoint_rows        the keypoint rows with IRLS weights, added in place to A and g
  prior_rows           the pose-prior rows (weight w_j / 2, Jacobian R_j [e_a]x, residual R_j - R0_j), added in place
  normal_equations     A (lower triangle used) and g before damping, in the kernel's order: keypoint rows, pose-prior
                       rows, measurement rows into the betas block, betas_w beta and expr_w psi into g; and the diagonal
                       of the keypoint rows alone (the first lambda)
  packed_solve         the kernel's Cholesky and triangular solves on the packed lower triangle, operation for
                       operation (the same operations as lm_oracle.cholesky_solve on a dense matrix)
  lm_keypoints_2d_step shapy_fit_lm_keypoints_2d_step, its measurement, perspective and expressive entries, for one
                       body (lm_kp2d_step_kernel<MEAS, PERSP>): the same fp64 operations in the same order (the kernel
                       is compiled with -fmad=false); exp / log1p of softplus may differ from the device's in the last
                       bit, so with the weak-perspective camera the loss and lambda agree to rounding, not bit for bit
"""
import math

import numpy as np

from oracle.lm_oracle import (DIAG_FLOOR, cholesky_solve, lm_accept, lm_diag_max, lm_kp_next_trial,  # noqa: F401
                              lm_lambda, lm_loss, lm_sq_norm, meas_loss, meas_rows)


def _f32(x):
    return float(np.float32(x))


def softplus(c0):
    """(s, ds/dc0) with F.softplus' threshold of 20."""
    c0 = float(c0)
    if c0 > 20.0:
        return c0, 1.0
    return math.log1p(math.exp(c0)), 1.0 / (1.0 + math.exp(-c0))


def project(kp, last, intr=None):
    """(K, 2): the weak-perspective projection with the camera last (intr None), or the perspective projection of
    Y = kp + last with the intrinsics intr."""
    kp = np.asarray(kp, np.float64)
    if intr is None:
        s, _ = softplus(last[0])
        return s * (kp[:, :2] + np.asarray(last[1:3], np.float64))
    f, px, py = (float(v) for v in intr)
    Y = kp + np.asarray(last, np.float64)
    return np.stack([f * (Y[:, 0] / Y[:, 2]) + px, f * (Y[:, 1] / Y[:, 2]) + py], 1)


def jacobian_2d(kp, jac3, camera):
    """(2K, P): rows 2k + c of the projection, s J_{3k+c} on the rotation and betas columns, ds (kp_kc + c_{1+c}) on
    c0, s on c_{1+c}; the transl columns of jac3 are not read."""
    kp, jac3 = np.asarray(kp, np.float64), np.asarray(jac3, np.float64)
    K, P = kp.shape[0], jac3.shape[1]
    s, ds = softplus(camera[0])
    oc = P - 3
    out = np.zeros((2 * K, P))
    for k in range(K):
        for c in range(2):
            out[2 * k + c, :oc] = s * jac3[3 * k + c, :oc]
            out[2 * k + c, oc] = ds * (kp[k, c] + float(camera[1 + c]))
            out[2 * k + c, oc + 1 + c] = s
    return out


def jacobian_persp(kp, jac3, transl, intr):
    """(2K, P), columns [delta | betas | t]; the transl columns of jac3 are not read."""
    f = float(intr[0])
    Y = np.asarray(kp, np.float64) + np.asarray(transl, np.float64)
    J = np.asarray(jac3, np.float64).copy()
    K, P = Y.shape[0], J.shape[1]
    J.reshape(K, 3, P)[:, :, P - 3:] = np.eye(3)
    out = np.zeros((2 * K, P))
    for k in range(K):
        for c in range(2):
            fz, bz = f / Y[k, 2], Y[k, c] / Y[k, 2]
            out[2 * k + c] = fz * (J[3 * k + c] - bz * J[3 * k + 2])
    return out


def rot_tangent(R, a):
    """R [e_a]x as 9 row-major entries."""
    E = np.zeros((3, 3))
    E[(a + 2) % 3, (a + 1) % 3], E[(a + 1) % 3, (a + 2) % 3] = 1.0, -1.0
    return (np.asarray(R, np.float64) @ E).reshape(9)


def keypoint_loss(targets, weights, kp, last, sigma=math.inf, intr=None):
    """sum_k w_k rho(|p_k - x_k|^2) in k order, weight <= 0 skipped, rho(e) = e sigma^2 / (sigma^2 + e) (e for an
    infinite sigma)."""
    if intr is not None:
        f = float(intr[0])
        if not (f > 0.0 and math.isfinite(f)):
            return math.inf
        Yz = np.asarray(kp, np.float64)[:, 2] + float(last[2])
    with np.errstate(invalid='ignore', over='ignore', divide='ignore'):
        p = project(kp, last, intr)
    s2 = float(sigma) * float(sigma)
    L = 0.0
    for k in range(len(weights)):
        w = float(weights[k])
        if not w > 0.0:
            continue
        if intr is not None and not (Yz[k] > 0.0 and math.isfinite(Yz[k])):
            return math.inf
        with np.errstate(invalid='ignore', over='ignore'):
            dx = p[k, 0] - float(targets[k, 0])
            dy = p[k, 1] - float(targets[k, 1])
            e = dx * dx + dy * dy
            L += w * (e * (s2 / (s2 + e)) if math.isfinite(sigma) else e)
    return L


def prior_loss(rot, anchor, w):
    return 0.5 * _f32(w) * lm_sq_norm(np.asarray(rot, np.float64) - np.asarray(anchor, np.float64))


def loss(targets, weights, kp, last, sigma=math.inf, rot=None, anchor=None, pose_w=0.0, betas=None, betas_w=0.0,
         intr=None, joint_w=None, expr=None, expr_w=0.0, meas=None):
    """The kernel's loss: last is the camera (intr None) or the translation (intr (f, px, py)); joint_w (n_rot,) the
    per-joint prior weights in place of pose_w; meas None or (meas_targets, meas_weights, meas)."""
    L = keypoint_loss(targets, weights, kp, last, sigma, intr)
    if joint_w is None:
        if pose_w > 0.0:
            L += prior_loss(np.asarray(rot, np.float64)[1:], np.asarray(anchor, np.float64)[1:], pose_w)
    else:
        for j in range(1, np.asarray(rot).shape[0]):
            if float(joint_w[j]) > 0.0:
                L += prior_loss(rot[j], anchor[j], joint_w[j])
    if meas is not None:
        L += meas_loss(*meas)
    if betas_w > 0.0:
        L += _f32(betas_w) * lm_sq_norm(betas)
    if expr is not None and expr_w > 0.0:
        L += _f32(expr_w) * lm_sq_norm(expr)
    return L


def keypoint_rows(A, g, targets, weights, p, J2, sigma=math.inf):
    """The rows of the weighted keypoints, x then y, added in place: IRLS weight w_k (sigma^2 / (sigma^2 + e_k))^2,
    Jacobian J2, residual p - x."""
    s2 = float(sigma) * float(sigma)
    for k in range(len(weights)):
        w = float(weights[k])
        if not w > 0.0:
            continue
        dx, dy = p[k, 0] - float(targets[k, 0]), p[k, 1] - float(targets[k, 1])
        wr = w
        if math.isfinite(sigma):
            q = s2 / (s2 + (dx * dx + dy * dy))
            wr = w * (q * q)
        if not wr > 0.0:
            continue
        for c, r in ((0, dx), (1, dy)):
            wj = wr * J2[2 * k + c]
            A += np.outer(wj, J2[2 * k + c])
            g += wj * r


def prior_rows(A, g, rot, anchor, pose_w=0.0, joint_w=None, o=0):
    """The pose-prior rows of joints 1 .. n_rot - 1 with weight w_j > 0 (joint_w[j], or pose_w), added in place in
    joint and e order; joint j's columns are o + 3j .. o + 3j + 2."""
    rot, anchor = np.asarray(rot, np.float64), np.asarray(anchor, np.float64)
    for j in range(1, rot.shape[0]):
        w = float(joint_w[j]) if joint_w is not None else float(pose_w)
        if not w > 0.0:
            continue
        hw = 0.5 * _f32(w)
        D = np.stack([rot_tangent(rot[j], a) for a in range(3)], 1)      # (9, 3)
        res = (rot[j] - anchor[j]).reshape(9)
        b = slice(o + 3 * j, o + 3 * j + 3)
        for e in range(9):
            wj = hw * D[e]
            A[b, b] += np.outer(wj, D[e])
            g[b] += wj * res[e]


def normal_equations(targets, weights, kp, jac3, last, sigma=math.inf, rot=None, anchor=None, pose_w=0.0, betas=None,
                     betas_w=0.0, intr=None, joint_w=None, expr=None, expr_w=0.0, meas=None):
    """(A, g, diag of the keypoint rows) before damping; meas None or (meas_targets, meas_weights, meas, meas_jac).
    Without rot there are no pose-prior rows."""
    with np.errstate(divide='ignore', invalid='ignore'):
        if intr is None:
            J2 = jacobian_2d(kp, jac3, last)
        else:
            J2 = jacobian_persp(kp, jac3, last, intr)
        p = project(kp, last, intr)
    P = J2.shape[1]
    A, g = np.zeros((P, P)), np.zeros(P)
    keypoint_rows(A, g, targets, weights, p, J2, sigma)
    dg = np.diag(A).copy()
    if rot is not None:
        prior_rows(A, g, rot, anchor, pose_w, joint_w)
    ne = 0 if expr is None else len(expr)
    if betas is not None:
        nb = len(betas)
        o = P - 3 - ne - nb
        if meas is not None:
            meas_rows(A, g, o, *meas)
        if betas_w > 0.0:
            g[o:o + nb] += _f32(betas_w) * np.asarray(betas, np.float64)
        if ne and expr_w > 0.0:
            g[o + nb:o + nb + ne] += _f32(expr_w) * np.asarray(expr, np.float64)
    return A, g, dg


def packed_solve(A, g):
    """The kernel's packed Cholesky of the lower triangle of A and the two triangular solves of A delta = -g:
    (delta, ok).  Column j is scaled by the root of its pivot, then the trailing triangle loses col_i col_k; L z = -g
    in column order, then L^T delta = z from the last column."""
    P = len(g)
    L = [np.array(A[i, :i + 1], np.float64) for i in range(P)]         # row i of the packed triangle
    ld = np.zeros(P)
    ok = True
    with np.errstate(invalid='ignore', divide='ignore'):
        for j in range(P):
            d = L[j][j]
            ok = ok and d > 0.0 and math.isfinite(d)
            ljj = math.sqrt(d) if d >= 0 else float('nan')
            ld[j] = ljj
            col = np.zeros(P)
            for i in range(j + 1, P):
                L[i][j] = L[i][j] / ljj
                col[i] = L[i][j]
            for i in range(j + 1, P):
                L[i][j + 1:i + 1] -= col[i] * col[j + 1:i + 1]
        y = -np.asarray(g, np.float64)
        z = np.zeros(P)
        for j in range(P):
            z[j] = y[j] / ld[j]
            for i in range(j + 1, P):
                y[i] -= L[i][j] * z[j]
        for j in range(P - 1, -1, -1):
            y[j] = z[j] / ld[j]
            z[:j] -= L[j][:j] * y[j]
    return y, ok


def lm_keypoints_2d_step(state, targets, weights, lambda_up, lambda_down, first, trial, trial_kp, trial_jac,
                         sigma=math.inf, anchor=None, pose_w=0.0, betas_w=0.0, intr=None, joint_w=None, expr_w=0.0,
                         meas=None, trial_meas=None, dtype=np.float32, solve=None):
    """One step for one body.  state: {'rot' (n_rot, 3, 3), 'betas', 'expression' (NE,) (absent: NE = 0), 'camera'
    (intr None) or 'transl' (intr (f, px, py)), 'keypoints' (K, 3) without t, 'jac' (3K, P), 'loss', 'lambda',
    'accepted'}, with meas also 'meas' (5,) and 'meas_jac' (5, NB) (not modified); trial: {'rot', 'betas',
    'expression', 'camera' or 'transl'}; meas None or (meas_targets, meas_weights), trial_meas (meas (5,), meas_jac
    (5, NB)) of the trial.  Returns (new state, next trial, accepted flag).  dtype: the storage precision (float32 as on
    the device; float64 gives a plain fp64 LM).  solve: packed_solve by default; lm_oracle.cholesky_solve gives the
    same bits."""
    f = dtype
    last = 'camera' if intr is None else 'transl'
    keys = ('rot', 'betas', 'expression', last) if 'expression' in trial else ('rot', 'betas', last)
    lt = loss(targets, weights, trial_kp, trial[last], sigma, trial['rot'], anchor, pose_w, trial['betas'], betas_w,
              intr, joint_w, trial.get('expression'), expr_w,
              None if meas is None else (meas[0], meas[1], trial_meas[0]))
    lcur = state.get('loss', f(np.nan))
    accept = lm_accept(first, lt, lcur)
    new = {k: np.array(v, copy=True) if isinstance(v, np.ndarray) else v for k, v in state.items()}
    lnew = lm_loss(accept, lt, lcur, f)
    if accept:
        new.update({k: np.asarray(trial[k], f).copy() for k in keys})
        new.update(keypoints=np.asarray(trial_kp, f).copy(), jac=np.asarray(trial_jac, f).copy(), loss=lnew)
        if meas is not None:
            new.update(meas=np.asarray(trial_meas[0], f).copy(), meas_jac=np.asarray(trial_meas[1], f).copy())
    A, g, dg = normal_equations(targets, weights, new['keypoints'], new['jac'], new[last], sigma, new['rot'], anchor,
                                pose_w, new['betas'], betas_w, intr, joint_w, new.get('expression'), expr_w,
                                None if meas is None else (meas[0], meas[1], new['meas'], new['meas_jac']))
    lam = lm_lambda(first, accept, state.get('lambda'), lm_diag_max(dg) if first else None, lambda_up, lambda_down, f)
    new['lambda'] = lam
    new['accepted'] = int(state.get('accepted', 0)) + (1 if accept and not first else 0)
    ne = len(new['expression']) if 'expression' in keys else 0
    o = 3 * new['rot'].shape[0]
    oe = o + len(new['betas'])
    for j in range(len(g)):
        if o <= j < oe:
            A[j, j] += _f32(betas_w) + float(lam)
        elif oe <= j < oe + ne:
            A[j, j] += _f32(expr_w) + float(lam)
        else:
            A[j, j] += float(lam)
    y, ok = (solve or packed_solve)(A, g)
    ok = ok and math.isfinite(float(lnew))
    return new, lm_kp_next_trial(new, y, ok, keys, f), accept
