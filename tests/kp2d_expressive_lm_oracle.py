"""NumPy float64 restatement of the wide 2D keypoint Levenberg-Marquardt step (test infrastructure), on top of
tests/kp_lm_oracle.py, tests/kp2d_lm_oracle.py and tests/kp2d_persp_lm_oracle.py.

  keypoint_jacobian_expr   shapy_smplx_keypoint_jacobian_expr for one body: kp_lm_oracle.keypoint_jacobian with the
                           expression rows appended to the shape basis (they are shape rows NB .. NC-1), columns
                           [delta_j | betas | expression | transl]
  loss                     the step's loss in fp64: the 2D (or perspective) keypoint term and pose prior (scalar or
                           per joint), the betas and expression regularisers
  normal_equations         A and g before damping, in the kernel's order, and the diagonal of the keypoint rows alone
  packed_solve             the kernel's Cholesky and triangular solves on the packed lower triangle, operation for
                           operation (the same operations as kp2d_lm_oracle._solve on a dense matrix)
  lm_keypoints_2d_expressive_step
                           shapy_fit_lm_keypoints_2d_expressive_step (intr None) or its perspective entry for one body
"""
import math

import numpy as np
import torch

import kp2d_lm_oracle as o2
import kp2d_persp_lm_oracle as op
from kp_lm_oracle import DIAG_FLOOR, LAMBDA_INIT, LAMBDA_MAX, LAMBDA_MIN, exp_gram_schmidt, keypoint_jacobian


def keypoint_jacobian_expr(model, betas, expr, rot, transl=None, use_face_contour=True):
    """One body: betas (NB,), expr (NE,), rot (n_rot, 3, 3) -> (keypoints (K, 3), jac (3K, 3 n_rot + NB + NE + 3))."""
    m = dict(model)
    m['shapedirs'] = torch.cat([torch.as_tensor(model['shapedirs']), torch.as_tensor(model['expr_dirs'])], 2)
    coef = np.concatenate([np.asarray(betas, np.float64), np.asarray(expr, np.float64)])
    return keypoint_jacobian(m, coef, rot, transl, use_face_contour)


def _f32(x):
    return float(np.float32(x))


def loss(targets, weights, kp, last, sigma=math.inf, rot=None, anchor=None, pose_w=0.0, joint_w=None, betas=None,
         betas_w=0.0, expr=None, expr_w=0.0, intr=None):
    """The kernel's loss: last is the camera (intr None) or the translation (intr (f, px, py))."""
    pw = 0.0 if joint_w is not None else pose_w
    if intr is None:
        L = o2.loss(targets, weights, kp, last, sigma, rot, anchor, pw)
    else:
        L = op.loss(targets, weights, kp, last, intr, sigma, rot, anchor, pw)
    if joint_w is not None:
        rot, anchor = np.asarray(rot, np.float64), np.asarray(anchor, np.float64)
        for j in range(1, rot.shape[0]):
            if not float(joint_w[j]) > 0.0:
                continue
            q = 0.0
            for d in (rot[j] - anchor[j]).reshape(-1):
                q += d * d
            L += (0.5 * _f32(joint_w[j])) * q
    for x, w in ((betas, betas_w), (expr, expr_w)):
        if w > 0.0:
            reg = 0.0
            for v in np.asarray(x, np.float64):
                reg += v * v
            L += _f32(w) * reg
    return L


def normal_equations(targets, weights, kp, jac3, last, sigma=math.inf, rot=None, anchor=None, pose_w=0.0,
                     joint_w=None, betas=None, betas_w=0.0, expr=None, expr_w=0.0, intr=None):
    """(A, g, diag of the keypoint rows) before damping: keypoint rows, then the pose-prior rows of joints 1 ..
    n_rot - 1 (weight w_j / 2), then betas_w beta and expr_w psi into g."""
    if intr is None:
        A, g, dg = o2.normal_equations(targets, weights, kp, jac3, last, sigma)
    else:
        A, g, dg = op.normal_equations(targets, weights, kp, jac3, last, intr, sigma)
    P = len(g)
    n_rot = np.asarray(rot).shape[0]
    rot = np.asarray(rot, np.float64)
    for j in range(1, n_rot):
        wj = float(joint_w[j]) if joint_w is not None else float(pose_w)
        if not wj > 0.0:
            continue
        hw = 0.5 * _f32(wj)
        anc = np.asarray(anchor, np.float64)
        D = np.stack([o2.rot_tangent(rot[j], a) for a in range(3)], 1)      # (9, 3)
        res = (rot[j] - anc[j]).reshape(9)
        for e in range(9):
            row = np.zeros(P)
            row[3 * j:3 * j + 3] = D[e]
            wj_row = hw * row
            A += np.outer(wj_row, row)
            g += wj_row * res[e]
    o = 3 * n_rot
    nb = len(betas)
    if betas_w > 0.0:
        g[o:o + nb] += _f32(betas_w) * np.asarray(betas, np.float64)
    if expr is not None and len(expr) and expr_w > 0.0:
        g[o + nb:o + nb + len(expr)] += _f32(expr_w) * np.asarray(expr, np.float64)
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


def lm_keypoints_2d_expressive_step(state, targets, weights, lambda_up, lambda_down, first, trial, trial_kp,
                                    trial_jac, sigma=math.inf, anchor=None, pose_w=0.0, joint_w=None, betas_w=0.0,
                                    expr_w=0.0, intr=None, dtype=np.float32, solve=None):
    """One step for one body.  state: {'rot' (n_rot, 3, 3), 'betas', 'expression' (NE,), 'camera' or 'transl',
    'keypoints' (K, 3), 'jac' (3K, P), 'loss', 'lambda', 'accepted'} (not modified); trial: {'rot', 'betas',
    'expression', 'camera' or 'transl'}.  Returns (new state, next trial, accepted flag).  dtype: the storage
    precision (float32 as on the device; float64 gives a plain fp64 LM).  solve: packed_solve by default; the dense
    kp2d_lm_oracle._solve gives the same bits."""
    f = dtype
    last = 'camera' if intr is None else 'transl'
    keys = ('rot', 'betas', 'expression', last)
    lt = loss(targets, weights, trial_kp, trial[last], sigma, trial['rot'], anchor, pose_w, joint_w, trial['betas'],
              betas_w, trial['expression'], expr_w, intr)
    lcur = state.get('loss', f(np.nan))
    accept = bool(first) or (math.isfinite(lt) and lt < float(lcur))
    new = {k: np.array(v, copy=True) if isinstance(v, np.ndarray) else v for k, v in state.items()}
    lnew = lcur
    if accept:
        lnew = f(lt) if math.isfinite(lt) else f(np.nan)
        new.update({k: np.asarray(trial[k], f).copy() for k in keys})
        new.update(keypoints=np.asarray(trial_kp, f).copy(), jac=np.asarray(trial_jac, f).copy(), loss=lnew)
    A, g, dg = normal_equations(targets, weights, new['keypoints'], new['jac'], new[last], sigma, new['rot'], anchor,
                                pose_w, joint_w, new['betas'], betas_w, new['expression'], expr_w, intr)
    P = len(g)
    n_rot, nb, ne = new['rot'].shape[0], len(new['betas']), len(new['expression'])
    o, oe = 3 * n_rot, 3 * n_rot + nb
    if first:
        dmax = DIAG_FLOOR
        for j in range(P):
            dmax = float(np.fmax(dmax, dg[j]))
        lam = f(LAMBDA_INIT * dmax)
    elif accept:
        lam = f(f(state['lambda']) / f(lambda_down))
    else:
        lam = f(f(state['lambda']) * f(lambda_up))
    lam = f(np.fmin(np.fmax(lam, f(LAMBDA_MIN)), f(LAMBDA_MAX)))
    new['lambda'] = lam
    new['accepted'] = int(state.get('accepted', 0)) + (1 if accept and not first else 0)
    for j in range(P):
        if o <= j < oe:
            A[j, j] += _f32(betas_w) + float(lam)
        elif oe <= j < oe + ne:
            A[j, j] += _f32(expr_w) + float(lam)
        else:
            A[j, j] += float(lam)
    y, ok = (solve or packed_solve)(A, g)
    ok = ok and math.isfinite(float(lnew))
    if not ok:
        nxt = {k: np.asarray(new[k], f).copy() for k in keys}
    else:
        nxt = {'rot': np.stack([exp_gram_schmidt(new['rot'][j], y[3 * j:3 * j + 3]) for j in range(n_rot)]).astype(f),
               'betas': np.array([f(float(new['betas'][i]) + y[o + i]) for i in range(nb)], f),
               'expression': np.array([f(float(new['expression'][i]) + y[oe + i]) for i in range(ne)], f),
               last: np.array([f(float(new[last][i]) + y[oe + ne + i]) for i in range(3)], f)}
    return new, nxt, accept
