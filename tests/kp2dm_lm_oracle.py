"""NumPy float64 restatement of the stacked 2D keypoint + measurement Levenberg-Marquardt step (test infrastructure),
on top of tests/kp2d_lm_oracle.py and tests/kpm_lm_oracle.py.

  loss                              the kernel's total, left to right: the 2D step's keypoint term and pose prior, the
                                    measurement sum (formed on its own, then added), the betas prior
  normal_equations                  A and g before damping: kp2d_lm_oracle's keypoint and pose-prior rows, then the
                                    five measurement rows into the betas block in m order, then betas_w beta into g;
                                    and the diagonal of the keypoint rows alone (the first lambda)
  lm_keypoints_2d_measurements_step shapy_fit_lm_keypoints_2d_measurements_step for one body, the same fp64 operations
                                    in the same order (the kernel is compiled with -fmad=false); as in kp2d_lm_oracle,
                                    softplus' exp / log1p may differ from the device's in the last bit
"""
import math

import numpy as np

import kp2d_lm_oracle as o2
from kp_lm_oracle import DIAG_FLOOR, LAMBDA_INIT, LAMBDA_MAX, LAMBDA_MIN, exp_gram_schmidt
from kpm_lm_oracle import meas_loss


def loss(targets, weights, kp, camera, meas_targets, meas_weights, meas, sigma=math.inf, rot=None, anchor=None,
         pose_w=0.0, betas=None, betas_w=0.0):
    L = o2.loss(targets, weights, kp, camera, sigma, rot, anchor, pose_w)
    L += meas_loss(meas_targets, meas_weights, meas)
    if betas_w > 0.0:
        reg = 0.0
        for x in np.asarray(betas, np.float64):
            reg += x * x
        L += float(np.float32(betas_w)) * reg
    return L


def normal_equations(targets, weights, kp, jac3, camera, meas_targets, meas_weights, meas, meas_jac, sigma=math.inf,
                     rot=None, anchor=None, pose_w=0.0, betas=None, betas_w=0.0):
    """(A, g, diag of the keypoint rows) before damping.  A dropped measurement's value and row are never read."""
    A, g, dg = o2.normal_equations(targets, weights, kp, jac3, camera, sigma, rot, anchor, pose_w)
    nb = len(betas)
    o = len(g) - 3 - nb
    Jm = np.asarray(meas_jac, np.float64)
    for m in range(5):
        u = float(meas_weights[m])
        if not u > 0.0:
            continue
        uj = u * Jm[m]
        A[o:o + nb, o:o + nb] += np.outer(uj, Jm[m])
        g[o:o + nb] += uj * (float(meas[m]) - float(meas_targets[m]))
    if betas_w > 0.0:
        g[o:o + nb] += float(np.float32(betas_w)) * np.asarray(betas, np.float64)
    return A, g, dg


def lm_keypoints_2d_measurements_step(state, targets, weights, meas_targets, meas_weights, lambda_up, lambda_down,
                                      first, trial, trial_kp, trial_jac, trial_meas, trial_meas_jac, sigma=math.inf,
                                      anchor=None, pose_w=0.0, betas_w=0.0, dtype=np.float32):
    """One step for one body.  state: kp2d_lm_oracle.lm_keypoints_2d_step's plus 'meas' (5,) and 'meas_jac' (5, NB)
    (not modified); trial: {'rot', 'betas', 'camera'}.  Returns (new state, next trial, accepted flag)."""
    f = dtype
    lt = loss(targets, weights, trial_kp, trial['camera'], meas_targets, meas_weights, trial_meas, sigma, trial['rot'],
              anchor, pose_w, trial['betas'], betas_w)
    lcur = state.get('loss', f(np.nan))
    accept = bool(first) or (math.isfinite(lt) and lt < float(lcur))
    new = {k: np.array(v, copy=True) if isinstance(v, np.ndarray) else v for k, v in state.items()}
    lnew = lcur
    if accept:
        lnew = f(lt) if math.isfinite(lt) else f(np.nan)
        new.update({k: np.asarray(trial[k], f).copy() for k in ('rot', 'betas', 'camera')})
        new.update(keypoints=np.asarray(trial_kp, f).copy(), jac=np.asarray(trial_jac, f).copy(),
                   meas=np.asarray(trial_meas, f).copy(), meas_jac=np.asarray(trial_meas_jac, f).copy(), loss=lnew)
    A, g, dg = normal_equations(targets, weights, new['keypoints'], new['jac'], new['camera'], meas_targets,
                                meas_weights, new['meas'], new['meas_jac'], sigma, new['rot'], anchor, pose_w,
                                new['betas'], betas_w)
    P = len(g)
    n_rot, nb = new['rot'].shape[0], len(new['betas'])
    o = 3 * n_rot
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
    damp = float(np.float32(betas_w)) + float(lam)
    for j in range(P):
        A[j, j] += damp if o <= j < o + nb else float(lam)
    y, ok = o2._solve(A, g)
    ok = ok and math.isfinite(float(lnew))
    if not ok:
        nxt = {k: np.asarray(new[k], f).copy() for k in ('rot', 'betas', 'camera')}
    else:
        nxt = {'rot': np.stack([exp_gram_schmidt(new['rot'][j], y[3 * j:3 * j + 3]) for j in range(n_rot)]).astype(f),
               'betas': np.array([f(float(new['betas'][i]) + y[o + i]) for i in range(nb)], f),
               'camera': np.array([f(float(new['camera'][i]) + y[o + nb + i]) for i in range(3)], f)}
    return new, nxt, accept
