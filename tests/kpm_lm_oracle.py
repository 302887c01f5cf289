"""NumPy float64 restatement of the stacked keypoint + measurement Levenberg-Marquardt step (test infrastructure).

  lm_keypoints_measurements_step    shapy_fit_lm_keypoints_measurements_step for one body: the fp64 operations of
                                    kp_lm_oracle.lm_keypoints_step with the five measurement rows and the betas
                                    regulariser stacked under the keypoint rows, in the kernel's order (the kernel is
                                    compiled with -fmad=false), so accept / reject, lambda and the loss agree bit for bit
                                    with float32 storage, and the next trial to the last bits of the fp64 solve and of
                                    sin / cos
"""
import math

import numpy as np

from kp_lm_oracle import DIAG_FLOOR, LAMBDA_INIT, LAMBDA_MAX, LAMBDA_MIN, exp_gram_schmidt, loss as kp_loss


def meas_loss(targets, weights, meas):
    """sum_{w_k > 0} w_k (t_k - m_k)^2 in k order, fp64 (lm_step_kernel's data term)."""
    L = 0.0
    for k in range(5):
        w = float(weights[k])
        if w > 0.0:
            r = float(targets[k]) - float(meas[k])
            L += w * r * r
    return L


def loss(kp_targets, kp_weights, kp, meas_targets, meas_weights, meas, rho, betas):
    """The kernel's total: L_kp + L_meas + rho |betas|^2, left to right; rho (float32) <= 0 adds nothing."""
    L = kp_loss(kp_targets, kp_weights, kp) + meas_loss(meas_targets, meas_weights, meas)
    rho = float(np.float32(rho))
    if rho > 0.0:
        reg = 0.0
        for x in betas:
            reg += float(x) * float(x)
        L += rho * reg
    return L


def lm_keypoints_measurements_step(state, targets, weights, meas_targets, meas_weights, betas_weight, lambda_up,
                                   lambda_down, first, trial, trial_kp, trial_jac, trial_meas, trial_meas_jac,
                                   dtype=np.float32, return_delta=False):
    """One step for one body.  state: kp_lm_oracle.lm_keypoints_step's plus 'meas' (5,) and 'meas_jac' (5, NB) (not
    modified); trial: {'rot', 'betas', 'transl'}.  Returns (new state, next trial, accepted flag), and with
    return_delta the solved step delta (P,) as a fourth item.  dtype: the storage precision (float32 as on the device;
    float64 gives a plain fp64 LM)."""
    f = dtype
    rho = float(np.float32(betas_weight))
    lt = loss(targets, weights, trial_kp, meas_targets, meas_weights, trial_meas, rho, trial['betas'])
    lcur = state.get('loss', f(np.nan))
    accept = bool(first) or (math.isfinite(lt) and lt < float(lcur))
    new = {k: np.array(v, copy=True) if isinstance(v, np.ndarray) else v for k, v in state.items()}
    lnew = lcur
    if accept:
        lnew = f(lt) if math.isfinite(lt) else f(np.nan)
        new.update({k: np.asarray(trial[k], f).copy() for k in ('rot', 'betas', 'transl')})
        new.update(keypoints=np.asarray(trial_kp, f).copy(), jac=np.asarray(trial_jac, f).copy(),
                   meas=np.asarray(trial_meas, f).copy(), meas_jac=np.asarray(trial_meas_jac, f).copy(), loss=lnew)
    Jk = np.asarray(new['jac'], np.float64)
    M = np.asarray(new['keypoints'], np.float64).reshape(-1)
    tg = np.asarray(targets, np.float64).reshape(-1)
    P = Jk.shape[1]
    n_rot = new['rot'].shape[0]
    nb = len(new['betas'])
    o = 3 * n_rot
    A, g = np.zeros((P, P)), np.zeros(P)
    # keypoint rows in keypoint-major xyz order, then the measurement rows into the betas block in k order
    for r in range(Jk.shape[0]):
        w = float(weights[r // 3])
        if not w > 0.0:
            continue
        wj = w * Jk[r]
        A += np.outer(wj, Jk[r])
        g += wj * (M[r] - tg[r])
    Jm = np.asarray(new['meas_jac'], np.float64)
    for k in range(5):
        w = float(meas_weights[k])
        if not w > 0.0:
            continue
        wj = w * Jm[k]
        A[o:o + nb, o:o + nb] += np.outer(wj, Jm[k])
        g[o:o + nb] += wj * (float(new['meas'][k]) - float(meas_targets[k]))
    if rho > 0.0:
        g[o:o + nb] += rho * np.asarray(new['betas'], np.float64)
    if first:
        dmax = DIAG_FLOOR
        for j in range(P):
            dmax = float(np.fmax(dmax, A[j, j]))
        lam = f(LAMBDA_INIT * dmax)
    elif accept:
        lam = f(f(state['lambda']) / f(lambda_down))
    else:
        lam = f(f(state['lambda']) * f(lambda_up))
    lam = f(np.fmin(np.fmax(lam, f(LAMBDA_MIN)), f(LAMBDA_MAX)))
    new['lambda'] = lam
    new['accepted'] = int(state.get('accepted', 0)) + (1 if accept and not first else 0)
    damp = rho + float(lam)
    for j in range(P):
        A[j, j] += damp if o <= j < o + nb else float(lam)
    ok = math.isfinite(float(lnew))
    with np.errstate(invalid='ignore', divide='ignore'):
        for j in range(P):
            d = A[j, j]
            ok = ok and d > 0.0 and math.isfinite(d)
            ljj = math.sqrt(d) if d >= 0 else float('nan')
            A[j, j] = ljj
            A[j + 1:, j] /= ljj
            A[j + 1:, j + 1:] -= np.outer(A[j + 1:, j], A[j + 1:, j])
        y = -g
        for j in range(P):
            y[j] = y[j] / A[j, j]
            y[j + 1:] -= A[j + 1:, j] * y[j]
        for j in range(P - 1, -1, -1):
            y[j] = y[j] / A[j, j]
            y[:j] -= A[j, :j] * y[j]
    if not ok:
        nxt = {k: np.asarray(new[k], f).copy() for k in ('rot', 'betas', 'transl')}
    else:
        nxt = {'rot': np.stack([exp_gram_schmidt(new['rot'][j], y[3 * j:3 * j + 3]) for j in range(n_rot)]).astype(f),
               'betas': np.array([f(float(new['betas'][i]) + y[o + i]) for i in range(nb)], f),
               'transl': np.array([f(float(new['transl'][i]) + y[o + nb + i]) for i in range(3)], f)}
    return (new, nxt, accept, y) if return_delta else (new, nxt, accept)
