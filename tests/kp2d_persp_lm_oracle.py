"""NumPy float64 restatement of the perspective 2D keypoint Levenberg-Marquardt step (test infrastructure), on top of
tests/kp_lm_oracle.py and tests/kp2d_lm_oracle.py.

  project              p_k = f (Y_k,x / Y_k,z, Y_k,y / Y_k,z) + (px, py), Y_k = kp_k + t
  jacobian_persp       the projected (2K, P) Jacobian: rows 2k + c = (f / Y_z) (J_{3k+c} - (Y_c / Y_z) J_{3k+2}), with
                       J_t = I on the t columns (the transl columns of the 3D Jacobian are not read)
  loss                 the kernel's loss in fp64: robust keypoint terms, chordal pose prior, betas prior; +inf when a
                       weighted keypoint has Y_z <= 0 or not finite, or f is not finite and > 0 (the depth rule)
  normal_equations     A and g before damping, in the kernel's order, and the diagonal of the keypoint rows alone
  lm_keypoints_2d_perspective_step
                       shapy_fit_lm_keypoints_2d_perspective_step for one body: the same fp64 operations in the same
                       order (the kernel is compiled with -fmad=false), so accept / reject, lambda and the loss agree bit
                       for bit with float32 storage, and the next trial to the last bits of the solve and of sin / cos
"""
import math

import numpy as np

import kp2d_lm_oracle as o2
from kp_lm_oracle import DIAG_FLOOR, LAMBDA_INIT, LAMBDA_MAX, LAMBDA_MIN, exp_gram_schmidt


def _points(kp, transl):
    """Y = kp + t in float64 (of the float32 values the kernel reads, when given float32)."""
    return np.asarray(kp, np.float64) + np.asarray(transl, np.float64)


def _intr(intr):
    f, px, py = (float(v) for v in intr)
    return f, px, py


def project(kp, transl, intr):
    f, px, py = _intr(intr)
    Y = _points(kp, transl)
    return np.stack([f * (Y[:, 0] / Y[:, 2]) + px, f * (Y[:, 1] / Y[:, 2]) + py], 1)


def jacobian_persp(kp, jac3, transl, intr):
    """(2K, P), columns [delta | betas | t]."""
    f, _, _ = _intr(intr)
    Y = _points(kp, transl)
    J = np.asarray(jac3, np.float64).copy()
    K, P = Y.shape[0], J.shape[1]
    J.reshape(K, 3, P)[:, :, P - 3:] = np.eye(3)
    out = np.zeros((2 * K, P))
    for k in range(K):
        for c in range(2):
            fz, bz = f / Y[k, 2], Y[k, c] / Y[k, 2]
            out[2 * k + c] = fz * (J[3 * k + c] - bz * J[3 * k + 2])
    return out


def loss(targets, weights, kp, transl, intr, sigma=math.inf, rot=None, anchor=None, pose_w=0.0, betas=None,
         betas_w=0.0):
    f, px, py = _intr(intr)
    if not (f > 0.0 and math.isfinite(f)):
        return math.inf
    Y = _points(kp, transl)
    s2 = float(sigma) * float(sigma)
    L = 0.0
    for k in range(len(weights)):
        w = float(weights[k])
        if not w > 0.0:
            continue
        if not (Y[k, 2] > 0.0 and math.isfinite(Y[k, 2])):
            return math.inf
        with np.errstate(invalid='ignore', over='ignore'):
            dx = f * (Y[k, 0] / Y[k, 2]) + px - float(targets[k, 0])
            dy = f * (Y[k, 1] / Y[k, 2]) + py - float(targets[k, 1])
            e = dx * dx + dy * dy
            L += w * (e * (s2 / (s2 + e)) if math.isfinite(sigma) else e)
    if pose_w > 0.0:
        q = 0.0
        for d in (np.asarray(rot, np.float64)[1:] - np.asarray(anchor, np.float64)[1:]).reshape(-1):
            q += d * d
        L += 0.5 * float(np.float32(pose_w)) * q
    if betas_w > 0.0:
        reg = 0.0
        for x in np.asarray(betas, np.float64):
            reg += x * x
        L += float(np.float32(betas_w)) * reg
    return L


def normal_equations(targets, weights, kp, jac3, transl, intr, sigma=math.inf, rot=None, anchor=None, pose_w=0.0,
                     betas=None, betas_w=0.0):
    """(A, g, diag of the keypoint rows) before damping: keypoint rows with IRLS weights at (kp, t), residual p - x,
    then the pose-prior rows (weight pose_w / 2, Jacobian R_j [e_a]x, residual R_j - R0_j), then betas_w beta into g."""
    with np.errstate(divide='ignore', invalid='ignore'):
        J2 = jacobian_persp(kp, jac3, transl, intr)
        p = project(kp, transl, intr)
    P = J2.shape[1]
    s2 = float(sigma) * float(sigma)
    A, g = np.zeros((P, P)), np.zeros(P)
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
    dg = np.diag(A).copy()
    if pose_w > 0.0:
        hw = 0.5 * float(np.float32(pose_w))
        rot, anchor = np.asarray(rot, np.float64), np.asarray(anchor, np.float64)
        for j in range(1, rot.shape[0]):
            D = np.stack([o2.rot_tangent(rot[j], a) for a in range(3)], 1)      # (9, 3)
            res = (rot[j] - anchor[j]).reshape(9)
            for e in range(9):
                row = np.zeros(P)
                row[3 * j:3 * j + 3] = D[e]
                wj = hw * row
                A += np.outer(wj, row)
                g += wj * res[e]
    if betas_w > 0.0:
        o = 3 * np.asarray(rot).shape[0]
        g[o:o + len(betas)] += float(np.float32(betas_w)) * np.asarray(betas, np.float64)
    return A, g, dg


def lm_keypoints_2d_perspective_step(state, targets, weights, intr, lambda_up, lambda_down, first, trial, trial_kp,
                                     trial_jac, sigma=math.inf, anchor=None, pose_w=0.0, betas_w=0.0,
                                     dtype=np.float32):
    """One step for one body.  state: {'rot' (n_rot, 3, 3), 'betas', 'transl', 'keypoints' (K, 3) without t, 'jac'
    (3K, P), 'loss', 'lambda', 'accepted'} (not modified); trial: {'rot', 'betas', 'transl'}; intr (f, px, py).
    Returns (new state, next trial, accepted flag).  dtype: the storage precision (float32 as on the device; float64
    gives a plain fp64 LM)."""
    f = dtype
    lt = loss(targets, weights, trial_kp, trial['transl'], intr, sigma, trial['rot'], anchor, pose_w, trial['betas'],
              betas_w)
    lcur = state.get('loss', f(np.nan))
    accept = bool(first) or (math.isfinite(lt) and lt < float(lcur))
    new = {k: np.array(v, copy=True) if isinstance(v, np.ndarray) else v for k, v in state.items()}
    lnew = lcur
    if accept:
        lnew = f(lt) if math.isfinite(lt) else f(np.nan)
        new.update({k: np.asarray(trial[k], f).copy() for k in ('rot', 'betas', 'transl')})
        new.update(keypoints=np.asarray(trial_kp, f).copy(), jac=np.asarray(trial_jac, f).copy(), loss=lnew)
    A, g, dg = normal_equations(targets, weights, new['keypoints'], new['jac'], new['transl'], intr, sigma,
                                new['rot'], anchor, pose_w, new['betas'], betas_w)
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
        nxt = {k: np.asarray(new[k], f).copy() for k in ('rot', 'betas', 'transl')}
    else:
        nxt = {'rot': np.stack([exp_gram_schmidt(new['rot'][j], y[3 * j:3 * j + 3]) for j in range(n_rot)]).astype(f),
               'betas': np.array([f(float(new['betas'][i]) + y[o + i]) for i in range(nb)], f),
               'transl': np.array([f(float(new['transl'][i]) + y[o + nb + i]) for i in range(3)], f)}
    return new, nxt, accept
