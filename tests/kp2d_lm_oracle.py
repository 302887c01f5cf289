"""NumPy float64 restatement of the 2D keypoint Levenberg-Marquardt step (test infrastructure), on top of
tests/kp_lm_oracle.py.

  project              the weak-perspective projection p_k = softplus(c0) (kp_k,xy + (c1, c2))
  jacobian_2d          the projected (2K, P) Jacobian from the 3D keypoint Jacobian, columns [delta | betas | c0 c1 c2]
  loss                 the kernel's loss in fp64: robust keypoint terms, chordal pose prior, betas prior
  normal_equations     A (lower triangle used) and g of the kernel before damping, and the diagonal of the keypoint
                       rows alone (the first lambda)
  lm_keypoints_2d_step shapy_fit_lm_keypoints_2d_step for one body: the same fp64 operations in the same order (the
                       kernel is compiled with -fmad=false); exp / log1p of softplus may differ from the device's in
                       the last bit, so the loss and lambda agree to rounding, not bit for bit
"""
import math

import numpy as np

from kp_lm_oracle import DIAG_FLOOR, LAMBDA_INIT, LAMBDA_MAX, LAMBDA_MIN, exp_gram_schmidt


def softplus(c0):
    """(s, ds/dc0) with F.softplus' threshold of 20."""
    c0 = float(c0)
    if c0 > 20.0:
        return c0, 1.0
    return math.log1p(math.exp(c0)), 1.0 / (1.0 + math.exp(-c0))


def project(kp, camera):
    s, _ = softplus(camera[0])
    kp = np.asarray(kp, np.float64)
    return s * (kp[:, :2] + np.asarray(camera[1:3], np.float64))


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


def rot_tangent(R, a):
    """R [e_a]x as 9 row-major entries."""
    E = np.zeros((3, 3))
    E[(a + 2) % 3, (a + 1) % 3], E[(a + 1) % 3, (a + 2) % 3] = 1.0, -1.0
    return (np.asarray(R, np.float64) @ E).reshape(9)


def loss(targets, weights, kp, camera, sigma=math.inf, rot=None, anchor=None, pose_w=0.0, betas=None, betas_w=0.0):
    s, _ = softplus(camera[0])
    cx, cy = float(camera[1]), float(camera[2])
    s2 = float(sigma) * float(sigma)
    L = 0.0
    for k in range(len(weights)):
        w = float(weights[k])
        if not w > 0.0:
            continue
        dx = s * (float(kp[k, 0]) + cx) - float(targets[k, 0])
        dy = s * (float(kp[k, 1]) + cy) - float(targets[k, 1])
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


def normal_equations(targets, weights, kp, jac3, camera, sigma=math.inf, rot=None, anchor=None, pose_w=0.0,
                     betas=None, betas_w=0.0):
    """(A, g, diag of the keypoint rows) before damping, in the kernel's order: keypoint rows with IRLS weights at
    (kp, camera), then the pose-prior rows (weight pose_w / 2, Jacobian R_j [e_a]x, residual R_j - R0_j), then
    betas_w beta into g."""
    kp = np.asarray(kp, np.float64)
    J2 = jacobian_2d(kp, jac3, camera)
    p = project(kp, camera)
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
            D = np.stack([rot_tangent(rot[j], a) for a in range(3)], 1)      # (9, 3)
            res = (rot[j] - anchor[j]).reshape(9)
            for e in range(9):
                row = np.zeros(P)
                row[3 * j:3 * j + 3] = D[e]
                wj = hw * row
                A += np.outer(wj, row)
                g += wj * res[e]
    if betas_w > 0.0:
        o = 3 * np.asarray(rot).shape[0] if rot is not None else P - 3 - len(betas)
        g[o:o + len(betas)] += float(np.float32(betas_w)) * np.asarray(betas, np.float64)
    return A, g, dg


def _solve(A, g):
    """The kernel's right-looking Cholesky and triangular solves of A delta = -g; (delta, ok)."""
    P = len(g)
    ok = True
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
    return y, ok


def lm_keypoints_2d_step(state, targets, weights, lambda_up, lambda_down, first, trial, trial_kp, trial_jac,
                         sigma=math.inf, anchor=None, pose_w=0.0, betas_w=0.0, dtype=np.float32):
    """One step for one body.  state: {'rot' (n_rot, 3, 3), 'betas', 'camera', 'keypoints' (K, 3), 'jac' (3K, P),
    'loss', 'lambda', 'accepted'} (not modified); trial: {'rot', 'betas', 'camera'}.  Returns (new state, next trial,
    accepted flag).  dtype: the storage precision (float32 as on the device; float64 gives a plain fp64 LM)."""
    f = dtype
    lt = loss(targets, weights, trial_kp, trial['camera'], sigma, trial['rot'], anchor, pose_w, trial['betas'],
              betas_w)
    lcur = state.get('loss', f(np.nan))
    accept = bool(first) or (math.isfinite(lt) and lt < float(lcur))
    new = {k: np.array(v, copy=True) if isinstance(v, np.ndarray) else v for k, v in state.items()}
    lnew = lcur
    if accept:
        lnew = f(lt) if math.isfinite(lt) else f(np.nan)
        new.update({k: np.asarray(trial[k], f).copy() for k in ('rot', 'betas', 'camera')})
        new.update(keypoints=np.asarray(trial_kp, f).copy(), jac=np.asarray(trial_jac, f).copy(), loss=lnew)
    A, g, dg = normal_equations(targets, weights, new['keypoints'], new['jac'], new['camera'], sigma, new['rot'],
                                anchor, pose_w, new['betas'], betas_w)
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
    y, ok = _solve(A, g)
    ok = ok and math.isfinite(float(lnew))
    if not ok:
        nxt = {k: np.asarray(new[k], f).copy() for k in ('rot', 'betas', 'camera')}
    else:
        nxt = {'rot': np.stack([exp_gram_schmidt(new['rot'][j], y[3 * j:3 * j + 3]) for j in range(n_rot)]).astype(f),
               'betas': np.array([f(float(new['betas'][i]) + y[o + i]) for i in range(nb)], f),
               'camera': np.array([f(float(new['camera'][i]) + y[o + nb + i]) for i in range(3)], f)}
    return new, nxt, accept
