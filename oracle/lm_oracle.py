"""TEST INFRASTRUCTURE ONLY -- NumPy restatement of the batched Levenberg-Marquardt fit of betas to measurements, and
the LM bookkeeping every step oracle shares, named after its fit.cu counterpart.

  lm_accept, lm_loss   the accept decision (the first step, or a finite trial loss below the state's) and the loss kept
                       after it (NaN for a non-finite accepted loss)
  lm_diag_max          the largest of a diagonal floored at DIAG_FLOOR, which sets the first lambda
  lm_lambda            the next lambda: LAMBDA_INIT dmax on the first step, over `down` after an accept, times `up` after
                       a reject, clamped to [LAMBDA_MIN, LAMBDA_MAX]; the caller supplies dmax, since the steps read
                       different diagonals for it
  lm_sq_norm           |x|^2 in fp64, in index order: every betas, expression and prior sum
  meas_loss            the five-measurement data term sum_{w_k > 0} w_k (t_k - m_k)^2 in k order
  meas_rows            the five measurement rows, added into the betas block of A and g in k order
  cholesky_solve       the kernels' dense right-looking Cholesky of A and the triangular solves of A delta = -g, on the
                       leading n columns (all by default)
  exp_gram_schmidt     R Exp(d), re-orthonormalised as the 6D decoder does
  lm_rot_next, lm_add_next, lm_kp_next_trial
                       the next trial: R Exp(delta) per rotation, x + delta for the additive blocks, all rounded to the
                       storage precision; a copy of the state when the step failed
  lm_step              shapy_fit_lm_step (shapy_b200/csrc/fit.cu), one body: the same fp64 operations in the same order
                       (the kernel is compiled with -fmad=false), so the accept decisions, lambda and the loss agree bit
                       for bit with float32 storage, and the next trial to the last bits of the fp64 solve
  jacobian_betas       shapy_measure_jacobian_betas: rows S^T . (measure_grad_oracle.measure_grad with cotangent e_k),
                       contracted in float64
"""
import math

import numpy as np

from oracle import measure_grad_oracle

LAMBDA_MIN, LAMBDA_MAX = np.float32(1e-9), np.float32(1e9)
LAMBDA_INIT, DIAG_FLOOR = 1e-3, 1e-6


def lm_accept(first, lt, lcur):
    return bool(first) or (math.isfinite(lt) and lt < float(lcur))


def lm_loss(accept, lt, lcur, f=np.float32):
    if not accept:
        return lcur
    return f(lt) if math.isfinite(lt) else f(np.nan)


def lm_diag_max(d, dmax=DIAG_FLOOR):
    for x in d:
        dmax = float(np.fmax(dmax, x))
    return dmax


def lm_lambda(first, accept, lam, dmax, up, down, f=np.float32):
    """lam: the state's lambda (unread on the first step); dmax: the first step's diagonal maximum (lm_diag_max)."""
    if first:
        lam = f(LAMBDA_INIT * dmax)
    elif accept:
        lam = f(f(lam) / f(down))
    else:
        lam = f(f(lam) * f(up))
    return f(np.fmin(np.fmax(lam, f(LAMBDA_MIN)), f(LAMBDA_MAX)))


def lm_sq_norm(x):
    s = 0.0
    for v in np.asarray(x, np.float64).reshape(-1):
        s += v * v
    return s


def meas_loss(targets, weights, meas):
    """sum_{w_k > 0} w_k (t_k - m_k)^2 in k order, fp64 (lm_step_kernel's data term)."""
    L = 0.0
    for k in range(5):
        w = float(weights[k])
        if w > 0.0:
            r = float(targets[k]) - float(meas[k])
            L += w * r * r
    return L


def meas_rows(A, g, o, targets, weights, meas, meas_jac):
    """The rows w_m J_m^T J_m and w_m J_m^T (m_m - t_m) added in place to A[o:o+nb, o:o+nb] and g[o:o+nb], m order;
    a dropped measurement's value and row are never read."""
    Jm = np.asarray(meas_jac, np.float64)
    nb = Jm.shape[1]
    for m in range(5):
        u = float(weights[m])
        if not u > 0.0:
            continue
        uj = u * Jm[m]
        A[o:o + nb, o:o + nb] += np.outer(uj, Jm[m])
        g[o:o + nb] += uj * (float(meas[m]) - float(targets[m]))


def cholesky_solve(A, g, n=None):
    """lm_kp_solve: the right-looking Cholesky of A's leading n columns in place (the trailing block becomes their Schur
    complement), L z = -g over those columns (the trailing entries of g lose their share), then L^T delta = z.  Returns
    (y, ok): y[:n] the solution, y[n:] the trailing right-hand side; ok when every pivot is positive and finite."""
    n = len(g) if n is None else n
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
    return y, ok


def exp_gram_schmidt(Rs, d):
    """R Exp(d) by Rodrigues in fp64, re-orthonormalised by the 6D decoder's Gram-Schmidt of the first two columns."""
    d = [float(x) for x in d]
    th2 = d[0] * d[0] + d[1] * d[1] + d[2] * d[2]
    th = math.sqrt(th2)
    if th < 1e-8:
        s, c = 1.0 - th2 / 6.0, 0.5 - th2 / 24.0
    else:
        s, c = math.sin(th) / th, (1.0 - math.cos(th)) / th2
    Kx = np.array([[0.0, -d[2], d[1]], [d[2], 0.0, -d[0]], [-d[1], d[0], 0.0]])
    E = np.eye(3) + s * Kx + c * (np.outer(d, d) - th2 * np.eye(3))
    M = np.asarray(Rs, np.float64) @ E
    a, b = M[:, 0], M[:, 1]
    b1 = a / max(math.sqrt(a @ a), 1e-12)
    u = b - (b1 @ b) * b1
    b2 = u / max(math.sqrt(u @ u), 1e-12)
    return np.stack([b1, b2, np.cross(b1, b2)], 1)


def lm_rot_next(rot, d, ok, f=np.float32):
    """rot (n, 3, 3): R_j Exp(d[3j:3j+3]) for each j, or a copy of rot when the step failed."""
    if not ok:
        return np.asarray(rot, f).copy()
    return np.stack([exp_gram_schmidt(rot[j], d[3 * j:3 * j + 3]) for j in range(len(rot))]).astype(f)


def lm_add_next(x, d, ok, f=np.float32):
    """x + d entry by entry, rounded to f, or a copy of x when the step failed."""
    if not ok:
        return np.asarray(x, f).copy()
    return np.array([f(float(x[i]) + d[i]) for i in range(len(x))], f)


def lm_kp_next_trial(state, y, ok, keys, f=np.float32):
    """The next trial from the state and delta y, whose blocks follow keys: the rotations keys[0], then the additive
    blocks in order."""
    nxt = {keys[0]: lm_rot_next(state[keys[0]], y, ok, f)}
    o = 3 * len(state[keys[0]])
    for k in keys[1:]:
        n = len(state[k])
        nxt[k] = lm_add_next(state[k], y[o:o + n], ok, f)
        o += n
    return nxt


def jacobian_betas(v, faces, S, lm=None):
    """(5, NB) float64 Jacobian of (mass, height, chest, waist, hips) with respect to betas at the vertices v (V, 3),
    S the shape basis (V, 3, NB), with the measurement backward's semantics."""
    S = np.asarray(S, np.float64)
    rows = []
    for k in range(5):
        g = measure_grad_oracle.measure_grad(np.asarray(v, np.float32), faces, np.eye(5)[k], lm)
        rows.append(np.einsum('vc,vcl->l', g, S))
    return np.stack(rows)


def loss(targets, weights, betas_weight, meas, betas):
    """The kernel's loss in fp64: the weighted data terms in k order (weight 0 skipped), then rho |beta|^2."""
    return meas_loss(targets, weights, meas) + float(betas_weight) * lm_sq_norm(betas)


def lm_step(state, targets, weights, betas_weight, lambda_up, lambda_down, first, trial, trial_meas, trial_jac,
            dtype=np.float32):
    """One step for one body.  state: {'betas' (NB,), 'meas' (5,), 'jac' (5, NB), 'loss', 'lambda', 'accepted'}
    (not modified).  Returns (new state, next trial, accepted flag).  dtype: the storage precision (float32 as on the
    device; float64 gives a plain fp64 LM)."""
    f = dtype
    rho = float(f(betas_weight))
    nb = len(trial)
    lt = loss(targets, weights, rho, trial_meas, trial)
    lcur = state.get('loss', f(np.nan))
    accept = lm_accept(first, lt, lcur)
    new = {k: np.array(v, copy=True) if isinstance(v, np.ndarray) else v for k, v in state.items()}
    lnew = lm_loss(accept, lt, lcur, f)
    if accept:
        new.update(betas=np.asarray(trial, f).copy(), meas=np.asarray(trial_meas, f).copy(),
                   jac=np.asarray(trial_jac, f).copy(), loss=lnew)
    A, g = np.zeros((nb, nb)), np.zeros(nb)
    meas_rows(A, g, 0, targets, weights, new['meas'], new['jac'])
    beta = new['betas']
    for i in range(nb):
        g[i] += rho * float(beta[i])
    lam = lm_lambda(first, accept, state.get('lambda'), lm_diag_max(np.diag(A)) if first else None, lambda_up,
                    lambda_down, f)
    new['lambda'] = lam
    new['accepted'] = int(state.get('accepted', 0)) + (1 if accept and not first else 0)
    damp = rho + float(lam)
    for i in range(nb):
        A[i, i] += damp
    y, ok = cholesky_solve(A, g)
    ok = ok and math.isfinite(float(lnew))
    return new, lm_add_next(beta, y, ok, f), accept
