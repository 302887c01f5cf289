"""TEST INFRASTRUCTURE ONLY -- NumPy restatement of the batched Levenberg-Marquardt fit of betas to measurements.

  lm_step          shapy_fit_lm_step (shapy_b200/csrc/fit.cu), one body: the same fp64 operations in the same order
                   (the kernel is compiled with -fmad=false), so the accept decisions, lambda and the loss agree bit for
                   bit with float32 storage, and the next trial to the last bits of the fp64 solve
  jacobian_betas   shapy_measure_jacobian_betas: rows S^T . (measure_grad_oracle.measure_grad with cotangent e_k),
                   contracted in float64
"""
import math

import numpy as np

from oracle import measure_grad_oracle

LAMBDA_MIN, LAMBDA_MAX = np.float32(1e-9), np.float32(1e9)
LAMBDA_INIT, DIAG_FLOOR = 1e-3, 1e-6


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
    data = 0.0
    for k in range(5):
        w = float(weights[k])
        if w > 0.0:
            r = float(targets[k]) - float(meas[k])
            data += w * r * r
    reg = 0.0
    for x in betas:
        reg += float(x) * float(x)
    return data + float(betas_weight) * reg


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
    accept = bool(first) or (math.isfinite(lt) and lt < float(lcur))
    new = {k: np.array(v, copy=True) if isinstance(v, np.ndarray) else v for k, v in state.items()}
    lnew = lcur
    if accept:
        lnew = f(lt) if math.isfinite(lt) else f(np.nan)
        new.update(betas=np.asarray(trial, f).copy(), meas=np.asarray(trial_meas, f).copy(),
                   jac=np.asarray(trial_jac, f).copy(), loss=lnew)
    J, M, beta = new['jac'], new['meas'], new['betas']
    A = np.zeros((nb, nb))
    g = np.zeros(nb)
    for k in range(5):
        w = float(weights[k])
        if not w > 0.0:
            continue
        r = float(M[k]) - float(targets[k])
        for i in range(nb):
            wi = w * float(J[k, i])
            for j in range(nb):
                A[i, j] += wi * float(J[k, j])
            g[i] += wi * r
    for i in range(nb):
        g[i] += rho * float(beta[i])
    if first:
        dmax = DIAG_FLOOR
        for j in range(nb):
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
    for i in range(nb):
        A[i, i] += damp
    ok = math.isfinite(float(lnew))
    with np.errstate(invalid='ignore', divide='ignore'):
        for j in range(nb):          # right-looking Cholesky, as the kernel's lanes do it
            d = A[j, j]
            ok = ok and d > 0.0 and math.isfinite(d)
            ljj = math.sqrt(d) if d >= 0 else float('nan')
            for i in range(j + 1, nb):
                A[i, j] /= ljj
            A[j, j] = ljj
            for k in range(j + 1, nb):
                for i in range(k, nb):
                    A[i, k] -= A[i, j] * A[k, j]
        y = -g.copy()
        for j in range(nb):
            y[j] = y[j] / A[j, j]
            for i in range(j + 1, nb):
                y[i] -= A[i, j] * y[j]
        for j in range(nb - 1, -1, -1):
            y[j] = y[j] / A[j, j]
            for i in range(j):
                y[i] -= A[j, i] * y[j]
    nxt = np.array([f(float(beta[i]) + y[i]) for i in range(nb)], f) if ok else np.asarray(beta, f).copy()
    return new, nxt, accept
