"""NumPy float64 restatement of the keypoint Jacobian and of the keypoint Levenberg-Marquardt step (test
infrastructure).

  keypoint_jacobian    shapy_smplx_keypoint_jacobian for one body: the closed form of DESIGN.md §6b in float64,
                       columns [delta_j (R_j Exp(delta_j) at delta = 0) | betas | transl]; with expr,
                       shapy_smplx_keypoint_jacobian_expr: the expression rows appended to the shape basis (they are
                       shape rows NB .. NC-1), columns [delta_j | betas | expression | transl]
  loss                 the kernel's loss in fp64: the keypoint term, then with measurements their sum and rho |betas|^2
  lm_keypoints_step    shapy_fit_lm_keypoints_step (and with `meas` shapy_fit_lm_keypoints_measurements_step) for one
                       body: the same fp64 operations in the same order (the kernel is compiled with -fmad=false), so
                       accept / reject, lambda and the loss agree bit for bit with float32 storage, and the next trial
                       to the last bits of the fp64 solve and of sin / cos
"""
import math

import numpy as np
import torch

from oracle import smplx_oracle
from oracle.lm_oracle import (DIAG_FLOOR, LAMBDA_INIT, LAMBDA_MAX, LAMBDA_MIN, cholesky_solve,  # noqa: F401
                              exp_gram_schmidt, lm_accept, lm_diag_max, lm_kp_next_trial, lm_lambda, lm_loss,
                              lm_sq_norm, meas_loss, meas_rows)


def _np(t, dtype=np.float64):
    return np.asarray(t.detach().cpu().numpy() if torch.is_tensor(t) else t, dtype)


def _opt(model, name):
    t = model.get(name)
    return None if t is None or (torch.is_tensor(t) and t.numel() == 0) else t


def _cross(w, q):
    return np.cross(np.broadcast_to(w, q.shape), q)


def keypoint_jacobian(model, betas, rot, transl=None, use_face_contour=True, expr=None):
    """One body: betas (NB,), rot (n_rot, 3, 3), transl (3,) or None, expr (NE,) or None -> (keypoints (K, 3), jac
    (3K, P)) float64."""
    if expr is not None:
        model = dict(model)
        model['shapedirs'] = torch.cat([torch.as_tensor(model['shapedirs']), torch.as_tensor(model['expr_dirs'])], 2)
        betas = np.concatenate([np.asarray(betas, np.float64), np.asarray(expr, np.float64)])
    vt, S, Pd = _np(model['v_template']), _np(model['shapedirs']), _np(model['posedirs'])
    Jreg, W = _np(model['J_regressor']), _np(model['lbs_weights'])
    parents = _np(model['parents'], np.int64)
    rot = _np(rot)
    beta = _np(betas)
    J, V, NB, n_rot = Jreg.shape[0], vt.shape[0], S.shape[2], rot.shape[0]
    P = 3 * n_rot + NB + 3
    R = np.tile(np.eye(3), (J, 1, 1))
    R[:n_rot] = rot
    vs = vt + S @ beta
    Jr = Jreg @ vs
    dJ = np.einsum('jv,vcl->jcl', Jreg, S)
    GR, Gt, dGt = np.zeros((J, 3, 3)), np.zeros((J, 3)), np.zeros((J, 3, NB))
    anc = [set() for _ in range(J)]                       # ancestors including the joint itself
    GR[0], Gt[0], dGt[0], anc[0] = R[0], Jr[0], dJ[0], {0}
    for j in range(1, J):
        p = int(parents[j])
        GR[j] = GR[p] @ R[j]
        Gt[j] = GR[p] @ (Jr[j] - Jr[p]) + Gt[p]
        dGt[j] = GR[p] @ (dJ[j] - dJ[p]) + dGt[p]
        anc[j] = anc[p] | {j}
    pf = (R[1:] - np.eye(3)).reshape(-1)
    vp = vs + (pf @ Pd).reshape(V, 3)

    def vertex_rows(idx):
        """(x (n, 3), jac (n, 3, P)) of the posed vertices idx."""
        n = len(idx)
        Wv = W[idx]
        M = np.einsum('ns,sab->nab', Wv, GR)
        y = np.einsum('sab,nsb->nsa', GR, vp[idx][:, None, :] - Jr[None]) + Gt[None]
        x = np.einsum('ns,nsa->na', Wv, y)
        jac = np.zeros((n, 3, P))
        for j in range(n_rot):
            mask = np.array([j in anc[s] for s in range(J)], np.float64)
            q = np.einsum('ns,nsa->na', Wv * mask, y) - (Wv * mask).sum(1)[:, None] * Gt[j]
            for a in range(3):
                d = _cross(GR[j][:, a], q)
                if j >= 1:
                    e = np.zeros(3)
                    e[a] = 1.0
                    D = np.stack([R[j] @ np.cross(e, np.eye(3)[c]) for c in range(3)], 1)    # R_j [e_a]x
                    Pj = Pd[9 * (j - 1):9 * j].reshape(9, V, 3)[:, idx, :]
                    d = d + np.einsum('nrc,nc->nr', M, np.einsum('e,enc->nc', D.reshape(9), Pj))
                jac[:, :, 3 * j + a] = d
        jac[:, :, 3 * n_rot:3 * n_rot + NB] = (np.einsum('nrc,ncl->nrl', M, S[idx]) +
                                               np.einsum('ns,scl->ncl', Wv, dGt - np.einsum('sab,sbl->sal', GR, dJ)))
        jac[:, :, 3 * n_rot + NB:] = np.eye(3)
        return x, jac

    def mix(idx, w):
        x, jac = vertex_rows(np.asarray(idx, np.int64))
        w = np.asarray(w, np.float64)
        return np.einsum('n,na->a', w, x), np.einsum('n,nap->ap', w, jac)

    kp, rows = [], []
    for k in range(J):
        jk = np.zeros((3, P))
        for j in range(n_rot):
            if j != k and j in anc[k]:
                for a in range(3):
                    jk[:, 3 * j + a] = np.cross(GR[j][:, a], Gt[k] - Gt[j])
        jk[:, 3 * n_rot:3 * n_rot + NB] = dGt[k]
        jk[:, 3 * n_rot + NB:] = np.eye(3)
        kp.append(Gt[k])
        rows.append(jk)
    faces = _np(model['faces_tensor'], np.int64)
    lmk = []
    if _opt(model, 'lmk_faces_idx') is not None:
        lmk += list(zip(faces[_np(model['lmk_faces_idx'], np.int64)], _np(model['lmk_bary_coords'])))
    if use_face_contour and _opt(model, 'dynamic_lmk_faces_idx') is not None:
        full = torch.from_numpy(R[None]).float()
        df, db = smplx_oracle.dynamic_landmarks(full, model['dynamic_lmk_faces_idx'],
                                                model['dynamic_lmk_bary_coords'].float(), model['neck_kin_chain'])
        lmk += list(zip(faces[_np(df[0], np.int64)], _np(db[0])))
    for vi, bc in lmk:
        x, jk = mix(vi, bc)
        kp.append(x)
        rows.append(jk)
    if _opt(model, 'extra_joint_regressor') is not None:
        reg = _np(model['extra_joint_regressor'])
        src, tgt = _np(model['source_idxs'], np.int64), _np(model['target_idxs'], np.int64)
        for s, t in zip(src, tgt):
            nz = np.nonzero(reg[t])[0]
            kp[s], rows[s] = mix(nz, reg[t, nz])
    kp = np.stack(kp)
    if transl is not None:
        kp = kp + _np(transl)
    return kp, np.concatenate(rows, 0)


def loss(targets, weights, kp, meas=None, betas=None, betas_weight=0.0):
    """The kernel's loss in fp64: w_k ((dx^2 + dy^2) + dz^2) summed in k order, weight <= 0 skipped; with meas
    (meas_targets, meas_weights, meas) the measurement sum and rho |betas|^2 follow, left to right, rho (float32) <= 0
    adding nothing."""
    L = 0.0
    for k in range(len(weights)):
        w = float(weights[k])
        if w > 0.0:
            r = [float(kp[k, c]) - float(targets[k, c]) for c in range(3)]
            L += w * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2])
    if meas is not None:
        L += meas_loss(*meas)
    rho = float(np.float32(betas_weight))
    if rho > 0.0:
        L += rho * lm_sq_norm(betas)
    return L


def lm_keypoints_step(state, targets, weights, lambda_up, lambda_down, first, trial, trial_kp, trial_jac, meas=None,
                      trial_meas=None, betas_weight=0.0, dtype=np.float32, return_delta=False):
    """One step for one body.  state: {'rot' (n_rot, 3, 3), 'betas', 'transl', 'keypoints' (K, 3), 'jac' (3K, P),
    'loss', 'lambda', 'accepted'}, with meas also 'meas' (5,) and 'meas_jac' (5, NB) (not modified); trial: {'rot',
    'betas', 'transl'}; meas None or (meas_targets, meas_weights), trial_meas (meas (5,), meas_jac (5, NB)) of the
    trial.  The measurement rows and the betas regulariser are stacked under the keypoint rows, and the first lambda
    reads the diagonal after them.  Returns (new state, next trial, accepted flag), and with return_delta the solved
    step delta (P,) as a fourth item.  dtype: the storage precision (float32 as on the device; float64 gives a plain
    fp64 LM)."""
    f = dtype
    rho = float(np.float32(betas_weight))
    lt = loss(targets, weights, trial_kp, None if meas is None else (meas[0], meas[1], trial_meas[0]), trial['betas'],
              rho)
    lcur = state.get('loss', f(np.nan))
    accept = lm_accept(first, lt, lcur)
    new = {k: np.array(v, copy=True) if isinstance(v, np.ndarray) else v for k, v in state.items()}
    lnew = lm_loss(accept, lt, lcur, f)
    if accept:
        new.update({k: np.asarray(trial[k], f).copy() for k in ('rot', 'betas', 'transl')})
        new.update(keypoints=np.asarray(trial_kp, f).copy(), jac=np.asarray(trial_jac, f).copy(), loss=lnew)
        if meas is not None:
            new.update(meas=np.asarray(trial_meas[0], f).copy(), meas_jac=np.asarray(trial_meas[1], f).copy())
    Jk = np.asarray(new['jac'], np.float64)
    M = np.asarray(new['keypoints'], np.float64).reshape(-1)
    tg = np.asarray(targets, np.float64).reshape(-1)
    P = Jk.shape[1]
    nb = len(new['betas'])
    o = 3 * new['rot'].shape[0]
    A, g = np.zeros((P, P)), np.zeros(P)
    # keypoint rows in keypoint-major xyz order, then the measurement rows into the betas block in k order
    for r in range(Jk.shape[0]):
        w = float(weights[r // 3])
        if not w > 0.0:
            continue
        wj = w * Jk[r]
        A += np.outer(wj, Jk[r])
        g += wj * (M[r] - tg[r])
    if meas is not None:
        meas_rows(A, g, o, meas[0], meas[1], new['meas'], new['meas_jac'])
    if rho > 0.0:
        g[o:o + nb] += rho * np.asarray(new['betas'], np.float64)
    lam = lm_lambda(first, accept, state.get('lambda'), lm_diag_max(np.diag(A)) if first else None, lambda_up,
                    lambda_down, f)
    new['lambda'] = lam
    new['accepted'] = int(state.get('accepted', 0)) + (1 if accept and not first else 0)
    damp = rho + float(lam)
    for j in range(P):
        A[j, j] += damp if o <= j < o + nb else float(lam)
    y, ok = cholesky_solve(A, g)
    ok = ok and math.isfinite(float(lnew))
    nxt = lm_kp_next_trial(new, y, ok, ('rot', 'betas', 'transl'), f)
    return (new, nxt, accept, y) if return_delta else (new, nxt, accept)
