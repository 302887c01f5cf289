"""NumPy float64 restatement of the keypoint Jacobian and of the keypoint Levenberg-Marquardt step (test
infrastructure).

  keypoint_jacobian    shapy_smplx_keypoint_jacobian for one body: the closed form of DESIGN.md §6b in float64,
                       columns [delta_j (R_j Exp(delta_j) at delta = 0) | betas | transl]
  lm_keypoints_step    shapy_fit_lm_keypoints_step for one body: the same fp64 operations in the same order (the
                       kernel is compiled with -fmad=false), so accept / reject, lambda and the loss agree bit for bit
                       with float32 storage, and the next trial to the last bits of the fp64 solve and of sin / cos
"""
import math

import numpy as np
import torch

from oracle import smplx_oracle

LAMBDA_MIN, LAMBDA_MAX = np.float32(1e-9), np.float32(1e9)
LAMBDA_INIT, DIAG_FLOOR = 1e-3, 1e-6


def _np(t, dtype=np.float64):
    return np.asarray(t.detach().cpu().numpy() if torch.is_tensor(t) else t, dtype)


def _opt(model, name):
    t = model.get(name)
    return None if t is None or (torch.is_tensor(t) and t.numel() == 0) else t


def _cross(w, q):
    return np.cross(np.broadcast_to(w, q.shape), q)


def keypoint_jacobian(model, betas, rot, transl=None, use_face_contour=True):
    """One body: betas (NB,), rot (n_rot, 3, 3), transl (3,) or None -> (keypoints (K, 3), jac (3K, P)) float64."""
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


def loss(targets, weights, kp):
    """The kernel's loss in fp64: w_k ((dx^2 + dy^2) + dz^2) summed in k order, weight <= 0 skipped."""
    L = 0.0
    for k in range(len(weights)):
        w = float(weights[k])
        if w > 0.0:
            r = [float(kp[k, c]) - float(targets[k, c]) for c in range(3)]
            L += w * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2])
    return L


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


def lm_keypoints_step(state, targets, weights, lambda_up, lambda_down, first, trial, trial_kp, trial_jac,
                      dtype=np.float32):
    """One step for one body.  state: {'rot' (n_rot, 3, 3), 'betas', 'transl', 'keypoints' (K, 3), 'jac' (3K, P),
    'loss', 'lambda', 'accepted'} (not modified); trial: {'rot', 'betas', 'transl'}.  Returns (new state, next trial,
    accepted flag).  dtype: the storage precision (float32 as on the device; float64 gives a plain fp64 LM)."""
    f = dtype
    lt = loss(targets, weights, trial_kp)
    lcur = state.get('loss', f(np.nan))
    accept = bool(first) or (math.isfinite(lt) and lt < float(lcur))
    new = {k: np.array(v, copy=True) if isinstance(v, np.ndarray) else v for k, v in state.items()}
    lnew = lcur
    if accept:
        lnew = f(lt) if math.isfinite(lt) else f(np.nan)
        new.update({k: np.asarray(trial[k], f).copy() for k in ('rot', 'betas', 'transl')})
        new.update(keypoints=np.asarray(trial_kp, f).copy(), jac=np.asarray(trial_jac, f).copy(), loss=lnew)
    Jm = np.asarray(new['jac'], np.float64)
    M = np.asarray(new['keypoints'], np.float64).reshape(-1)
    tg = np.asarray(targets, np.float64).reshape(-1)
    P = Jm.shape[1]
    A, g = np.zeros((P, P)), np.zeros(P)
    for r in range(Jm.shape[0]):
        w = float(weights[r // 3])
        if not w > 0.0:
            continue
        wj = w * Jm[r]
        A += np.outer(wj, Jm[r])
        g += wj * (M[r] - tg[r])
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
    for j in range(P):
        A[j, j] += float(lam)
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
    n_rot = new['rot'].shape[0]
    nb = len(new['betas'])
    if not ok:
        nxt = {k: np.asarray(new[k], f).copy() for k in ('rot', 'betas', 'transl')}
    else:
        nxt = {'rot': np.stack([exp_gram_schmidt(new['rot'][j], y[3 * j:3 * j + 3]) for j in range(n_rot)]).astype(f),
               'betas': np.array([f(float(new['betas'][i]) + y[3 * n_rot + i]) for i in range(nb)], f),
               'transl': np.array([f(float(new['transl'][i]) + y[3 * n_rot + nb + i]) for i in range(3)], f)}
    return new, nxt, accept
