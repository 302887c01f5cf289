"""NumPy float64 restatement of the vertex Jacobian and of the scan Levenberg-Marquardt step (test infrastructure).

  vertex_jacobian   shapy_smplx_vertex_jacobian for one body: the closed form of kp_lm_oracle.keypoint_jacobian over
                    every vertex, columns [delta_j | betas | transl]
  rows              the rows of one trial at its held correspondences: the chunk partial sums of J^T U J, J^T U r and
                    the loss share, in the kernel's order (chunks of CHUNK points, then of CHUNK vertices)
  lm_scan_step      shapy_fit_lm_scan_step for one body: the chunks summed in chunk order, the policy of
                    kp_lm_oracle.lm_keypoints_step, the prior and measurement rows at the state
"""
import math

import numpy as np

from oracle.lm_oracle import (cholesky_solve, lm_accept, lm_diag_max, lm_kp_next_trial, lm_lambda, lm_loss,
                              lm_sq_norm, meas_loss, meas_rows)

CHUNK = 1024           # kScanChunk of fit.cu
THREADS = 256          # the step kernel's threads: sum_{w > 0} w is strided over them


def _np(t):
    return np.asarray(t.detach().cpu().numpy() if hasattr(t, 'detach') else t, np.float64)


def vertex_jacobian(model, betas, rot, transl=None):
    """One body: betas (NB,), rot (n_rot, 3, 3), transl (3,) or None -> (vertices (V, 3), jac (V, 3, P)) float64."""
    vt, S, Pd = _np(model['v_template']), _np(model['shapedirs']), _np(model['posedirs'])
    Jreg, W = _np(model['J_regressor']), _np(model['lbs_weights'])
    parents = np.asarray(_np(model['parents']), np.int64)
    rot, beta = _np(rot), _np(betas)
    J, V, NB, n_rot = Jreg.shape[0], vt.shape[0], S.shape[2], rot.shape[0]
    P = 3 * n_rot + NB + 3
    R = np.tile(np.eye(3), (J, 1, 1))
    R[:n_rot] = rot
    vs = vt + S @ beta
    Jr = Jreg @ vs
    dJ = np.einsum('jv,vcl->jcl', Jreg, S)
    GR, Gt, dGt = np.zeros((J, 3, 3)), np.zeros((J, 3)), np.zeros((J, 3, NB))
    anc = np.zeros((J, J), bool)                  # anc[s, j]: j is s or one of its ancestors
    GR[0], Gt[0], dGt[0], anc[0, 0] = R[0], Jr[0], dJ[0], True
    for j in range(1, J):
        p = int(parents[j])
        GR[j] = GR[p] @ R[j]
        Gt[j] = GR[p] @ (Jr[j] - Jr[p]) + Gt[p]
        dGt[j] = GR[p] @ (dJ[j] - dJ[p]) + dGt[p]
        anc[j] = anc[p]
        anc[j, j] = True
    pf = (R[1:] - np.eye(3)).reshape(-1)
    vp = vs + (pf @ Pd).reshape(V, 3)
    M = np.einsum('vs,sab->vab', W, GR)
    y = np.einsum('sab,vsb->vsa', GR, vp[:, None, :] - Jr[None]) + Gt[None]
    x = np.einsum('vs,vsa->va', W, y)
    jac = np.zeros((V, 3, P))
    Pd9 = Pd.reshape(-1, 9, V, 3) if Pd.shape[0] else None
    for j in range(n_rot):
        Wm = W * anc[:, j][None]
        q = np.einsum('vs,vsa->va', Wm, y) - Wm.sum(1)[:, None] * Gt[j]
        for a in range(3):
            d = np.cross(np.broadcast_to(GR[j][:, a], q.shape), q)
            if j >= 1:
                e = np.zeros(3)
                e[a] = 1.0
                D = np.stack([R[j] @ np.cross(e, np.eye(3)[c]) for c in range(3)], 1)    # R_j [e_a]x
                d = d + np.einsum('vrc,vc->vr', M, np.einsum('e,evc->vc', D.reshape(9), Pd9[j - 1]))
            jac[:, :, 3 * j + a] = d
    jac[:, :, 3 * n_rot:3 * n_rot + NB] = (np.einsum('vrc,vcl->vrl', M, S) +
                                           np.einsum('vs,scl->vcl', W, dGt - np.einsum('sab,sbl->sal', GR, dJ)))
    jac[:, :, 3 * n_rot + NB:] = np.eye(3)
    if transl is not None:
        x = x + _np(transl)
    return x, jac


def _rho(sigma, e):
    """(rho(e), rho'(e)) in the kernel's operations: Geman-McClure at sigma, least squares at sigma = inf."""
    if math.isinf(sigma):
        return e, 1.0
    s2 = float(np.float32(sigma)) ** 2
    q = s2 / (s2 + e)
    return e * q, q * q


def rows(verts, jac, points, weights, faces, face_idx, bary, nearest, sigma, P):
    """The chunk partial sums of one body's trial: a list of (A (P, P) lower triangle, g (P,), loss), the point chunks
    then the vertex chunks (nearest None: no vertex rows), each row accumulated in row order as the kernel does."""
    verts, jac = np.asarray(verts, np.float32), np.asarray(jac, np.float32)
    N, V = len(weights), verts.shape[0]
    out = []

    def chunk(items):
        A, g, L = np.zeros((P, P)), np.zeros(P), 0.0
        for ls, rws in items:
            L += ls
            for u, r, j in rws:
                if not u > 0.0:
                    continue
                uj = u * j
                A += np.outer(uj, j)
                g += uj * r
        return np.tril(A), g, L

    def point(i):
        w = float(weights[i])
        if not w > 0.0:
            return 0.0, []
        vi = faces[int(face_idx[i])]
        b = [float(x) for x in bary[i]]
        X = [verts[int(v)].astype(np.float64) for v in vi]
        p = np.asarray(points[i], np.float64)
        d = np.array([b[0] * X[0][q] + b[1] * X[1][q] + b[2] * X[2][q] - p[q] for q in range(3)])
        rho, drho = _rho(sigma, d[0] * d[0] + d[1] * d[1] + d[2] * d[2])
        u = w * drho
        e1, e2 = X[1] - X[0], X[2] - X[0]
        nv = np.array([e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0]])
        nn = math.sqrt(nv[0] * nv[0] + nv[1] * nv[1] + nv[2] * nv[2])
        Jv = [jac[int(v)].astype(np.float64) for v in vi]
        mix = [b[0] * Jv[0][q] + b[1] * Jv[1][q] + b[2] * Jv[2][q] for q in range(3)]
        if b[0] > 0 and b[1] > 0 and b[2] > 0 and nn > 0:
            n = nv / nn
            return w * rho, [(u, n[0] * d[0] + n[1] * d[1] + n[2] * d[2], n[0] * mix[0] + n[1] * mix[1] + n[2] * mix[2])]
        return w * rho, [(u, d[q], mix[q]) for q in range(3)]

    def vertex(v):
        q = int(nearest[v])
        if q < 0:
            return 0.0, []
        d = verts[v].astype(np.float64) - np.asarray(points[q], np.float64)
        rho, drho = _rho(sigma, d[0] * d[0] + d[1] * d[1] + d[2] * d[2])
        return rho, [(drho, d[c], jac[v, c].astype(np.float64)) for c in range(3)]

    for c0 in range(0, N, CHUNK):
        out.append(chunk([point(i) for i in range(c0, min(N, c0 + CHUNK))]))
    for c0 in range(0, V, CHUNK):
        out.append(chunk([vertex(v) for v in range(c0, min(V, c0 + CHUNK))]) if nearest is not None else
                   (np.zeros((P, P)), np.zeros(P), 0.0))
    return out


def weight_sum(weights):
    """sum_{w > 0} w as the step kernel forms it: THREADS strided partial sums, then those in thread order."""
    part = []
    for t in range(THREADS):
        s = 0.0
        for w in weights[t::THREADS]:
            if float(w) > 0.0:
                s += float(w)
        part.append(s)
    W = 0.0
    for s in part:
        W += s
    return W


def _tangent(R, a):
    """R [e_a]x as a 9-vector."""
    e = np.zeros(3)
    e[a] = 1.0
    return np.stack([R @ np.cross(e, np.eye(3)[c]) for c in range(3)], 1).reshape(9)


def lm_scan_step(state, trial, chunks, ns, weights, V, s2m, m2s, lambda_up, lambda_down, first, anchor=None,
                 pose_w=0.0, betas_w=0.0, meas=None, trial_meas=None):
    """One step for one body.  state: {'rot' (n_rot, 3, 3), 'betas', 'transl', 'A' (P, P), 'g' (P,), 'loss',
    'lambda', 'accepted'}, with meas also 'meas' and 'meas_jac'; trial {'rot', 'betas', 'transl'}; chunks: rows() of
    the trial, the first ns of them the point chunks; meas (targets, weights) and trial_meas (meas, meas_jac).  Returns
    (new state, next trial, accepted flag)."""
    f = np.float32
    W = weight_sum(weights)
    cs, cm = float(np.float32(s2m)) / (W if W > 0.0 else 1.0), float(np.float32(m2s)) / float(V)
    Ls, Lm = 0.0, 0.0
    for c, (_, _, L) in enumerate(chunks):
        if c < ns:
            Ls += L
        else:
            Lm += L
    lt = cs * Ls + cm * Lm
    pw, bw = float(np.float32(pose_w)), float(np.float32(betas_w))
    if pw > 0.0:
        q = 0.0
        for v, a in zip(np.asarray(trial['rot'], np.float64).reshape(-1)[9:], np.asarray(anchor, np.float64).reshape(-1)[9:]):
            q += (v - a) * (v - a)
        lt += 0.5 * pw * q
    if meas is not None:
        lt += meas_loss(meas[0], meas[1], trial_meas[0])
    if bw > 0.0:
        lt += bw * lm_sq_norm(trial['betas'])
    lcur = state.get('loss', f(np.nan))
    accept = lm_accept(first, lt, lcur)
    new = {k: np.array(v, copy=True) if isinstance(v, np.ndarray) else v for k, v in state.items()}
    lnew = lm_loss(accept, lt, lcur, f)
    P = chunks[0][1].shape[0]
    if accept:
        new.update({k: np.asarray(trial[k], f).copy() for k in ('rot', 'betas', 'transl')})
        new['loss'] = lnew
        As, Am, gs, gm = np.zeros((P, P)), np.zeros((P, P)), np.zeros(P), np.zeros(P)
        for c, (A, g, _) in enumerate(chunks):
            if c < ns:
                As, gs = As + A, gs + g
            else:
                Am, gm = Am + A, gm + g
        A = cs * As + cm * Am
        new['A'] = np.tril(A) + np.tril(A, -1).T
        new['g'] = cs * gs + cm * gm
        if meas is not None:
            new.update(meas=np.asarray(trial_meas[0], f).copy(), meas_jac=np.asarray(trial_meas[1], f).copy())
    A, g = np.tril(np.asarray(new['A'], np.float64)), np.asarray(new['g'], np.float64).copy()
    dg = np.diag(A).copy()
    n_rot, nb = new['rot'].shape[0], len(new['betas'])
    o = 3 * n_rot
    if pw > 0.0:
        hw = 0.5 * pw
        R = np.asarray(new['rot'], np.float64)
        for j in range(1, n_rot):
            T = [_tangent(R[j], a) for a in range(3)]
            for a in range(3):
                for c in range(a + 1):
                    s = A[3 * j + a, 3 * j + c]
                    for e in range(9):
                        s += (hw * T[a][e]) * T[c][e]
                    A[3 * j + a, 3 * j + c] = s
                s = g[3 * j + a]
                for e in range(9):
                    s += (hw * T[a][e]) * (R[j].reshape(9)[e] - float(np.asarray(anchor, np.float64)[j].reshape(9)[e]))
                g[3 * j + a] = s
    if meas is not None:
        meas_rows(A, g, o, meas[0], meas[1], new['meas'], new['meas_jac'])
    if bw > 0.0:
        g[o:o + nb] += bw * np.asarray(new['betas'], np.float64)
    lam = lm_lambda(first, accept, state.get('lambda'), lm_diag_max(dg) if first else None, lambda_up, lambda_down, f)
    new['lambda'] = lam
    new['accepted'] = int(state.get('accepted', 0)) + (1 if accept and not first else 0)
    for j in range(P):
        A[j, j] += bw + float(lam) if o <= j < o + nb else float(lam)
    A = np.tril(A) + np.tril(A, -1).T
    y, ok = cholesky_solve(A, g)
    ok = ok and math.isfinite(float(lnew))
    nxt = lm_kp_next_trial(new, y, ok, ('rot', 'betas', 'transl'), f)
    return new, nxt, accept
