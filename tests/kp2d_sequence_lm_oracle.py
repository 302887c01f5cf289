"""NumPy float64 restatement of the sequence 2D keypoint Levenberg-Marquardt step (test infrastructure), on top of
tests/kp2d_lm_oracle.py (its perspective camera) and tests/kp2dg_lm_oracle.py: the frames of one sequence share their betas, each keeps
its rotations and camera-frame translation, and consecutive frames are tied by smoothness rows, so the normal matrix
of a sequence is block tridiagonal in its frames with an arrow of betas columns.

  smooth_loss      the smoothness term of one pair of frames (t, t + 1)
  smooth_rows      the pair's rows (weights, residuals, Jacobian on the columns [frame t | frame t + 1], each
                   [delta | tau]): the pose prior's rows with the anchor replaced by the neighbour, then the translation's
  frame_scratch    launch 1 for one frame: the bracket of its trial loss and, on the first step, the max of its
                   keypoint-row diagonal over [delta | tau] and its betas entries
  frame_system     launch 2 for one frame: its normal equations in the column order [delta | tau | beta] (keypoint rows,
                   pose-prior rows, the smoothness diagonal blocks and gradient of its neighbours), before damping
  coupling         C_t, the block of frame t + 1's rows and frame t's columns
  dense_system     the whole damped normal matrix of a sequence, [x_0 | .. | x_{T-1} | beta], and its right-hand side
  sweep            the block LDL^T sweep of launch 3 (block Thomas with the arrow carried along)
  lm_sequence_step shapy_fit_lm_keypoints_2d_sequence_step for one sequence: the loss, decision and lambda in the
                   kernels' fp64 order (bit for bit with float32 storage), the step by the sweep to rounding
"""
import math

import numpy as np

import kp2d_lm_oracle as o2
import kp2dg_lm_oracle as og
from oracle.lm_oracle import exp_gram_schmidt, lm_diag_max, lm_sq_norm


def smooth_loss(rot0, rot1, t0, t1, srw=0.0, stw=0.0):
    """srot_w / 2 sum_j |R1_j - R0_j|_F^2 (j order, row-major entries) + stransl_w |t1 - t0|^2, in fp64."""
    L = 0.0
    if srw > 0.0:
        L += o2.prior_loss(rot1, rot0, srw)
    if stw > 0.0:
        L += float(np.float32(stw)) * lm_sq_norm(np.asarray(t1, np.float64) - np.asarray(t0, np.float64))
    return L


def _tangents(R):
    """(9, 3): column a is R [e_a]x as row-major entries."""
    return np.stack([o2.rot_tangent(np.asarray(R, np.float64), a) for a in range(3)], 1)


def smooth_rows(rot0, rot1, t0, t1, srw=0.0, stw=0.0):
    """(w (m,), r (m,), J (m, 2 n1)) of the pair, columns [delta_0 | tau_0 | delta_1 | tau_1]: 9 n_rot rotation rows
    (weight srw / 2, residual R1 - R0, Jacobian -R0 [e_a]x and +R1 [e_a]x), then 3 translation rows (weight stw,
    residual t1 - t0, Jacobian -I and +I)."""
    rot0, rot1 = np.asarray(rot0, np.float64), np.asarray(rot1, np.float64)
    n_rot = rot0.shape[0]
    n1 = 3 * n_rot + 3
    w, r, J = [], [], []
    for j in range(n_rot):
        D0, D1 = _tangents(rot0[j]), _tangents(rot1[j])
        res = (rot1[j] - rot0[j]).reshape(9)
        for e in range(9):
            row = np.zeros(2 * n1)
            row[3 * j:3 * j + 3] = -D0[e]
            row[n1 + 3 * j:n1 + 3 * j + 3] = D1[e]
            w.append(0.5 * float(np.float32(srw)))
            r.append(res[e])
            J.append(row)
    for c in range(3):
        row = np.zeros(2 * n1)
        row[n1 - 3 + c] = -1.0
        row[2 * n1 - 3 + c] = 1.0
        w.append(float(np.float32(stw)))
        r.append(float(t1[c]) - float(t0[c]))
        J.append(row)
    return np.array(w), np.array(r), np.array(J)


def frame_scratch(targets, weights, intr, trial_kp, trial_jac, trial, first, nxt=None, sigma=math.inf, anchor=None,
                  pose_w=0.0, srw=0.0, stw=0.0, dtype=np.float32):
    """(bracket, dmax over [delta | tau] from DIAG_FLOOR, the betas diagonal) of one frame's trial; nxt: the next
    frame's trial {'rot', 'transl'} when it is in the sequence."""
    lt = o2.loss(targets, weights, trial_kp, trial['transl'], sigma, trial['rot'], anchor, pose_w, intr=intr)
    if nxt is not None:
        lt += smooth_loss(trial['rot'], nxt['rot'], trial['transl'], nxt['transl'], srw, stw)
    if not first:
        return lt, None, None
    f = dtype
    with np.errstate(all='ignore'):
        _, _, dg = o2.normal_equations(targets, weights, np.asarray(trial_kp, f), np.asarray(trial_jac, f),
                                       np.asarray(trial['transl'], f), sigma, intr=intr)
    nb = len(trial['betas'])
    n_rot = np.asarray(trial['rot']).shape[0]
    dg = dg[og.reorder(n_rot, nb)]
    return lt, lm_diag_max(dg[:3 * n_rot + 3]), dg[3 * n_rot + 3:].copy()


def frame_system(targets, weights, intr, kp, jac, rot, transl, neighbours=(), sigma=math.inf, anchor=None, pose_w=0.0,
                 srw=0.0, stw=0.0):
    """(A, g) of one frame at its state, columns [delta | tau | beta], undamped, without the betas prior; neighbours:
    the (rot, transl) of the previous and the next frame, those in the sequence."""
    nb = np.asarray(jac).shape[1] - 3 * np.asarray(rot).shape[0] - 3
    with np.errstate(all='ignore'):
        A, g, _ = o2.normal_equations(targets, weights, kp, jac, transl, sigma, rot, anchor, pose_w, intr=intr)
    perm = og.reorder(np.asarray(rot).shape[0], nb)
    A, g = A[perm][:, perm].copy(), g[perm].copy()
    rot, transl = np.asarray(rot, np.float64), np.asarray(transl, np.float64)
    o = 3 * rot.shape[0]
    for Rn, Tn in neighbours:
        if srw > 0.0:
            hw = 0.5 * float(np.float32(srw))
            for j in range(rot.shape[0]):
                D = _tangents(rot[j])
                A[3 * j:3 * j + 3, 3 * j:3 * j + 3] += hw * D.T @ D
                g[3 * j:3 * j + 3] += hw * D.T @ (rot[j] - np.asarray(Rn, np.float64)[j]).reshape(9)
        if stw > 0.0:
            w = float(np.float32(stw))
            A[o:o + 3, o:o + 3] += w * np.eye(3)
            g[o:o + 3] += w * (transl - np.asarray(Tn, np.float64))
    return A, g


def coupling(rot0, rot1, srw=0.0, stw=0.0):
    """C_t (n1, n1): rows of frame t + 1 (rot1), columns of frame t (rot0)."""
    rot0, rot1 = np.asarray(rot0, np.float64), np.asarray(rot1, np.float64)
    n_rot = rot0.shape[0]
    n1 = 3 * n_rot + 3
    C = np.zeros((n1, n1))
    if srw > 0.0:
        hw = 0.5 * float(np.float32(srw))
        for j in range(n_rot):
            C[3 * j:3 * j + 3, 3 * j:3 * j + 3] = -hw * _tangents(rot1[j]).T @ _tangents(rot0[j])
    C[n1 - 3:, n1 - 3:] = -float(np.float32(stw)) * np.eye(3)
    return C


def _blocks(frames, st, lam, sigma, pose_w, srw, stw):
    """Per frame (A_t, g_t) with the frame block damped by lam, and the couplings C_t, at the state st."""
    T = len(frames)
    sys_, C = [], []
    for t in range(T):
        nbrs = [(st['rot'][u], st['transl'][u]) for u in (t - 1, t + 1) if 0 <= u < T]
        fr = frames[t]
        A, g = frame_system(fr['targets'], fr['weights'], fr['intr'], st['keypoints'][t], st['jac'][t], st['rot'][t],
                            st['transl'][t], nbrs, sigma, fr.get('anchor'), pose_w, srw, stw)
        n1 = 3 * np.asarray(st['rot'][t]).shape[0] + 3
        A[np.arange(n1), np.arange(n1)] += float(lam)
        sys_.append((A, g))
        if t + 1 < T:
            C.append(coupling(st['rot'][t], st['rot'][t + 1], srw, stw))
    return sys_, C


def dense_system(frames, st, lam, sigma=math.inf, pose_w=0.0, betas_w=0.0, srw=0.0, stw=0.0):
    """(M, rhs): the damped normal matrix of a sequence at the state st, columns [x_0 | .. | x_{T-1} | beta], and
    -g (the betas prior included)."""
    sys_, C = _blocks(frames, st, lam, sigma, pose_w, srw, stw)
    T = len(frames)
    n1 = 3 * np.asarray(st['rot'][0]).shape[0] + 3
    nb = len(st['betas'])
    N = T * n1 + nb
    M, rhs = np.zeros((N, N)), np.zeros(N)
    for t, (A, g) in enumerate(sys_):
        a = slice(t * n1, (t + 1) * n1)
        M[a, a] = np.tril(A[:n1, :n1]) + np.tril(A[:n1, :n1], -1).T
        M[T * n1:, a] = A[n1:, :n1]
        M[a, T * n1:] = A[n1:, :n1].T
        M[T * n1:, T * n1:] += np.tril(A[n1:, n1:]) + np.tril(A[n1:, n1:], -1).T
        rhs[a] = -g[:n1]
        rhs[T * n1:] -= g[n1:]
        if t + 1 < T:
            b = slice((t + 1) * n1, (t + 2) * n1)
            M[b, a] = C[t]
            M[a, b] = C[t].T
    beta = np.asarray(st['betas'], np.float64)
    M[T * n1 + np.arange(nb), T * n1 + np.arange(nb)] += float(np.float32(betas_w)) + float(lam)
    rhs[T * n1:] -= float(np.float32(betas_w)) * beta
    return M, rhs


def sweep(D, C, B, E, r, rb):
    """The block LDL^T sweep: D (T blocks n1 x n1, damped), C (T - 1 blocks, rows of frame t + 1, columns of frame t),
    B (T blocks n1 x nb), E (nb x nb, damped), right-hand sides r (T vectors n1) and rb (nb).  Returns (x (T vectors),
    dbeta, ok: every pivot positive)."""
    T = len(D)
    Et, et = np.array(E, np.float64), np.array(rb, np.float64)
    ys, Xs, Ys = [], [], []
    for t in range(T):
        Dt, Bt, rt = np.array(D[t], np.float64), np.array(B[t], np.float64), np.array(r[t], np.float64)
        if t > 0:
            Dt = Dt - C[t - 1] @ Ys[-1]
            Bt = Bt - C[t - 1] @ Xs[-1]
            rt = rt - C[t - 1] @ ys[-1]
        try:
            L = np.linalg.cholesky(Dt)
        except np.linalg.LinAlgError:
            return None, None, False
        sol = lambda b: np.linalg.solve(L.T, np.linalg.solve(L, b))  # noqa: E731
        ys.append(sol(rt))
        Xs.append(sol(Bt))
        Ys.append(sol(C[t].T) if t + 1 < T else None)
        Et = Et - Bt.T @ Xs[-1]
        et = et - Bt.T @ ys[-1]
    try:
        np.linalg.cholesky(Et)
    except np.linalg.LinAlgError:
        return None, None, False
    db = np.linalg.solve(Et, et)
    x = [None] * T
    for t in range(T - 1, -1, -1):
        v = ys[t] - Xs[t] @ db
        if t + 1 < T:
            v = v - Ys[t] @ x[t + 1]
        x[t] = v
    return x, db, True


def lm_sequence_step(state, frames, lambda_up, lambda_down, first, trial, sigma=math.inf, pose_w=0.0, betas_w=0.0,
                     srw=0.0, stw=0.0, dtype=np.float32):
    """One step for one sequence.  state: {'rot', 'transl', 'keypoints', 'jac': lists over the frames, 'betas' (nb,),
    'loss', 'lambda', 'accepted'}; frames: a list of {'targets', 'weights', 'intr', 'anchor', 'trial_kp', 'trial_jac'};
    trial: {'rot', 'transl': lists, 'betas' (nb,)}.  Returns (new state, next trial, accepted flag).  dtype: the
    storage precision (float64 gives a plain fp64 LM)."""
    f = dtype
    T = len(frames)
    nb = len(trial['betas'])
    scratch = []
    for t, fr in enumerate(frames):
        tr = {'rot': trial['rot'][t], 'transl': trial['transl'][t], 'betas': trial['betas']}
        nxt = {'rot': trial['rot'][t + 1], 'transl': trial['transl'][t + 1]} if t + 1 < T else None
        scratch.append(frame_scratch(fr['targets'], fr['weights'], fr['intr'], fr['trial_kp'], fr['trial_jac'], tr,
                                     first, nxt, sigma, fr.get('anchor'), pose_w, srw, stw, dtype))
    lcur = state.get('loss', f(np.nan))
    accept, lnew, lam = og.decide(scratch, first, lcur, state.get('lambda', 0.0), lambda_up, lambda_down,
                                  trial['betas'], betas_w, None, dtype)
    new = {k: ([np.array(x, copy=True) for x in v] if isinstance(v, list) else
               np.array(v, copy=True) if isinstance(v, np.ndarray) else v) for k, v in state.items()}
    if accept:
        for k in ('rot', 'transl'):
            new[k] = [np.asarray(x, f).copy() for x in trial[k]]
        new['keypoints'] = [np.asarray(fr['trial_kp'], f).copy() for fr in frames]
        new['jac'] = [np.asarray(fr['trial_jac'], f).copy() for fr in frames]
        new['betas'] = np.asarray(trial['betas'], f).copy()
        new['loss'] = lnew
    new['lambda'] = lam
    new['accepted'] = int(state.get('accepted', 0)) + (1 if accept and not first else 0)
    sys_, C = _blocks(frames, new, lam, sigma, pose_w, srw, stw)
    n_rot = np.asarray(new['rot'][0]).shape[0]
    n1, o = 3 * n_rot + 3, 3 * n_rot
    sym = lambda A: np.tril(A) + np.tril(A, -1).T  # noqa: E731
    D = [sym(A[:n1, :n1]) for A, _ in sys_]
    B = [A[n1:, :n1].T for A, _ in sys_]
    E = sum(sym(A[n1:, n1:]) for A, _ in sys_)
    beta = np.asarray(new['betas'], np.float64)
    E = E + (float(np.float32(betas_w)) + float(lam)) * np.eye(nb)
    rb = -sum(g[n1:] for _, g in sys_) - float(np.float32(betas_w)) * beta
    with np.errstate(all='ignore'):
        x, db, ok = sweep(D, C, B, E, [-g[:n1] for _, g in sys_], rb)
    ok = ok and math.isfinite(float(lnew)) and all(np.isfinite(v).all() for v in x) and np.isfinite(db).all()
    if not ok:
        nxt = {'rot': [np.asarray(r, f).copy() for r in new['rot']],
               'transl': [np.asarray(r, f).copy() for r in new['transl']], 'betas': np.asarray(new['betas'], f).copy()}
        return new, nxt, accept
    nxt = {'rot': [np.stack([exp_gram_schmidt(new['rot'][t][j], x[t][3 * j:3 * j + 3]) for j in range(n_rot)]).astype(f)
                   for t in range(T)],
           'transl': [np.array([f(float(new['transl'][t][c]) + x[t][o + c]) for c in range(3)], f) for t in range(T)],
           'betas': np.array([f(float(new['betas'][l]) + db[l]) for l in range(nb)], f)}
    return new, nxt, accept
