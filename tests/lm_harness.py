"""Helpers shared by the Levenberg-Marquardt and model-shape tests: small tensor helpers, the synthetic SMPL-X modules
and model variants, the CPU tests' toy problems, the random-Jacobian case builders of the 3D keypoint, the
single-image 2D and the grouped 2D steps, and one comparison of a stepped device state with its oracle.  Imports
without a GPU."""
import functools
import math

import numpy as np
import torch

import kp2d_lm_oracle as o2
import kp2dg_lm_oracle as og
import kp_lm_oracle
from oracle.lm_oracle import meas_loss
from shapy_b200 import synth

NAMES = ('mass', 'height', 'chest', 'waist', 'hips')
N_ROT = 22
TOL = 1e-4                        # the keypoint Jacobian's bar: per body and column block, 1e-4 max |J64|
F, PP = 1000.0, (500.0, 500.0)    # the perspective tests' camera


# ------------------------------------------------------------------------------------------------ small helpers
def bits(t):
    return t.contiguous().view(torch.int32)


def rodrigues(aa):
    """(..., 3, 3) float64 rotation matrices of the axis-angle vectors aa (tensor or array)."""
    aa = torch.as_tensor(aa, dtype=torch.float64)
    th = aa.norm(dim=-1, keepdim=True)
    k = aa / th.clamp_min(1e-300)
    kx, ky, kz = k.unbind(-1)
    z = torch.zeros_like(kx)
    K = torch.stack([z, -kz, ky, kz, z, -kx, -ky, kx, z], -1).view(*aa.shape[:-1], 3, 3)
    s, c = th.sin()[..., None], th.cos()[..., None]
    return torch.eye(3, dtype=torch.float64) + s * K + (1 - c) * (K @ K)


def launches_without_sync(fn):
    """fn() run with host synchronisation an error; returns (the launches it made, its result)."""
    from shapy_b200 import _lib
    L = _lib.lib()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        n0 = L.shapy_launch_count()
        res = fn()
        return L.shapy_launch_count() - n0, res
    finally:
        torch.cuda.set_sync_debug_mode(0)


# ------------------------------------------------------------------------------------------------ CPU toy problems
def expm(d):
    """exp([d]x) as a float64 NumPy matrix."""
    return rodrigues(np.asarray(d, np.float64)).numpy()


def toy_problem(seed, K=12):
    """Keypoints kp = R0 p (first half), R0 R1 p (second half) + beta q + t: two chained rotations, one betas, and
    its (3K, 10) Jacobian with the transl columns last (P = 3 * 2 + 1 + 3)."""
    rng = np.random.default_rng(seed)
    p = rng.normal(size=(K, 3))
    q = rng.normal(size=(K, 3)) * 0.2
    t = rng.normal(size=3) * 0.1
    half = K // 2

    def evaluate(rot, beta):
        kp = np.zeros((K, 3))
        kp[:half] = p[:half] @ rot[0].T
        kp[half:] = p[half:] @ (rot[0] @ rot[1]).T
        kp += beta[0] * q + t
        jac = np.zeros((3 * K, 10))
        for k in range(K):
            x = kp[k] - beta[0] * q[k] - t
            for a in range(3):
                jac[3 * k:3 * k + 3, a] = np.cross(rot[0][:, a], x)
                if k >= half:
                    jac[3 * k:3 * k + 3, 3 + a] = np.cross((rot[0] @ rot[1])[:, a], x)
            jac[3 * k:3 * k + 3, 6] = q[k]
            jac[3 * k:3 * k + 3, 7:] = np.eye(3)
        return kp, jac
    return evaluate, rng


def _skew(d):
    z = torch.zeros_like(d[..., 0])
    return torch.stack([z, -d[..., 2], d[..., 1], d[..., 2], z, -d[..., 0], -d[..., 1], d[..., 0], z],
                       -1).view(*d.shape[:-1], 3, 3)


def keypoints_at(model, betas, rot, transl, params):
    """Keypoints (N, K, 3) at the parameter offsets params (N, P) = [delta (3 n_rot) | betas | transl], float64."""
    from smplx_grad_ref import forward_differentiable
    N, n_rot = params.shape[0], rot.shape[0]
    nb = betas.shape[0]
    d = params[:, :3 * n_rot].reshape(N, n_rot, 3)
    R = rot.double()[None] @ torch.linalg.matrix_exp(_skew(d))
    out = forward_differentiable(model, betas.double()[None] + params[:, 3 * n_rot:3 * n_rot + nb], R)
    return out['joints'] + (transl.double()[None] + params[:, 3 * n_rot + nb:])[:, None]


# ------------------------------------------------------------------------------------------------ model variants
# Variants of synth.make_smplx() for the model-shape tests (test_model_shapes_cpu.py describes them).
KP_CACHE_ENTRIES = 2048           # kKpCacheEntries of smplx.cu: keypoint entries the Jacobian caches in shared memory
# name -> (NB, NE, J14 non-zeros per row or None for synth.make_smplx's own 14 x 32)
VARIANTS = {
    'nb1_ne0': (1, 0, None),
    'nb10_ne0': (10, 0, None),
    'nb16_ne16': (16, 16, None),
    'nb27_ne5_dense': (27, 5, [150] * 14),
    'edge_2048': (10, 10, [132] * 13 + [128]),
    'edge_2049': (10, 10, [132] * 13 + [128]),
}
EDGE_EXTRA = 0.02                 # the weight of edge_2049's added non-zero


@functools.lru_cache(maxsize=None)
def _base():
    return synth.make_smplx()


def _j14(seed, counts):
    V = synth.NUM_VERTS
    g = torch.Generator().manual_seed(seed)
    R = torch.zeros(len(counts), V)
    for r, n in enumerate(counts):
        idx = torch.randperm(V, generator=g)[:n]
        R[r, idx] = torch.softmax(torch.randn(n, generator=g), 0)
    return R


@functools.lru_cache(maxsize=None)
def _variant(name):
    NB, NE, counts = VARIANTS[name]
    m = dict(_base())
    V = m['v_template'].shape[0]
    g = torch.Generator().manual_seed(NB * 100 + NE)
    m['shapedirs'] = torch.randn(V, 3, NB, generator=g) * 5e-3
    m['expr_dirs'] = torch.randn(V, 3, NE, generator=g) * 5e-3      # (V, 3, 0) when NE = 0: no expression basis
    if counts is not None:
        R = _j14(sum(counts), counts)
        if name == 'edge_2049':
            free = [int(v) for v in torch.randperm(V, generator=torch.Generator().manual_seed(5)) if R[-1, v] == 0]
            R[-1, free[0]] = EDGE_EXTRA
        m['extra_joint_regressor'] = R
    return m


def variant_model(name):
    """A fresh dict of the variant's tensors (the tensors are shared: do not edit them in place)."""
    return dict(_variant(name))


def keypoint_entries(m, use_face_contour=True):
    """3 (L + D) + nnz(J14): the entry count the keypoint Jacobian compares with KP_CACHE_ENTRIES."""
    L = m['lmk_faces_idx'].shape[0]
    D = m['dynamic_lmk_faces_idx'].shape[1] if use_face_contour else 0
    return 3 * (L + D) + int((m['extra_joint_regressor'] != 0).sum())


def inputs(seed, B, n_rot, NB, NE=0):
    """Rotations, betas (B, NB), expression (B, NE) or None, transl, camera; necks turned past both ends of the contour
    LUT in bodies 0 and 1."""
    gen = torch.Generator().manual_seed(seed)
    rot = rodrigues(torch.randn(B, n_rot, 3, generator=gen, dtype=torch.float64) * 0.4).float()
    if n_rot > 15 and B > 1:
        rot[0, 12] = rodrigues(torch.tensor([0.0, 1.2, 0.0])).float()
        rot[1, 12] = rodrigues(torch.tensor([0.0, -1.2, 0.0])).float()
    return dict(rot=rot, betas=torch.randn(B, NB, generator=gen),
                expression=torch.randn(B, NE, generator=gen) if NE else None,
                transl=torch.randn(B, 3, generator=gen) * 0.1,
                camera=torch.randn(B, 3, generator=gen) * torch.tensor([3.0, 0.2, 0.2]) + torch.tensor([1.0, 0, 0]))


# ------------------------------------------------------------------------------------------------ SMPL-X modules
_MODULES = {}


def smplx_module(variant='full'):
    """The synthetic SMPL-X module on the device, built once per variant: 'full' (face contour and J14),
    'no_contour_no_j14', or a name of VARIANTS."""
    if variant not in _MODULES:
        from shapy_b200.human_shape.models.body_models.body_models import SMPLX
        if variant in VARIANTS:
            NB, NE, _ = VARIANTS[variant]
            m = SMPLX(data_struct=variant_model(variant), betas={'num': NB}, expression={'num': NE},
                      use_face_contour=True)
        else:
            d = dict(synth.make_smplx())
            if variant == 'no_contour_no_j14':
                for k in ('extra_joint_regressor', 'source_idxs', 'target_idxs'):
                    d.pop(k)
            m = SMPLX(data_struct=d, use_face_contour=variant == 'full')
        _MODULES[variant] = m.cuda()
    return _MODULES[variant]


def smplx_and_measurements():
    """The 'full' module and the synthetic BodyMeasurements, both on the device, built once."""
    if 'measurements' not in _MODULES:
        from shapy_b200.body_measurements import BodyMeasurements
        _MODULES['measurements'] = BodyMeasurements({'landmarks': synth.load_landmarks()}).cuda()
    return smplx_module(), _MODULES['measurements']


def measure(module, bm, betas):
    """(B, 5) measurements of the betas, in the order of NAMES."""
    with torch.no_grad():
        m = bm.forward_vertices(module.forward_shape(betas=betas)['v_shaped'], module.faces_i32)['measurements']
    return torch.stack([m[k]['tensor'] for k in NAMES], 1)


# ------------------------------------------------------------------------------------------------ 2D fit quality
def quality_2d(module, bm, p, res, w=None, rms_threshold=2e-3):
    """Shares of the bodies with height within 1 mm, mass within 1 % and 2D RMS (crop frame) within rms_threshold;
    the median |beta - beta*| and root-aligned 3D joint error [m]."""
    from shapy_b200.metrics import PointError, build_alignment
    meas = res['measurements'] if 'measurements' in res else measure(module, bm, res['betas'])
    tgt = p['tgt']
    ok = torch.isfinite(tgt).all(1) & torch.isfinite(meas).all(1)
    d = (res['proj_joints'] - p['x']).pow(2).sum(-1)
    rms = d.mean(1).sqrt() if w is None else ((d * w).sum(1) / w.sum()).sqrt()
    pe = PointError(build_alignment('root'))
    pe(res['keypoints'].contiguous(), p['joints'])
    return {'height_1mm': float((((meas[:, 1] - tgt[:, 1]).abs() < 1e-3) & ok).float().mean()),
            'mass_1pct': float((((meas[:, 0] - tgt[:, 0]).abs() / tgt[:, 0].abs() < 1e-2) & ok).float().mean()),
            'circ_0.5pct': float(((((meas - tgt).abs() / tgt.abs())[:, 2:] < 5e-3).all(1) & ok).float().mean()),
            'frac_rms2d': float((rms < rms_threshold).float().mean()), 'median_rms2d': float(rms.median()),
            'median_beta_err': float((res['betas'] - p['bstar']).norm(dim=1).median()),
            'median_root_mpjpe_m': float(pe.last_mean.median())}


def quality_groups(module, bm, p, res, grouped):
    """quality_2d over the images of p['groups']; grouped: the betas error and height share per identity."""
    q = quality_2d(module, bm, dict(p, tgt=p['tgt'][p['groups']], bstar=p['bstar'][p['groups']]),
                   dict(res, betas=res['betas'][p['groups']],
                        **({'measurements': res['measurements'][p['groups']]} if 'measurements' in res else {})),
                   p.get('w'))
    if grouped:                       # per identity, not per image
        meas = res['measurements'] if 'measurements' in res else measure(module, bm, res['betas'])
        q['median_beta_err'] = float((res['betas'] - p['bstar']).norm(dim=1).median())
        q['height_1mm'] = float(((meas[:, 1] - p['tgt'][:, 1]).abs() < 1e-3).float().mean())
    return q


# ------------------------------------------------------------------------------------------------ step comparison
def numpy_of(d):
    return {k: v.cpu().numpy() for k, v in d.items()}


def rows_of(d, n):
    """The first n rows of a dict of arrays, one dict per row."""
    return [{k: v[r] for k, v in d.items()} for r in range(n)]


def check_step(got, nxt, oracle, state_keys, trial_keys, exact):
    """Row by row, the device's stepped state got[r] and next trial nxt[r] (dicts of NumPy arrays) against the oracle's
    (new, want, accepted) = oracle[r]: accepted equal; lambda and loss equal (exact) or within rtol 3e-7 (fp32
    rounding of exp / log1p); every state field in state_keys bit for bit, NaN equal; every next-trial field in
    trial_keys within 2e-6 max(1, |want|), per item where want[k] is a list of items.  Zero-width fields are skipped.
    Returns (the oracle's accepted flags, the largest trial error over its bar)."""
    flags, worst = [], 0.0
    for r, (g, x, (new, want, acc)) in enumerate(zip(got, nxt, oracle)):
        flags.append(acc)
        assert g['accepted'] == new['accepted'], r
        if exact:
            assert g['lambda'] == new['lambda'], (r, g['lambda'], new['lambda'])
            assert np.array_equal(g['loss'], new['loss'], equal_nan=True), (r, g['loss'], new['loss'])
        else:
            assert np.isclose(g['lambda'], new['lambda'], rtol=3e-7, atol=0), (r, g['lambda'], new['lambda'])
            assert np.isclose(g['loss'], new['loss'], rtol=3e-7, atol=0, equal_nan=True), (r, g['loss'], new['loss'])
        for k in state_keys:
            assert np.array_equal(g[k], np.asarray(new[k]), equal_nan=True), (r, k)
        for k in trial_keys:
            items = list(zip(x[k], want[k])) if isinstance(want[k], list) else [(x[k], want[k])]
            for j, (a, b) in enumerate(items):
                if b.size == 0:
                    continue
                bar = 2e-6 * max(1.0, np.abs(b).max())
                err = np.abs(a - b).max()
                assert err <= bar, (r, k, j, err)
                worst = max(worst, err / bar)
    return flags, worst


# ------------------------------------------------------------------------------------------------ 3D keypoint step
def kp_random_case(n_rot, nb, K, meas, rho=0.0):
    """Six bodies with random well-conditioned Jacobians: body 0's trial hits its targets (accepted), body 1's state
    does and its trial is far (rejected), body 2 has a weighted NaN trial keypoint (rejected), with measurements body
    3 a weighted NaN trial measurement (rejected), 4 and 5 random.  With K >= 6 keypoint 5 has weight 0 and NaN
    keypoints and rows in state and trial; with measurements the height has weight 0 and NaN values and rows.  The
    state's loss is the oracle's (float32) at betas weight rho."""
    B, P = 6, 3 * n_rot + nb + 3
    gen = torch.Generator().manual_seed(1000 * n_rot + 10 * nb + K + (7 if meas else 0))
    rn = lambda *s: torch.randn(*s, generator=gen)  # noqa: E731
    rot = rodrigues(rn(B, n_rot, 3) * 0.5).float()
    trot = (rot.double() @ rodrigues(rn(B, n_rot, 3) * 0.05)).float()
    betas, transl = rn(B, nb), rn(B, 3) * 0.1
    tbetas, ttransl = betas + 0.05 * rn(B, nb), transl + 0.01 * rn(B, 3)
    kp, jac = rn(B, K, 3), rn(B, 3 * K, P)
    tkp, tjac = kp + 0.05 * rn(B, K, 3), jac + 0.1 * rn(B, 3 * K, P)
    tg = kp + 0.05 * rn(B, K, 3)
    w = torch.rand(B, K, generator=gen) + 0.5
    kp[0] = tkp[0] + 0.5
    tg[0] = tkp[0]
    tg[1], tkp[1] = kp[1], kp[1] + 0.5
    tkp[2, 0, 1] = float('nan')
    if K >= 6:
        w[:, 5] = 0.0
        for t in (kp, tkp):
            t[:, 5] = float('nan')
        for t in (jac, tjac):
            t[:, 15:18] = float('nan')
    c = dict(rot=rot, betas=betas, transl=transl, kp=kp, jac=jac, trot=trot, tbetas=tbetas, ttransl=ttransl, tkp=tkp,
             tjac=tjac, tg=tg, w=w, lam=torch.rand(B, generator=gen) + 0.01)
    n = lambda t: t.numpy()  # noqa: E731
    if meas:
        m, mj = torch.rand(B, 5, generator=gen) + 0.5, rn(B, 5, nb)
        tm, tmj = m + 0.01 * rn(B, 5), mj + 0.1 * rn(B, 5, nb)
        mt = m + 0.02 * rn(B, 5)
        mt[0], mt[1] = tm[0], m[1]
        mw = torch.rand(B, 5, generator=gen) * 2 + 0.5
        mw[:, 1] = 0.0
        for t in (m, tm, mj, tmj):
            t[:, 1] = float('nan')
        tm[3, 3] = float('nan')
        c.update(meas=m, mjac=mj, tmeas=tm, tmjac=tmj, mt=mt, mw=mw)
        loss = [kp_lm_oracle.loss(n(tg[b]), n(w[b]), n(kp[b]), (n(mt[b]), n(mw[b]), n(m[b])), n(betas[b]), rho)
                for b in range(B)]
    else:
        loss = [kp_lm_oracle.loss(n(tg[b]), n(w[b]), n(kp[b])) for b in range(B)]
    c['loss'] = torch.tensor(np.array(loss, np.float32))
    return c


def kp_check(c, state, trial, first, rho=None):
    """The stepped device state and next trial against kp_lm_oracle body by body, from the case's state (rho None: the
    keypoint step, else the measurement step at betas weight rho); returns (the accepted flags, the largest trial error
    over its bar).  Loss and lambda are bit for bit: the kernel is built with -fmad=false."""
    B = c['rot'].shape[0]
    n = lambda t: t.numpy()  # noqa: E731
    oracle = []
    for b in range(B):
        s = {'rot': n(c['rot'][b]), 'betas': n(c['betas'][b]), 'transl': n(c['transl'][b]), 'keypoints': n(c['kp'][b]),
             'jac': n(c['jac'][b]), 'loss': n(c['loss'][b]), 'lambda': n(c['lam'][b]), 'accepted': 0}
        tr = {'rot': n(c['trot'][b]), 'betas': n(c['tbetas'][b]), 'transl': n(c['ttransl'][b])}
        kw = {} if rho is None else dict(meas=(n(c['mt'][b]), n(c['mw'][b])), betas_weight=rho,
                                         trial_meas=(n(c['tmeas'][b]), n(c['tmjac'][b])))
        if rho is not None:
            s.update(meas=n(c['meas'][b]), meas_jac=n(c['mjac'][b]))
        oracle.append(kp_lm_oracle.lm_keypoints_step(s, n(c['tg'][b]), n(c['w'][b]), 10.0, 3.0, first, tr,
                                                     n(c['tkp'][b]), n(c['tjac'][b]), **kw))
    keys = ('rot', 'betas', 'transl')
    got, nxt = numpy_of(state), numpy_of(trial)
    return check_step(rows_of(got, B), rows_of(nxt, B), oracle,
                      keys + ('keypoints', 'jac') + (() if rho is None else ('meas', 'meas_jac')), keys, exact=True)


def kp_device(c, rho=None):
    """A 3D keypoint case's state (with its measurement block unless rho is None) and trial on the device."""
    B = c['rot'].shape[0]
    cu = lambda t: t.cuda().contiguous()  # noqa: E731
    state = {'rot': cu(c['rot']), 'betas': cu(c['betas']), 'transl': cu(c['transl']), 'keypoints': cu(c['kp']),
             'jac': cu(c['jac']), 'loss': cu(c['loss']), 'lambda': cu(c['lam']),
             'accepted': torch.zeros(B, dtype=torch.int32, device='cuda')}
    if rho is not None:
        state.update(meas=cu(c['meas']), meas_jac=cu(c['mjac']))
    trial = {'rot': cu(c['trot']), 'betas': cu(c['tbetas']), 'transl': cu(c['ttransl'])}
    return state, trial


def kp_step(c, state, trial, first, rho=None):
    """One 3D keypoint step on the case (rho None), or one measurement step at betas weight rho."""
    from shapy_b200 import ops
    cu = lambda t: t.cuda().contiguous()  # noqa: E731
    if rho is None:
        ops.fit_lm_keypoints_step(state, trial, cu(c['tg']), cu(c['w']), 10.0, 3.0, first, cu(c['tkp']), cu(c['tjac']))
    else:
        ops.fit_lm_keypoints_measurements_step(state, trial, cu(c['tg']), cu(c['w']), cu(c['mt']), cu(c['mw']), rho,
                                               10.0, 3.0, first, cu(c['tkp']), cu(c['tjac']), cu(c['tmeas']),
                                               cu(c['tmjac']))


# ------------------------------------------------------------------------------------------------ single-image 2D step
# (robust_sigma, pose_prior_weight, betas_weight) of the plain and measurement entries, sigma in pixels under the
# perspective camera; (robust_sigma, pose_prior_weight ('joint': per-joint weights), betas_weight, expression_weight)
# of the expressive entry
KP2D_TERMS = {'weak': [(math.inf, 0.0, 0.0), (0.3, 0.5, 0.1)], 'persp': [(math.inf, 0.0, 0.0), (20.0, 500.0, 100.0)]}
EXPR_TERMS = {'weak': [(math.inf, 0.0, 0.0, 0.0), (0.3, 'joint', 1.0, 0.5), (0.3, 2.0, 0.1, 0.0)],
              'persp': [(math.inf, 0.0, 0.0, 0.0), (30.0, 'joint', 1.0, 0.5), (30.0, 2.0, 0.1, 0.0)]}


def kp2d_case(n_rot, nb, K, terms, persp=False, meas=False, ne=None):
    """Eight bodies with random Jacobians for the single-image 2D step: weak-perspective, or keypoints about 3-4 m in
    front of a 1000 px camera (persp); ne None: the plain entries, ne >= 0: the expressive entry with ne expression
    columns.  Body 0's trial hits its targets (accepted), body 1's state does and its trial is far (rejected), body 2
    has a weighted NaN trial keypoint (rejected); with `meas` (five random measurements and rows) body 3 a weighted NaN
    trial measurement (rejected) and the height weight 0 with NaN values and rows in state and trial; under the
    perspective camera body 4's trial a weighted keypoint behind the camera (rejected) and, with K >= 8, body 5's trial
    a dropped one behind it (not read); the rest random.  With K >= 8 keypoint 7 has weight 0 and NaN targets,
    keypoints and rows in state and trial."""
    sigma, pw, bw, ew = (tuple(terms) + (0.0,))[:4]
    NE = 0 if ne is None else ne
    B, P = 8, 3 * n_rot + nb + NE + 3
    gen = torch.Generator().manual_seed(1000 * n_rot + 100 * NE + 10 * nb + K + 3 * bool(pw) + 5 * persp + 7 * meas +
                                        11 * (ne is not None) + 13 * (ew > 0))
    rn = lambda *s: torch.randn(*s, generator=gen)  # noqa: E731
    # scales: keypoints, rows, trial keypoint and row noise, the offset of the far keypoints, trial camera / translation
    # noise and target noise
    sk, sj, dk, dj, far, dl, noise = (0.4, 0.3, 0.01, 0.03, 0.1, 0.02, 5.0) if persp else \
        (1.0, 1.0, 0.05, 0.1, 0.5, 0.01, 0.05)
    rot = rodrigues(rn(B, n_rot, 3) * 0.5).float()
    trot = (rot.double() @ rodrigues(rn(B, n_rot, 3) * 0.05)).float()
    anchor = (rot.double() @ rodrigues(rn(B, n_rot, 3) * 0.1)).float()
    betas, expr = rn(B, nb), rn(B, NE)
    if persp:
        last = torch.cat([0.3 * rn(B, 2), 3.0 + torch.rand(B, 1, generator=gen)], 1)
        intr = torch.tensor([F, *PP]).repeat(B, 1)
        intr[6:, 0] = 800.0 + 400.0 * torch.rand(2, generator=gen)
    else:
        last = rn(B, 3) * torch.tensor([0.5, 0.1, 0.1])
        intr = None
    tbetas, texpr, tlast = betas + 0.05 * rn(B, nb), expr + 0.05 * rn(B, NE), last + dl * rn(B, 3)
    anchor[0], tbetas[0], texpr[0] = trot[0], 0.9 * betas[0], 0.9 * expr[0]     # the priors favour body 0's trial ...
    anchor[1], tbetas[1], texpr[1] = rot[1], 1.1 * betas[1], 1.1 * expr[1]     # ... and body 1's state
    kp, jac = sk * rn(B, K, 3), sj * rn(B, 3 * K, P)
    tkp, tjac = kp + dk * rn(B, K, 3), jac + dj * rn(B, 3 * K, P)
    kp[0] = tkp[0] + far
    tkp[1] = kp[1] + far

    def proj(k, c, b):
        return torch.from_numpy(o2.project(k.numpy(), c.numpy(), None if intr is None else intr[b].numpy())).float()
    tg = torch.stack([proj(kp[b], last[b], b) for b in range(B)]) + noise * rn(B, K, 2)
    tg[0], tg[1] = proj(tkp[0], tlast[0], 0), proj(kp[1], last[1], 1)
    tkp[2, 0, 1] = float('nan')
    if persp:
        tkp[4, 0, 2] = -tlast[4, 2] - 0.5                # Y_z = -0.5
    w = torch.rand(B, K, generator=gen) + 0.5
    if K >= 8:
        w[:, 7] = 0.0
        tg[:, 7] = float('nan')
        for t in (kp, tkp):
            t[:, 7] = float('nan')
        for t in (jac, tjac):
            t[:, 21:24] = float('nan')
        if persp:
            tkp[5, 7, 2] = -10.0                         # dropped and behind the camera: not read
    jw = None
    if pw == 'joint':
        jw = torch.rand(n_rot, generator=gen) * 3.0
        jw[0] = 0.0
        if n_rot > 3:
            jw[2] = 0.0
        pw = 0.0
    c = dict(rot=rot, betas=betas, last=last, kp=kp, jac=jac, trot=trot, tbetas=tbetas, tlast=tlast, tkp=tkp,
             tjac=tjac, tg=tg, w=w, intr=intr, anchor=anchor, jw=jw, lam=torch.rand(B, generator=gen) + 0.01,
             sigma=sigma, pw=pw, bw=bw, ew=ew, lastkey='transl' if persp else 'camera')
    if ne is not None:
        c.update(expr=expr, texpr=texpr)
    if meas:
        m, mj = torch.rand(B, 5, generator=gen) + 0.5, rn(B, 5, nb)
        tm, tmj = m + 0.01 * rn(B, 5), mj + 0.1 * rn(B, 5, nb)
        mt = m + 0.02 * rn(B, 5)
        mt[0], mt[1] = tm[0], m[1]
        mw = torch.rand(B, 5, generator=gen) * 2 + 0.5
        mw[:, 1] = 0.0
        for t in (m, tm, mj, tmj):
            t[:, 1] = float('nan')
        tm[3, 3] = float('nan')
        c.update(meas=m, mjac=mj, tmeas=tm, tmjac=tmj, mt=mt, mw=mw)
    return c


def _kp2d_kw(c, b):
    """The oracle's keyword arguments for body b of the case."""
    n = lambda t: None if t is None else t.numpy()  # noqa: E731
    kw = dict(sigma=c['sigma'], anchor=n(c['anchor'][b]), pose_w=c['pw'], joint_w=n(c['jw']), betas_w=c['bw'],
              expr_w=c['ew'], intr=None if c['intr'] is None else n(c['intr'][b]))
    if 'meas' in c:
        kw.update(meas=(n(c['mt'][b]), n(c['mw'][b])), trial_meas=(n(c['tmeas'][b]), n(c['tmjac'][b])))
    return kw


def kp2d_state_np(c, b):
    """Body b's state for the oracle, its loss the oracle's (float32)."""
    n = lambda t: t.numpy()  # noqa: E731
    s = {'rot': n(c['rot'][b]), 'betas': n(c['betas'][b]), c['lastkey']: n(c['last'][b]), 'keypoints': n(c['kp'][b]),
         'jac': n(c['jac'][b]), 'lambda': n(c['lam'][b]), 'accepted': 0}
    if 'expr' in c:
        s['expression'] = n(c['expr'][b])
    if 'meas' in c:
        s.update(meas=n(c['meas'][b]), meas_jac=n(c['mjac'][b]))
    kw = _kp2d_kw(c, b)
    s['loss'] = np.float32(o2.loss(n(c['tg'][b]), n(c['w'][b]), s['keypoints'], s[c['lastkey']], kw['sigma'],
                                   s['rot'], kw['anchor'], kw['pose_w'], s['betas'], kw['betas_w'], kw['intr'],
                                   kw['joint_w'], s.get('expression'), kw['expr_w'],
                                   (n(c['mt'][b]), n(c['mw'][b]), s['meas']) if 'meas' in c else None))
    return s


def kp2d_device(c):
    """The case's state and trial on the device, the state's loss from the oracle."""
    B = c['rot'].shape[0]
    cu = lambda t: t.cuda().contiguous()  # noqa: E731
    lk = c['lastkey']
    state = {'rot': cu(c['rot']), 'betas': cu(c['betas']), lk: cu(c['last']), 'keypoints': cu(c['kp']),
             'jac': cu(c['jac']), 'loss': cu(torch.tensor(np.array([kp2d_state_np(c, b)['loss'] for b in range(B)]))),
             'lambda': cu(c['lam']), 'accepted': torch.zeros(B, dtype=torch.int32, device='cuda')}
    trial = {'rot': cu(c['trot']), 'betas': cu(c['tbetas']), lk: cu(c['tlast'])}
    if 'expr' in c:
        state['expression'], trial['expression'] = cu(c['expr']), cu(c['texpr'])
    if 'meas' in c:
        state.update(meas=cu(c['meas']), meas_jac=cu(c['mjac']))
    return state, trial


def kp2d_step(c, state, trial, first, meas=None):
    """One step of the case's entry (the expressive entry when the case has expression columns) on its inputs, read in
    place when they are on the device.  meas: (targets, weights, trial_meas, trial_meas_jac) for the measurement entry,
    by default the case's own when it has them."""
    from shapy_b200 import ops
    cu = lambda t: None if t is None else t.cuda().contiguous()  # noqa: E731
    if meas is None and 'meas' in c:
        meas = tuple(cu(c[k]) for k in ('mt', 'mw', 'tmeas', 'tmjac'))
    head = (state, trial, cu(c['tg']), cu(c['w']))
    terms = (c['sigma'], c['pw'], c['bw'])
    tail = (10.0, 3.0, first, cu(c['tkp']), cu(c['tjac']))
    anchor = cu(c['anchor'])
    if 'expr' in c:
        ops.fit_lm_keypoints_2d_expressive_step(*head, *terms, c['ew'], *tail, pose_anchor=anchor,
                                                joint_weights=cu(c['jw']), intrinsics=cu(c['intr']))
    elif c['intr'] is not None and meas is not None:
        ops.fit_lm_keypoints_2d_perspective_measurements_step(*head, cu(c['intr']), *terms, meas[0], meas[1], *tail,
                                                              meas[2], meas[3], pose_anchor=anchor)
    elif c['intr'] is not None:
        ops.fit_lm_keypoints_2d_perspective_step(*head, cu(c['intr']), *terms, *tail, pose_anchor=anchor)
    elif meas is not None:
        ops.fit_lm_keypoints_2d_measurements_step(*head, *terms, meas[0], meas[1], *tail, meas[2], meas[3],
                                                  pose_anchor=anchor)
    else:
        ops.fit_lm_keypoints_2d_step(*head, *terms, *tail, pose_anchor=anchor)


def kp2d_run(first, **case):
    """kp2d_case(**case) stepped once on the device and checked by kp2d_check; returns the largest trial error over its
    bar."""
    c = kp2d_case(**case)
    state, trial = kp2d_device(c)
    kp2d_step(c, state, trial, first)
    return kp2d_check(c, state, trial, first)


def kp2d_oracle(c, first):
    """The oracle's (new, want, accepted) for every body of the case."""
    n = lambda t: t.numpy()  # noqa: E731
    out = []
    for b in range(c['rot'].shape[0]):
        tr = {'rot': n(c['trot'][b]), 'betas': n(c['tbetas'][b]), c['lastkey']: n(c['tlast'][b])}
        if 'expr' in c:
            tr['expression'] = n(c['texpr'][b])
        out.append(o2.lm_keypoints_2d_step(kp2d_state_np(c, b), n(c['tg'][b]), n(c['w'][b]), 10.0, 3.0, first, tr,
                                           n(c['tkp'][b]), n(c['tjac'][b]), **_kp2d_kw(c, b)))
    return out


def kp2d_keys(c):
    """The case's (state keys, next-trial keys) compared with the oracle."""
    trial = ('rot', 'betas') + (('expression',) if 'expr' in c else ()) + (c['lastkey'],)
    return trial + ('keypoints', 'jac') + (('meas', 'meas_jac') if 'meas' in c else ()), trial


def kp2d_check(c, state, trial, first):
    """The stepped device state and next trial of a kp2d_case against the oracle by check_step, and the accept pattern
    of its roles: every body accepts a first step; otherwise body 0 accepts and 1, 2, 3 (with measurements) and 4
    (perspective) reject.  A first step from behind the camera reports NaN and does not move, and the dropped keypoint
    behind the camera is not read.  Returns the largest trial error over its bar."""
    B = c['rot'].shape[0]
    got, nxt = numpy_of(state), numpy_of(trial)
    flags, worst = check_step(rows_of(got, B), rows_of(nxt, B), kp2d_oracle(c, first), *kp2d_keys(c), exact=False)
    kp2d_expected_flags(c, first, flags)
    if c['intr'] is not None and first:
        assert math.isnan(got['loss'][4]) and np.array_equal(nxt['transl'][4], c['tlast'][4].numpy())
    if c['intr'] is not None and c['kp'].shape[1] >= 8:
        assert math.isfinite(got['loss'][5])
    return worst


def kp2d_expected_flags(c, first, flags):
    """The accept pattern of the case's roles."""
    if first:
        assert all(flags), flags
        return
    assert flags[0] and not flags[1] and not flags[2], flags
    assert 'meas' not in c or not flags[3], flags
    assert c['intr'] is None or not flags[4], flags


# ------------------------------------------------------------------------------------------------ grouped 2D step
def random_group_case(n_rot, nb, K, terms, sizes):
    """Groups of `sizes` images with random Jacobians at (n_rot, nb): group 0 targets the trial (accepted), 1 the state
    with the priors on its side and a trial 0.5 away (rejected), 2 the trial (accepted), the rest noisy targets.  With
    K >= 8 keypoint 7 has weight 0 and NaN targets, keypoints and rows in state and trial; measurement 2 of group 2 (of
    the last group when there are fewer) is dropped with NaN values and rows."""
    sigma, pw, bw = terms
    G, B, P = len(sizes), sum(sizes), 3 * n_rot + nb + 3
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    gidx = torch.repeat_interleave(torch.arange(G), torch.tensor(sizes))
    gen = torch.Generator().manual_seed(1000 * n_rot + 10 * nb + K + B + (3 if pw else 0))
    rn = lambda *s: torch.randn(*s, generator=gen)  # noqa: E731
    rot = rodrigues(rn(B, n_rot, 3) * 0.5).float()
    trot = (rot.double() @ rodrigues(rn(B, n_rot, 3) * 0.05)).float()
    anchor = (rot.double() @ rodrigues(rn(B, n_rot, 3) * 0.1)).float()
    betas, cam = rn(G, nb), rn(B, 3) * torch.tensor([0.5, 0.1, 0.1])
    tbetas, tcam = betas + 0.05 * rn(G, nb), cam + 0.01 * rn(B, 3)
    kp, jac = rn(B, K, 3), rn(B, 3 * K, P)
    tkp, tjac = kp + 0.05 * rn(B, K, 3), jac + 0.1 * rn(B, 3 * K, P)
    m, mj = torch.rand(G, 5, generator=gen) + 0.5, rn(G, 5, nb)
    tm, tmj = m + 0.01 * rn(G, 5), mj + 0.1 * rn(G, 5, nb)
    proj = lambda k, c: torch.stack([torch.from_numpy(o2.project(k[b].numpy(), c[b].numpy())).float()  # noqa: E731
                                     for b in range(k.shape[0])])
    tg = proj(kp, cam) + 0.05 * rn(B, K, 2)
    mt = m + 0.02 * rn(G, 5)
    for g, to_trial in zip(range(G), (True, False, True)):
        r = slice(off[g], off[g + 1])
        if to_trial:
            kp[r] = tkp[r] + 0.5
            tg[r], anchor[r], tbetas[g], mt[g] = proj(tkp[r], tcam[r]), trot[r], 0.9 * betas[g], tm[g]
        else:
            tkp[r] = kp[r] + 0.5
            tg[r], anchor[r], tbetas[g], mt[g] = proj(kp[r], cam[r]), rot[r], 1.1 * betas[g], m[g]
    w = torch.rand(B, K, generator=gen) + 0.5
    if K >= 8:
        w[:, 7] = 0.0
        tg[:, 7] = float('nan')
        for t in (kp, tkp):
            t[:, 7] = float('nan')
        for t in (jac, tjac):
            t[:, 21:24] = float('nan')
    mw = torch.rand(G, 5, generator=gen) * 2 + 0.5
    gd = min(2, G - 1)
    mw[gd, 2] = 0.0
    for t in (m, tm, mj, tmj):
        t[gd, 2] = float('nan')
    return dict(off=off, gidx=gidx, rot=rot, betas=betas, cam=cam, kp=kp, jac=jac, meas=m, mjac=mj, trot=trot,
                tbetas=tbetas, tcam=tcam, tkp=tkp, tjac=tjac, tmeas=tm, tmjac=tmj, tg=tg, w=w, mt=mt, mw=mw,
                anchor=anchor, lam=torch.rand(G, generator=gen) + 0.01, sigma=sigma, pw=pw, bw=bw)


def _groups_state_loss(c, g, with_meas):
    n = lambda t: t.numpy()  # noqa: E731
    L = 0.0
    for i in range(c['off'][g], c['off'][g + 1]):
        L += o2.loss(n(c['tg'][i]), n(c['w'][i]), n(c['kp'][i]), n(c['cam'][i]), c['sigma'], n(c['rot'][i]),
                     n(c['anchor'][i]), c['pw'])
    if with_meas:
        L += meas_loss(n(c['mt'][g]), n(c['mw'][g]), n(c['meas'][g]))
    if c['bw'] > 0:
        L += float(np.float32(c['bw'])) * float(np.sum(n(c['betas'][g]).astype(np.float64) ** 2))
    return L


def groups_device(c, with_meas):
    """A grouped case's state and trial on the device, the state's loss from the oracle; returns (state, trial, B,
    G)."""
    G = len(c['off']) - 1
    B = c['rot'].shape[0]
    cu = lambda t: t.cuda().contiguous()  # noqa: E731
    loss = torch.tensor([_groups_state_loss(c, g, with_meas) for g in range(G)]).float()
    state = {'rot': cu(c['rot']), 'betas': cu(c['betas']), 'camera': cu(c['cam']), 'keypoints': cu(c['kp']),
             'jac': cu(c['jac']), 'loss': cu(loss), 'lambda': cu(c['lam']),
             'accepted': torch.zeros(G, dtype=torch.int32, device='cuda')}
    if with_meas:
        state.update(meas=cu(c['meas']), meas_jac=cu(c['mjac']))
    trial = {'rot': cu(c['trot']), 'betas': cu(c['tbetas']), 'image_betas': cu(c['tbetas'][c['gidx']]),
             'camera': cu(c['tcam'])}
    return state, trial, B, G


def groups_step(c, state, trial, first, with_meas, ws=None):
    """One grouped step on the case at its n_rot and nb; ws: the workspace (by default a fresh one)."""
    from shapy_b200 import ops
    cu = lambda t: t.cuda().contiguous()  # noqa: E731
    B, G = c['rot'].shape[0], len(c['off']) - 1
    if ws is None:
        ws = ops.fit_lm_groups_workspace(B, G, c['rot'].shape[1], c['betas'].shape[1], 'cuda')
    off = torch.from_numpy(c['off'])
    if with_meas:
        ops.fit_lm_keypoints_2d_groups_measurements_step(
            state, trial, cu(c['tg']), cu(c['w']), c['sigma'], c['pw'], c['bw'], cu(c['mt']), cu(c['mw']), 10.0, 3.0,
            first, cu(c['tkp']), cu(c['tjac']), cu(c['tmeas']), cu(c['tmjac']), off, ws, pose_anchor=cu(c['anchor']))
    else:
        ops.fit_lm_keypoints_2d_groups_step(state, trial, cu(c['tg']), cu(c['w']), c['sigma'], c['pw'], c['bw'], 10.0,
                                            3.0, first, cu(c['tkp']), cu(c['tjac']), off, ws,
                                            pose_anchor=cu(c['anchor']))


def group_rows(c, got, nxt, G, image_keys, group_keys):
    """The stepped device state and next trial (NumPy) as one row per group: the group's images' fields stacked
    (image_keys), its own fields (group_keys and the accept, loss and lambda counters) as they are."""
    gs, xs = [], []
    for g in range(G):
        a, b = int(c['off'][g]), int(c['off'][g + 1])
        gs.append({k: v[a:b] if k in image_keys else v[g] for k, v in got.items()})
        xs.append({k: v[a:b] if k in image_keys else v[g] for k, v in nxt.items()})
    return gs, xs


def check_groups_vs_oracle(c, s0, state, trial, first, with_meas):
    """The stepped device state and next trial against kp2dg_lm_oracle group by group, from the state s0 (NumPy) before
    the step, by check_step; each image's trial betas must be its group's.  Returns (the groups' accepted flags, the
    largest trial error over its bar)."""
    G = len(c['off']) - 1
    n = lambda t: t.numpy()  # noqa: E731
    oracle = []
    for g in range(G):
        r = range(c['off'][g], c['off'][g + 1])
        st = {k: [s0[k][i] for i in r] for k in ('rot', 'camera', 'keypoints', 'jac')}
        st.update(betas=s0['betas'][g], loss=s0['loss'][g], accepted=0, **{'lambda': s0['lambda'][g]})
        if with_meas:
            st.update(meas=s0['meas'][g], meas_jac=s0['meas_jac'][g])
        images = [{'targets': n(c['tg'][i]), 'weights': n(c['w'][i]), 'anchor': n(c['anchor'][i]),
                   'trial_kp': n(c['tkp'][i]), 'trial_jac': n(c['tjac'][i])} for i in r]
        tr = {'rot': [n(c['trot'][i]) for i in r], 'camera': [n(c['tcam'][i]) for i in r],
              'betas': n(c['tbetas'][g])}
        mb = None if not with_meas else {'targets': n(c['mt'][g]), 'weights': n(c['mw'][g]),
                                         'trial_meas': n(c['tmeas'][g]), 'trial_meas_jac': n(c['tmjac'][g])}
        oracle.append(og.lm_groups_step(st, images, 10.0, 3.0, first, tr, c['sigma'], c['pw'], c['bw'], mb)[:3])
    got, nxt = numpy_of(state), numpy_of(trial)
    for g in range(G):
        for i in range(c['off'][g], c['off'][g + 1]):
            assert np.array_equal(nxt['image_betas'][i], nxt['betas'][g]), (g, i)
    image = ('rot', 'camera', 'keypoints', 'jac')
    gs, xs = group_rows(c, got, nxt, G, image, ())
    return check_step(gs, xs, oracle, image + ('betas',) + (('meas', 'meas_jac') if with_meas else ()),
                      ('rot', 'camera', 'betas'), exact=False)


def check_groups_of_one(c, first):
    """The grouped step on a case of groups of one against shapy_fit_lm_keypoints_2d_step on the same images: loss,
    lambda, accepted and the state bit for bit; the next trial within 4e-6 max(1, |x|) (the CPU oracle test bounds the
    two eliminations' fp64 difference by 1e-10; what is left is the fp32 rounding of the result)."""
    from shapy_b200 import ops
    state, trial, B, G = groups_device(c, False)
    b_state = {k: v.clone() for k, v in state.items()}
    b_trial = {k: v.clone() for k, v in trial.items() if k != 'image_betas'}
    groups_step(c, state, trial, first, False)
    cu = lambda t: t.cuda().contiguous()  # noqa: E731
    ops.fit_lm_keypoints_2d_step(b_state, b_trial, cu(c['tg']), cu(c['w']), c['sigma'], c['pw'], c['bw'], 10.0, 3.0,
                                 first, cu(c['tkp']), cu(c['tjac']), pose_anchor=cu(c['anchor']))
    for k in ('rot', 'betas', 'camera', 'keypoints', 'jac', 'loss', 'lambda', 'accepted'):
        assert torch.equal(bits(state[k]), bits(b_state[k])), k
    for k in ('rot', 'betas', 'camera'):
        err = (trial[k] - b_trial[k]).abs().max()
        assert float(err) <= 4e-6 * max(1.0, float(b_trial[k].abs().max())), (k, float(err))


def check_dropped_measurements(c, first):
    """Every measurement of the case dropped (weight 0 or -1, NaN values and rows): the grouped measurements entry
    equals the plain grouped entry bit for bit."""
    for k in ('meas', 'tmeas', 'mjac', 'tmjac'):
        c[k][:] = float('nan')
    c['mw'][:] = 0.0
    c['mw'][:, 1] = -1.0
    a_state, a_trial, _, _ = groups_device(c, True)
    b_state = {k: v.clone() for k, v in a_state.items() if k not in ('meas', 'meas_jac')}
    b_trial = {k: v.clone() for k, v in a_trial.items()}
    groups_step(c, a_state, a_trial, first, True)
    groups_step(c, b_state, b_trial, first, False)
    for k in ('rot', 'betas', 'camera', 'keypoints', 'jac', 'loss', 'lambda', 'accepted'):
        assert torch.equal(bits(a_state[k]), bits(b_state[k])), k
    for k in ('rot', 'betas', 'image_betas', 'camera'):
        assert torch.equal(bits(a_trial[k]), bits(b_trial[k])), k
