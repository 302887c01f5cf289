"""CPU: the model variants of the shape tests (tests/test_gpu_model_shapes.py) and the float64 restatements at their
shapes, before the GPU kernels are compared with them.

Variants of synth.make_smplx(), defined in tests/lm_harness.py (shape and expression rows randn * 5e-3 seeded as in
test_gpu_smplx_poses.test_shape_expression_counts, J14 rows seeded random supports with softmax weights as in
synth.make_smplx's sparse_rows):

  nb1_ne0          NB 1, NE 0, the synthetic J14 (448 non-zeros)      smallest coefficient count
  nb10_ne0         NB 10, NE 0, the synthetic J14                    NC = NB, no expression rows
  nb16_ne16        NB 16, NE 16, the synthetic J14                   NC = 32 = kMaxCoef, NB = 16 = kMaxJacBetas
  nb27_ne5_dense   NB 27, NE 5, J14 14 x 150                         NC = 32, P = 96 at n_rot = 22, uncached Jacobian
  edge_2048        NB 10, NE 10, J14 with 1 844 non-zeros            2 048 keypoint entries: the last cached count
  edge_2049        edge_2048 plus one non-zero in the last J14 row    2 049 entries: the first uncached count

  * kp_lm_oracle.keypoint_jacobian against central differences of the float64 forward on nb1_ne0 and nb27_ne5_dense
  * kp_lm_oracle.lm_keypoints_step, with and without measurements, against a dense solve of the damped normal
    equations at P = 7 and P = 96
  * kp2d_lm_oracle (with and without measurements) and kp2dg_lm_oracle against explicitly stacked 2D rows and dense
    solves at
    nb = 1 to 27 and P = 7 to 96 (the toy problems of the 2D CPU tests have nb = 1, where a Schur block, X_i and each
    measurement row's outer product have one entry)
  * fit_body_to_keypoints(method='lm') and fit_body_to_keypoints_2d(method='lm') refuse more than 96 parameters before
    they touch the device"""
import math

import numpy as np
import pytest
import torch

import kp2d_lm_oracle as o2
import kp2dg_lm_oracle as og
import kp_lm_oracle
from lm_harness import KP_CACHE_ENTRIES, VARIANTS, keypoint_entries, keypoints_at, rodrigues, variant_model
from shapy_b200 import synth

LM_KP_MAX_P = 96                  # kLmKpMaxP of fit.cu


# ------------------------------------------------------------------------------------------------ variants
def test_variants_have_their_shapes():
    want_nnz = {'nb1_ne0': 448, 'nb10_ne0': 448, 'nb16_ne16': 448, 'nb27_ne5_dense': 2100, 'edge_2048': 1844,
                'edge_2049': 1845}
    for name, (NB, NE, _) in VARIANTS.items():
        m = variant_model(name)
        assert m['shapedirs'].shape[-1] == NB and m['expr_dirs'].shape[-1] == NE, name
        assert int((m['extra_joint_regressor'] != 0).sum()) == want_nnz[name], name
        assert NB + NE <= 32, name
    entries = {name: keypoint_entries(variant_model(name)) for name in VARIANTS}
    assert entries['edge_2048'] == KP_CACHE_ENTRIES and entries['edge_2049'] == KP_CACHE_ENTRIES + 1
    assert entries['nb27_ne5_dense'] == 2304 > KP_CACHE_ENTRIES
    assert 3 * 22 + VARIANTS['nb27_ne5_dense'][0] + 3 == LM_KP_MAX_P
    # edge_2049 is edge_2048 with one added non-zero in the last J14 row, everything else shared
    a, b = variant_model('edge_2048'), variant_model('edge_2049')
    diff = (a['extra_joint_regressor'] != b['extra_joint_regressor']).nonzero()
    assert diff.shape[0] == 1 and int(diff[0, 0]) == 13 and float(a['extra_joint_regressor'][tuple(diff[0])]) == 0.0
    for k in a:
        if k != 'extra_joint_regressor':
            assert a[k] is b[k] or torch.equal(a[k], b[k]), k


# ------------------------------------------------------------------------------------------------ oracle Jacobian
@pytest.mark.parametrize('name', ['nb1_ne0', 'nb27_ne5_dense'])
def test_oracle_jacobian_vs_central_differences(name):
    """The recipe and bar of test_fit_lm_keypoints_cpu.test_oracle_jacobian_vs_central_differences at the variant's
    NB (and its own J14)."""
    model = variant_model(name)
    NB = VARIANTS[name][0]
    gen = torch.Generator().manual_seed(4)
    n_rot = 22
    P = 3 * n_rot + NB + 3
    for b, neck in enumerate((1.2, -1.2)):                 # necks turned past both ends of the contour LUT
        rot = rodrigues(torch.randn(n_rot, 3, generator=gen, dtype=torch.float64) * 0.4).float()
        rot[12] = rodrigues(torch.tensor([0.0, neck, 0.0])).float()
        betas = torch.randn(NB, generator=gen)
        transl = torch.randn(3, generator=gen) * 0.1
        kp, jac = kp_lm_oracle.keypoint_jacobian(model, betas, rot, transl)
        assert jac.shape == (3 * 123, P) and kp.shape == (123, 3)
        base = keypoints_at(model, betas, rot, transl, torch.zeros(1, P, dtype=torch.float64))[0].numpy()
        assert np.abs(kp - base).max() <= 1e-9 * np.abs(base).max()
        h = 1e-5
        fd = []
        for half in (range(0, P // 2), range(P // 2, P)):
            e = torch.zeros(2 * len(half), P, dtype=torch.float64)
            for i, c in enumerate(half):
                e[2 * i, c], e[2 * i + 1, c] = h, -h
            y = keypoints_at(model, betas, rot, transl, e).reshape(len(half), 2, -1).numpy()
            fd.append(((y[:, 0] - y[:, 1]) / (2 * h)).T)
        fd = np.concatenate(fd, 1)
        for block, cols in (('rot', slice(0, 3 * n_rot)), ('betas', slice(3 * n_rot, 3 * n_rot + NB)),
                            ('transl', slice(3 * n_rot + NB, P))):
            err = np.abs(jac[:, cols] - fd[:, cols]).max()
            assert err <= 1e-6 * np.abs(fd[:, cols]).max(), (b, block, err)


# ------------------------------------------------------------------------------------------------ oracle steps
# (n_rot, nb) -> P = 3 n_rot + nb + 3: the smallest and the largest parameter count the step kernel takes
STEP_SHAPES = {7: (1, 1), 96: (22, 27)}


def _random_step_problem(seed, n_rot, nb, K):
    """A random state of one body: rotations, betas, transl, keypoints, a (3K, P) Jacobian, targets and weights with
    a dropped keypoint whose keypoint and rows are NaN, five measurements with one dropped (NaN value and row)."""
    rng = np.random.default_rng(seed)
    P = 3 * n_rot + nb + 3
    x = {'rot': np.stack([kp_lm_oracle.exp_gram_schmidt(np.eye(3), rng.normal(size=3)) for _ in range(n_rot)]),
         'betas': rng.normal(size=nb), 'transl': rng.normal(size=3) * 0.1}
    kp, jac = rng.normal(size=(K, 3)), rng.normal(size=(3 * K, P))
    tg = kp + rng.normal(size=(K, 3)) * 0.1
    w = rng.uniform(0.5, 1.5, K)
    w[K // 2] = 0.0
    kp[K // 2], jac[3 * (K // 2):3 * (K // 2) + 3] = np.nan, np.nan
    meas, mjac = rng.uniform(0.5, 1.5, 5), rng.normal(size=(5, nb))
    mt, mw = meas + rng.normal(size=5) * 0.02, np.array([3.0, 0.0, 20.0, 10.0, 5.0])
    meas[1], mjac[1] = np.nan, np.nan
    return x, kp, jac, tg, w, meas, mjac, mt, mw


def _random_2d_problem(seed, n_rot, nb, K):
    """_random_step_problem's body seen through a weak-perspective camera: 2D targets (the projection of its 3D targets,
    NaN at the dropped keypoint), a camera [c, tx, ty] in place of transl and a pose anchor near the rotations."""
    x, kp, jac, tg, w, meas, mjac, mt, mw = _random_step_problem(seed, n_rot, nb, K)
    rng = np.random.default_rng(seed + 7)
    x['camera'] = np.array([0.4, 0.05, -0.1]) + 0.1 * rng.normal(size=3)
    del x['transl']
    tg2 = o2.project(tg, x['camera'])
    tg2[K // 2] = np.nan
    anchor = np.stack([kp_lm_oracle.exp_gram_schmidt(R, rng.normal(size=3) * 0.1) for R in x['rot']])
    return x, kp, jac, tg2, w, anchor, meas, mjac, mt, mw


def _dense(jac, kp, tg, w, o, nb, mjac=None, meas=None, mt=None, mw=None, rho=0.0, camera=None, sigma=math.inf,
           rot=None, anchor=None, pose_w=0.0):
    """A and g of the stacked weighted residual, built densely, the rows of a dropped term left out.  With a camera
    the keypoint rows are 2D: the projected rows of kp2d_lm_oracle.jacobian_2d and residuals p_k - tg_k, weighted by
    the IRLS weight w_k q_k^2, q_k = sigma^2 / (sigma^2 + |p_k - tg_k|^2); then, with pose_w > 0, the pose-prior rows
    R_j [e_a]x of rotations 1.. against the anchor, weighted pose_w / 2."""
    rows, res = [], []
    P = jac.shape[1]
    if camera is None:
        for k in range(len(w)):
            if w[k] > 0:
                for c in range(3):
                    rows.append(math.sqrt(w[k]) * jac[3 * k + c])
                    res.append(math.sqrt(w[k]) * (kp[k, c] - tg[k, c]))
    else:
        J2, p = o2.jacobian_2d(kp, jac, camera), o2.project(kp, camera)
        s2 = float(sigma) * float(sigma)
        for k in range(len(w)):
            if w[k] > 0:
                d = p[k] - tg[k]
                sw = math.sqrt(w[k]) * (s2 / (s2 + float(d @ d)) if math.isfinite(sigma) else 1.0)
                for c in range(2):
                    rows.append(sw * J2[2 * k + c])
                    res.append(sw * d[c])
        if pose_w > 0:
            sw = math.sqrt(0.5 * float(np.float32(pose_w)))
            for j in range(1, len(rot)):
                D = np.stack([o2.rot_tangent(rot[j], a) for a in range(3)], 1)       # (9, 3)
                d = (rot[j] - anchor[j]).reshape(9)
                for e in range(9):
                    row = np.zeros(P)
                    row[3 * j:3 * j + 3] = sw * D[e]
                    rows.append(row)
                    res.append(sw * d[e])
    if mjac is not None:
        for k in range(5):
            if mw[k] > 0:
                row = np.zeros(P)
                row[o:o + nb] = math.sqrt(mw[k]) * mjac[k]
                rows.append(row)
                res.append(math.sqrt(mw[k]) * (meas[k] - mt[k]))
    J, r = np.array(rows), np.array(res)
    return J.T @ J, J.T @ r, r


@pytest.mark.parametrize('P', sorted(STEP_SHAPES))
def test_oracle_keypoint_step_vs_dense_solve(P):
    n_rot, nb = STEP_SHAPES[P]
    x, kp, jac, tg, w, _, _, _, _ = _random_step_problem(P, n_rot, nb, 40)
    o = 3 * n_rot
    new, nxt, acc = kp_lm_oracle.lm_keypoints_step({}, tg, w, 10.0, 3.0, True, x, kp, jac, dtype=np.float64)
    assert acc
    A, g, r = _dense(jac, kp, tg, w, o, nb)
    lam = float(new['lambda'])
    assert lam == pytest.approx(1e-3 * max(np.diag(A).max(), 1e-6), rel=1e-12)
    assert float(new['loss']) == pytest.approx(float(r @ r), rel=1e-12)
    want = np.linalg.solve(A + lam * np.eye(P), -g)
    scale = max(1.0, np.abs(want).max())
    assert np.abs(nxt['betas'] - (x['betas'] + want[o:o + nb])).max() <= 1e-8 * scale
    assert np.abs(nxt['transl'] - (x['transl'] + want[o + nb:])).max() <= 1e-8 * scale
    for j in range(n_rot):
        R = kp_lm_oracle.exp_gram_schmidt(x['rot'][j], want[3 * j:3 * j + 3])
        assert np.abs(nxt['rot'][j] - R).max() <= 1e-8 * scale, j


@pytest.mark.parametrize('rho', [0.0, 0.05])
@pytest.mark.parametrize('P', sorted(STEP_SHAPES))
def test_oracle_keypoint_measurement_step_vs_dense_solve(P, rho):
    """As test_fit_lm_kp_meas_cpu.test_delta_solves_stacked_normal_equations, at P = 7 and P = 96; without
    measurement rows and rho the step is the keypoint step's, bit for bit."""
    n_rot, nb = STEP_SHAPES[P]
    x, kp, jac, tg, w, meas, mjac, mt, mw = _random_step_problem(P + 1, n_rot, nb, 40)
    o = 3 * n_rot
    new, _, acc, delta = kp_lm_oracle.lm_keypoints_step(
        {}, tg, w, 10.0, 3.0, True, x, kp, jac, meas=(mt, mw), trial_meas=(meas, mjac), betas_weight=rho,
        dtype=np.float64, return_delta=True)
    assert acc
    A, g, r = _dense(jac, kp, tg, w, o, nb, mjac, meas, mt, mw)
    rho32 = float(np.float32(rho))
    lam = float(new['lambda'])
    assert lam == pytest.approx(1e-3 * max(np.diag(A).max(), 1e-6), rel=1e-12)   # the first lambda leaves rho out
    A[o:o + nb, o:o + nb] += rho32 * np.eye(nb)
    g[o:o + nb] += rho32 * x['betas']
    assert float(new['loss']) == pytest.approx(float(r @ r) + rho32 * float(x['betas'] @ x['betas']), rel=1e-12)
    want = np.linalg.solve(A + lam * np.eye(P), -g)
    assert np.abs(delta - want).max() <= 1e-8 * np.abs(want).max()
    # no measurement rows, rho = 0: the keypoint step, bit for bit
    f = lambda t: np.asarray(t, np.float32)  # noqa: E731
    x32 = {k: f(v) for k, v in x.items()}
    a = kp_lm_oracle.lm_keypoints_step({}, f(tg), f(w), 10.0, 3.0, True, x32, f(kp), f(jac))
    b = kp_lm_oracle.lm_keypoints_step({}, f(tg), f(w), 10.0, 3.0, True, x32, f(kp), f(jac),
                                       meas=(f(mt), np.zeros(5, np.float32)), trial_meas=(f(meas), f(mjac)),
                                       betas_weight=0.0)
    for k in ('rot', 'betas', 'transl', 'loss', 'lambda', 'accepted'):
        assert np.array_equal(a[0][k], b[0][k]), k
    for k in ('rot', 'betas', 'transl'):
        assert np.array_equal(a[1][k], b[1][k]), k


# ------------------------------------------------------------------------------------------------ 2D oracle steps
# (n_rot, nb): P = 7 (no pose-prior rows, 1 x 1 Schur factor), 54, 55 (twice), 79 (the model's own NB) and 96; at nb > 1
# the Schur blocks have off-diagonals and every measurement row's outer product is a matrix
SHAPES_2D = [(1, 1), (8, 27), (12, 16), (17, 1), (22, 10), (22, 27)]
TERMS_2D = [(math.inf, 0.0, 0.0), (0.3, 0.5, 0.2)]          # (sigma, pose_w, betas_w)
K_2D = 60                                                   # 2K = 120 keypoint rows, more than P


def _check_step(nxt, x, want, o, nb, bar):
    """The next trial (fp64) against the step `want` over [delta | beta | c] from the state x."""
    assert np.abs(nxt['betas'] - (x['betas'] + want[o:o + nb])).max() <= bar
    assert np.abs(nxt['camera'] - (x['camera'] + want[o + nb:])).max() <= bar
    for j in range(len(x['rot'])):
        R = kp_lm_oracle.exp_gram_schmidt(x['rot'][j], want[3 * j:3 * j + 3])
        assert np.abs(nxt['rot'][j] - R).max() <= bar, j


@pytest.mark.parametrize('with_meas', [False, True], ids=['kp2d', 'kp2dm'])
@pytest.mark.parametrize('sigma,pose_w,betas_w', TERMS_2D)
@pytest.mark.parametrize('n_rot,nb', SHAPES_2D)
def test_oracle_2d_step_vs_dense_solve(n_rot, nb, sigma, pose_w, betas_w, with_meas):
    """kp2d_lm_oracle, with and without measurements: A and g are J^T W J and J^T W r of the explicitly stacked
    rows (projected keypoints with IRLS weights, pose prior, measurements) plus betas_w beta, the first lambda comes
    from the keypoint rows alone, and the fp64 step solves the damped system."""
    x, kp, jac, tg, w, anchor, meas, mjac, mt, mw = _random_2d_problem(100 * n_rot + nb, n_rot, nb, K_2D)
    o, P = 3 * n_rot, 3 * n_rot + nb + 3
    bw = float(np.float32(betas_w))
    mrows = dict(mjac=mjac, meas=meas, mt=mt, mw=mw) if with_meas else {}
    A, g, _ = _dense(jac, kp, tg, w, o, nb, camera=x['camera'], sigma=sigma, rot=x['rot'], anchor=anchor,
                     pose_w=pose_w, **mrows)
    g[o:o + nb] += bw * x['betas']
    dkp = np.diag(_dense(jac, kp, tg, w, o, nb, camera=x['camera'], sigma=sigma)[0])
    A2, g2, dg = o2.normal_equations(tg, w, kp, jac, x['camera'], sigma, x['rot'], anchor, pose_w, x['betas'],
                                     betas_w, meas=(mt, mw, meas, mjac) if with_meas else None)
    mkw = dict(meas=(mt, mw), trial_meas=(meas, mjac)) if with_meas else {}
    new, nxt, acc = o2.lm_keypoints_2d_step({}, tg, w, 10.0, 3.0, True, x, kp, jac, sigma, anchor, pose_w, betas_w,
                                            dtype=np.float64, **mkw)
    assert acc
    assert np.abs(A2 - A).max() <= 1e-12 * np.abs(A).max()
    assert np.abs(g2 - g).max() <= 1e-12 * np.abs(g).max()
    assert np.abs(dg - dkp).max() <= 1e-12 * np.abs(dkp).max()
    lam = float(new['lambda'])
    assert lam == pytest.approx(1e-3 * max(dkp.max(), kp_lm_oracle.DIAG_FLOOR), rel=1e-12)
    D = A + lam * np.eye(P)
    D[o:o + nb, o:o + nb] += bw * np.eye(nb)
    want = np.linalg.solve(D, -g)
    _check_step(nxt, x, want, o, nb, 1e-8 * max(1.0, np.abs(want).max()))


@pytest.mark.parametrize('with_meas', [False, True], ids=['kp2dg', 'kp2dgm'])
@pytest.mark.parametrize('M', [1, 2, 5])
@pytest.mark.parametrize('sigma,pose_w,betas_w', TERMS_2D)
@pytest.mark.parametrize('n_rot,nb', SHAPES_2D)
def test_oracle_groups_step_vs_dense_block_arrow_solve(n_rot, nb, sigma, pose_w, betas_w, M, with_meas):
    """kp2dg_lm_oracle on the first step of M views sharing betas: [delta_1 .. delta_M | dbeta] solves the block-arrow
    system assembled from the dense rows of every view (test_fit_lm_kp2d_groups_cpu's toy test at real sizes), each
    view's S_i, s_i, X_i, x_i are C - B^T A^-1 B, g_beta - B^T A^-1 g, A^-1 B and A^-1 g of its damped leading block A,
    and lambda is 1e-3 max(floor, the views' [delta | c] diagonal, the betas diagonal summed over the views)."""
    views = [_random_2d_problem(10000 * n_rot + 100 * nb + i, n_rot, nb, K_2D) for i in range(M)]
    x0, _, _, _, _, _, meas, mjac, mt, mw = views[0]
    betas = x0['betas']
    images = [{'targets': v[3], 'weights': v[4], 'anchor': v[5], 'trial_kp': v[1], 'trial_jac': v[2]} for v in views]
    trial = {'rot': [v[0]['rot'] for v in views], 'camera': [v[0]['camera'] for v in views], 'betas': betas}
    mb = {'targets': mt, 'weights': mw, 'trial_meas': meas, 'trial_meas_jac': mjac} if with_meas else None
    new, _, acc, blocks, db = og.lm_groups_step({}, images, 10.0, 3.0, True, trial, sigma, pose_w, betas_w, mb,
                                                dtype=np.float64)
    assert acc
    lam, bw = float(new['lambda']), float(np.float32(betas_w))
    o, n1 = 3 * n_rot, 3 * n_rot + 3
    dc, bc = list(range(o)) + [o + nb, o + nb + 1, o + nb + 2], list(range(o, o + nb))
    N = M * n1 + nb
    Af, gf = np.zeros((N, N)), np.zeros(N)
    dmax, dbeta = kp_lm_oracle.DIAG_FLOOR, np.zeros(nb)
    for i, (x, kp, jac, tg, w, anchor, *_) in enumerate(views):
        A, g, _ = _dense(jac, kp, tg, w, o, nb, camera=x['camera'], sigma=sigma, rot=x['rot'], anchor=anchor,
                         pose_w=pose_w)
        dk = np.diag(_dense(jac, kp, tg, w, o, nb, camera=x['camera'], sigma=sigma)[0])
        dmax, dbeta = max(dmax, dk[dc].max()), dbeta + dk[bc]
        A11, A12, A22 = A[np.ix_(dc, dc)] + lam * np.eye(n1), A[np.ix_(dc, bc)], A[np.ix_(bc, bc)]
        r = slice(i * n1, (i + 1) * n1)
        Af[r, r], Af[r, M * n1:], Af[M * n1:, r] = A11, A12, A12.T
        Af[M * n1:, M * n1:] += A22
        gf[r] = g[dc]
        gf[M * n1:] += g[bc]
        S, s, X, xv, ok = blocks[i]
        X64, x64 = np.linalg.solve(A11, A12), np.linalg.solve(A11, g[dc])
        assert ok
        assert np.abs(S - np.tril(A22 - A12.T @ X64)).max() <= 1e-10 * np.abs(A22).max(), i
        assert np.abs(s - (g[bc] - A12.T @ x64)).max() <= 1e-10 * np.abs(g[bc]).max(), i
        assert np.abs(X - X64).max() <= 1e-10 * np.abs(X64).max(), i
        assert np.abs(xv - x64).max() <= 1e-10 * np.abs(x64).max(), i
    if with_meas:                   # the measurement rows alone: _dense with every keypoint weight 0
        Am, gm, _ = _dense(views[0][2], views[0][1], views[0][3], np.zeros(K_2D), o, nb, mjac, meas, mt, mw)
        Af[M * n1:, M * n1:] += Am[np.ix_(bc, bc)]
        gf[M * n1:] += gm[bc]
    gf[M * n1:] += bw * betas
    Af[M * n1:, M * n1:] += (bw + lam) * np.eye(nb)
    assert lam == pytest.approx(1e-3 * max(dmax, dbeta.max()), rel=1e-12)
    want = np.linalg.solve(Af, -gf)
    got = np.concatenate([-b[3] - b[2] @ db for b in blocks] + [db])
    assert np.abs(got - want).max() <= 1e-10 * np.abs(want).max()


# ------------------------------------------------------------------------------------------------ fit arguments
def _nb28_module():
    """An SMPLX module on the CPU with NB = 28, NE = 4 (NC = 32)."""
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    m = dict(synth.make_smplx())
    g = torch.Generator().manual_seed(2800)
    m['shapedirs'] = torch.randn(m['v_template'].shape[0], 3, 28, generator=g) * 5e-3
    m['expr_dirs'] = m['expr_dirs'][:, :, :4]
    return SMPLX(data_struct=m, betas={'num': 28}, expression={'num': 4}, use_face_contour=True)


def test_lm_fit_refuses_more_than_96_parameters():
    """NB = 28 gives P = 3 * 22 + 28 + 3 = 97: a ValueError naming the limit, raised before the model is packed or any
    kernel launched (the module here is on the CPU, where either would fail)."""
    from shapy_b200.fit import fit_body_to_keypoints
    module = _nb28_module()
    kp = torch.zeros(2, 123, 3)
    with pytest.raises(ValueError, match='96'):
        fit_body_to_keypoints(module, kp, method='lm')
    assert module._packed is None


@pytest.mark.parametrize('groups', [None, [0, 1, 1]])
def test_lm_fit_2d_refuses_more_than_96_parameters(groups):
    """fit_body_to_keypoints_2d(method='lm') at NB = 28 (22 rotations, 28 betas and the camera: 97 parameters), per
    image and grouped: the same ValueError before the model is packed."""
    from shapy_b200.fit import fit_body_to_keypoints_2d
    module = _nb28_module()
    with pytest.raises(ValueError, match='96'):
        fit_body_to_keypoints_2d(module, torch.zeros(3, 123, 2), method='lm',
                                 groups=None if groups is None else torch.tensor(groups))
    assert module._packed is None
