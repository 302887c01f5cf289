"""GPU: the stacked keypoint + measurement Levenberg-Marquardt step (shapy_fit_lm_keypoints_measurements_step) against
its NumPy restatement (tests/kp_lm_oracle.py with `meas`) and against shapy_fit_lm_keypoints_step when the measurement block is
empty; and fit_body_to_keypoints with measurements (LM and Adam) against the keypoint-only LM fit."""
import numpy as np
import pytest
import torch

import kp_lm_oracle
import lm_harness as harness
from lm_harness import bits, rodrigues
from shapy_b200 import synth

pytestmark = pytest.mark.gpu
NAMES, N_ROT = harness.NAMES, harness.N_ROT


@pytest.fixture(scope='module')
def model():
    return harness.smplx_and_measurements()


def _evaluate(packed, lm, faces, rot, betas, transl):
    from shapy_b200 import ops
    c = lambda t: t.cuda().contiguous()  # noqa: E731
    kp, jac = ops.smplx_keypoint_jacobian(packed, c(betas), c(rot), c(transl))
    meas, mjac, _ = ops.measure_jacobian_betas(packed, lm, ops.smplx_forward_shape(packed, c(betas)), faces)
    return [t.cpu() for t in (kp, jac, meas, mjac)]


# ------------------------------------------------------------------------------------------------ step
def _step_case(model):
    """Eight bodies: the state at one pose and shape, the trial at a nearby one.  Body 0 targets the trial (accepted),
    1 the state (rejected), 2 the trial with a dropped measurement whose value and row are NaN in state and trial
    (accepted), 3 a weighted NaN trial measurement (rejected), 4 a non-finite start (NaN state loss, a NaN weighted
    trial keypoint), 5 to 7 random targets."""
    from shapy_b200 import ops
    smplx, bm = model
    packed, faces, lm = smplx.packed(), smplx.faces_i32, bm.landmarks()
    B = 8
    gen = torch.Generator().manual_seed(41)
    rot = rodrigues(torch.randn(B, N_ROT, 3, generator=gen, dtype=torch.float64) * 0.3).float()
    betas = torch.randn(B, 10, generator=gen).clamp(-2, 2)
    transl = torch.randn(B, 3, generator=gen) * 0.1
    trot = (rot.double() @ rodrigues(torch.randn(B, N_ROT, 3, generator=gen, dtype=torch.float64) * 0.02)).float()
    tbetas = betas + 0.05 * torch.randn(B, 10, generator=gen)
    ttransl = transl + 0.01 * torch.randn(B, 3, generator=gen)
    ttransl[1] += 0.05                                          # body 1's trial clearly worse, whatever rho
    kp, jac, meas, mjac = _evaluate(packed, lm, faces, rot, betas, transl)
    tkp, tjac, tmeas, tmjac = _evaluate(packed, lm, faces, trot, tbetas, ttransl)
    K = packed.K
    tg = kp + 0.05 * torch.randn(B, K, 3, generator=gen)
    mt = tmeas * (1 + 0.02 * torch.randn(B, 5, generator=gen))
    for b in (0, 2, 3):
        tg[b], mt[b] = tkp[b], tmeas[b]
    tg[1], mt[1] = kp[1], meas[1]
    w = torch.rand(B, K, generator=gen) + 0.5
    mw = torch.tensor([1.0, 100.0, 2000.0, 1000.0, 1000.0]).repeat(B, 1)
    mw[2, 2] = 0.0
    for t in (meas, tmeas):
        t[2, 2] = float('nan')
    for t in (mjac, tmjac):
        t[2, 2] = float('nan')
    tmeas[3, 3] = float('nan')
    tkp[4, 7, 0] = float('nan')
    return dict(rot=rot, betas=betas, transl=transl, kp=kp, jac=jac, meas=meas, mjac=mjac, trot=trot, tbetas=tbetas,
                ttransl=ttransl, tkp=tkp, tjac=tjac, tmeas=tmeas, tmjac=tmjac, tg=tg, w=w, mt=mt, mw=mw,
                lam=torch.rand(B, generator=gen) + 0.01)


def _state(c, rho):
    B = c['rot'].shape[0]
    loss = torch.tensor([kp_lm_oracle.loss(c['tg'][b].numpy(), c['w'][b].numpy(), c['kp'][b].numpy(),
                                           (c['mt'][b].numpy(), c['mw'][b].numpy(), c['meas'][b].numpy()),
                                           c['betas'][b].numpy(), rho)
                         for b in range(B)]).float()
    loss[4] = float('nan')
    cu = lambda t: t.cuda().contiguous()  # noqa: E731
    state = {'rot': cu(c['rot']), 'betas': cu(c['betas']), 'transl': cu(c['transl']), 'keypoints': cu(c['kp']),
             'jac': cu(c['jac']), 'meas': cu(c['meas']), 'meas_jac': cu(c['mjac']), 'loss': cu(loss),
             'lambda': cu(c['lam']), 'accepted': torch.zeros(B, dtype=torch.int32, device='cuda')}
    trial = {'rot': cu(c['trot']), 'betas': cu(c['tbetas']), 'transl': cu(c['ttransl'])}
    return state, trial


@pytest.mark.parametrize('rho', [0.0, 0.05])
@pytest.mark.parametrize('first', [False, True])
def test_step_kernel_vs_oracle(model, first, rho):
    from shapy_b200 import ops
    c = _step_case(model)
    B = c['rot'].shape[0]
    state, trial = _state(c, rho)
    s0 = {k: v.cpu().numpy() for k, v in state.items()}
    cu = lambda t: t.cuda().contiguous()  # noqa: E731
    ops.fit_lm_keypoints_measurements_step(state, trial, cu(c['tg']), cu(c['w']), cu(c['mt']), cu(c['mw']), rho, 10.0,
                                           3.0, first, cu(c['tkp']), cu(c['tjac']), cu(c['tmeas']), cu(c['tmjac']))
    n = lambda t: t.numpy()  # noqa: E731
    oracle = []
    for b in range(B):
        s = {k: s0[k][b] for k in s0}
        s['accepted'] = 0
        tr = {'rot': n(c['trot'][b]), 'betas': n(c['tbetas'][b]), 'transl': n(c['ttransl'][b])}
        oracle.append(kp_lm_oracle.lm_keypoints_step(
            s, n(c['tg'][b]), n(c['w'][b]), 10.0, 3.0, first, tr, n(c['tkp'][b]), n(c['tjac'][b]),
            meas=(n(c['mt'][b]), n(c['mw'][b])), trial_meas=(n(c['tmeas'][b]), n(c['tmjac'][b])), betas_weight=rho))
    got, nxt = harness.numpy_of(state), harness.numpy_of(trial)
    keys = ('rot', 'betas', 'transl')
    flags, _ = harness.check_step(harness.rows_of(got, B), harness.rows_of(nxt, B), oracle,
                             keys + ('keypoints', 'jac', 'meas', 'meas_jac'), keys, exact=True)
    if first:
        assert all(flags) and np.isnan(got['loss'][4])
    else:
        assert flags[:5] == [True, False, True, False, False], flags
    for k in ('rot', 'betas', 'transl'):              # the non-finite body does not move
        src = c['t' + k][4] if first else c[k][4]
        assert np.array_equal(nxt[k][4], src.numpy()), k


@pytest.mark.parametrize('first', [False, True])
def test_empty_measurement_block_equals_keypoint_step(model, first):
    """Every measurement weight 0 (NaN measurements and rows) and rho = 0: torch.equal to shapy_fit_lm_keypoints_step
    on state and trial."""
    from shapy_b200 import ops
    c = _step_case(model)
    for k in ('meas', 'tmeas', 'mjac', 'tmjac'):
        c[k][:] = float('nan')
    c['mw'][:] = 0.0
    a_state, a_trial = _state(c, 0.0)
    b_state = {k: v.clone() for k, v in a_state.items()}
    b_trial = {k: v.clone() for k, v in a_trial.items()}
    cu = lambda t: t.cuda().contiguous()  # noqa: E731
    ops.fit_lm_keypoints_measurements_step(a_state, a_trial, cu(c['tg']), cu(c['w']), cu(c['mt']), cu(c['mw']), 0.0,
                                           10.0, 3.0, first, cu(c['tkp']), cu(c['tjac']), cu(c['tmeas']),
                                           cu(c['tmjac']))
    ops.fit_lm_keypoints_step(b_state, b_trial, cu(c['tg']), cu(c['w']), 10.0, 3.0, first, cu(c['tkp']), cu(c['tjac']))
    for k in ('rot', 'betas', 'transl', 'keypoints', 'jac', 'loss', 'lambda', 'accepted'):
        assert torch.equal(bits(a_state[k]), bits(b_state[k])), k
    for k in ('rot', 'betas', 'transl'):
        assert torch.equal(bits(a_trial[k]), bits(b_trial[k])), k


# ------------------------------------------------------------------------------------------------ fit
FITS = {}
# Shares of the 256 bodies after 50 LM iterations with known height and mass (test_fit_quality_256_bodies), set just
# below the first run on an H100 80GB HBM3 (700 W).  First run, combined / keypoint-only: all keypoints 0.410 / 0.395
# within 1 cm RMS, height 0.480 / 0.448, circumferences 0.405 / 0.393, mass 1.0 / 0.849, median |beta - beta*| 2.32 /
# 2.48; body joints 0.992 / 0.996, 1.0 / 0.413, 0.175 / 0.099, 1.0 / 0.988, 0.41 / 0.51.
BARS = {'all': {'kp_rms_1cm': 0.39, 'height_1mm': 0.46, 'circ_0.5pct': 0.38, 'mass_1pct': 0.98},
        'body': {'kp_rms_1cm': 0.97, 'height_1mm': 0.98, 'circ_0.5pct': 0.15, 'mass_1pct': 0.98}}


def _targets(module, bm, B, seed=31):
    """The recipe of test_gpu_fit_lm_keypoints._targets (seed 31, betas clipped to +-2, raw pose = mean + 0.3 N(0, 1)),
    plus the measurements of the generating betas."""
    from shapy_b200 import ops
    gen = torch.Generator().manual_seed(seed)
    bstar = torch.randn(B, 10, generator=gen).clamp(-2, 2)
    raw = synth.mean_params()[:132] + 0.3 * torch.randn(B, 132, generator=gen)
    with torch.no_grad():
        rot = ops.decode_rot6d(raw.cuda())
        kp = module(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=bstar.cuda())['joints'][:].clone()
        m = bm.forward_vertices(module.forward_shape(betas=bstar.cuda())['v_shaped'], module.faces_i32)['measurements']
    return kp, {k: m[k]['tensor'].clone() for k in NAMES}, bstar.cuda()


def _weights(module, K, which):
    w = torch.ones(K, device='cuda')
    if which == 'body':                       # only the posed skeleton joints of the 22 fitted rotations
        w[N_ROT:] = 0.0
    return w


def _fit(module, kp, **kw):
    from shapy_b200.fit import fit_body_to_keypoints
    mean = synth.mean_params()
    B = kp.shape[0]
    init = {'global_rot': mean[:6].expand(B, 6), 'body_pose': mean[6:132].expand(B, 126)}
    return fit_body_to_keypoints(module, kp, init=init, **kw)


def _shares(res, meas, kp, w, tgt, bstar):
    ok = torch.isfinite(tgt).all(1)
    rms = ((res['keypoints'] - kp).pow(2).sum(-1) * w).sum(1).div(w.sum()).sqrt()
    rel = ((meas - tgt).abs() / tgt.abs())[ok]
    return {'kp_rms_1cm': float((rms < 1e-2).float().mean()),
            'height_1mm': float(((meas[:, 1] - tgt[:, 1]).abs()[ok] < 1e-3).float().mean()),
            'circ_0.5pct': float((rel[:, 2:] < 5e-3).all(1).float().mean()),
            'mass_1pct': float((rel[:, 0] < 1e-2).float().mean()),
            'median_beta_err': float((res['betas'] - bstar).norm(dim=1).median())}


@pytest.mark.parametrize('which', ['all', 'body'])
def test_fit_quality_256_bodies(model, which):
    """Known height and mass (the rows with exact Jacobians) with all keypoints or only the 22 body joints.  With the
    three circumferences at their default weights too, LM stalls (lambda reaches its 1e9 clamp) because their rows
    leave out the motion of the slicing planes; test_adam_runs_and_lm_beats_it covers that case."""
    module, bm = model
    kp, tg, bstar = _targets(module, bm, 256)
    tgt = torch.stack([tg[k] for k in NAMES], 1)
    w = _weights(module, kp.shape[1], which)
    kw = dict(body_measurements=bm, measurements={k: tg[k] for k in ('height', 'mass')})
    comb = _fit(module, kp, weights=w, method='lm', **kw)
    kpo = _fit(module, kp, weights=w, method='lm')
    start = _fit(module, kp, weights=w, method='lm', iterations=0, **kw)['loss']
    FITS[which] = (kp, kw['measurements'], w, comb)
    sc = _shares(comb, comb['measurements'], kp, w, tgt, bstar)
    sk = _shares(kpo, harness.measure(module, bm, kpo['betas']), kp, w, tgt, bstar)
    print(f'fit_kp_meas_lm_256[{which}]', {'combined': sc, 'keypoints_only': sk,
                                            'median_loss': float(comb['loss'].median()),
                                            'median_start': float(start.median())})
    fin = torch.isfinite(start)
    assert bool((comb['loss'][fin] <= start[fin]).all())
    for k in ('height_1mm', 'circ_0.5pct', 'mass_1pct'):
        assert sc[k] > sk[k], (k, sc[k], sk[k])
    assert all(sc[k] >= BARS[which][k] for k in BARS[which]), sc
    # the returned measurements are those of the returned betas
    torch.testing.assert_close(comb['measurements'], harness.measure(module, bm, comb['betas']), rtol=1e-6, atol=1e-7,
                               equal_nan=True)


def test_adam_runs_and_lm_beats_it(model):
    """All keypoints and all five measurements at their default weights.  First run on an H100 80GB HBM3 (700 W):
    median loss LM(50) 10.77, Adam(600) 12.34, from 197.2."""
    module, bm = model
    kp, tg, _ = _targets(module, bm, 256)
    kw = dict(body_measurements=bm, measurements=tg)
    lm = _fit(module, kp, method='lm', **kw)
    adam = _fit(module, kp, **kw)
    start = _fit(module, kp, method='lm', iterations=0, **kw)['loss']
    assert adam['measurements'].shape == (256, 5) and bool(torch.isfinite(adam['loss']).any())
    med = {'lm': float(lm['loss'].median()), 'adam': float(adam['loss'].median()), 'start': float(start.median())}
    print('fit_kp_meas_256 median loss', med)
    fin = torch.isfinite(start)
    assert bool((lm['loss'][fin] <= start[fin]).all())
    assert med['lm'] < med['adam']


def test_lm_fit_8_bodies_alone_equal_their_batch_rows(model):
    module, bm = model
    if 'all' not in FITS:
        pytest.skip('needs test_fit_quality_256_bodies[all]')
    kp, tg, w, lm = FITS['all']
    rows = [3, 40, 77, 101, 150, 199, 230, 255]
    res8 = _fit(module, kp[rows].contiguous(), weights=w, method='lm', body_measurements=bm,
                measurements={k: v[rows].contiguous() for k, v in tg.items()})
    for k in ('global_rot', 'body_pose', 'betas', 'transl', 'measurements'):
        assert torch.equal(bits(res8[k]), bits(lm[k][rows])), k


def test_lm_loop_never_synchronises(model):
    module, bm = model
    from shapy_b200.fit import fit_body_to_keypoints
    kp, tg, _ = _targets(module, bm, 32)
    mean = synth.mean_params().cuda()
    init = {'global_rot': mean[:6].expand(32, 6), 'body_pose': mean[6:132].expand(32, 126)}
    kw = dict(init=init, method='lm', body_measurements=bm, measurements=tg, betas_weight=0.01)
    fit_body_to_keypoints(module, kp, iterations=1, **kw)      # packs the model, builds the incidence table
    _, res = harness.launches_without_sync(lambda: fit_body_to_keypoints(module, kp, iterations=3, **kw))
    assert res['measurements'].shape == (32, 5)


def test_argument_errors_and_empty_batch(model):
    from shapy_b200 import _lib, ops
    module, bm = model
    L = _lib.lib()
    packed = module.packed()
    K = packed.K
    z = lambda *s: torch.zeros(*s, device='cuda')  # noqa: E731
    kp, tg, _ = _targets(module, bm, 4)
    with pytest.raises(ValueError):
        _fit(module, kp, method='lm', measurements=tg)                           # no body_measurements
    with pytest.raises(ValueError):
        _fit(module, kp, method='lm', body_measurements=bm, measurements={'height': z(3) + 1.7})
    for m in ('lm', 'adam'):
        with pytest.raises(ValueError):
            _fit(module, kp, method=m, betas_weight=0.1)                         # no prior without measurements
    torch.cuda.synchronize()
    n0 = L.shapy_launch_count()

    def step(B, n_rot, nb, null=False, rho=0.0, up=10.0):
        P = 3 * n_rot + nb + 3
        p = [_lib.ptr(t) for t in (z(B, n_rot, 3, 3), z(B, nb), z(B, 3), z(B, K, 3), z(B, 3 * K, P), z(B, 5),
                                   z(B, 5, nb), z(B), z(B), torch.zeros(B, dtype=torch.int32, device='cuda'))]
        if null:
            p[6] = None
        return L.shapy_fit_lm_keypoints_measurements_step(
            B, K, n_rot, nb, _lib.ptr(z(B, K, 3)), _lib.ptr(z(B, K)), _lib.ptr(z(B, 5)), _lib.ptr(z(B, 5)), rho, up,
            3.0, 1, *p, _lib.ptr(z(B, n_rot, 3, 3)), _lib.ptr(z(B, nb)), _lib.ptr(z(B, 3)), _lib.ptr(z(B, K, 3)),
            _lib.ptr(z(B, 3 * K, P)), _lib.ptr(z(B, 5)), _lib.ptr(z(B, 5, nb)), None)
    assert step(2, 30, 10) == -3                    # P = 103 > 96
    assert step(2, 22, 10, null=True) == -1
    assert step(2, 22, 10, rho=-0.1) == -1
    assert step(2, 22, 10, up=0.5) == -1
    st = {'rot': z(0, 22, 3, 3), 'betas': z(0, 10), 'transl': z(0, 3), 'keypoints': z(0, K, 3), 'jac': z(0, 3 * K, 79),
          'meas': z(0, 5), 'meas_jac': z(0, 5, 10), 'loss': z(0), 'lambda': z(0),
          'accepted': torch.zeros(0, dtype=torch.int32, device='cuda')}
    ops.fit_lm_keypoints_measurements_step(st, {'rot': z(0, 22, 3, 3), 'betas': z(0, 10), 'transl': z(0, 3)},
                                           z(0, K, 3), z(0, K), z(0, 5), z(0, 5), 0.0, 10.0, 3.0, True, z(0, K, 3),
                                           z(0, 3 * K, 79), z(0, 5), z(0, 5, 10))
    assert L.shapy_launch_count() == n0
