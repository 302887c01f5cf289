"""GPU: the measurement fits with circumference_derivative='exact' on the 256-body recipes of test_gpu_fit_lm.py
(betas to all five measurements) and test_gpu_fit_lm_kp_meas.py (all keypoints and all five measurements, default
weights): every body's LM loss is non-increasing, the median final loss is no higher than with the reference rows, the
LM loops never synchronise with the host, and Adam runs with the exact gradient."""
import pytest
import torch

import lm_harness as harness
from shapy_b200 import synth

pytestmark = pytest.mark.gpu
NAMES = ('mass', 'height', 'chest', 'waist', 'hips')


@pytest.fixture(scope='module')
def model():
    from shapy_b200.body_measurements import BodyMeasurements
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    return (SMPLX(data_struct=synth.make_smplx(), use_face_contour=True).cuda(),
            BodyMeasurements({'landmarks': synth.load_landmarks()}).cuda())


def _measure(module, bm, betas):
    with torch.no_grad():
        m = bm.forward_vertices(module.forward_shape(betas=betas)['v_shaped'], module.faces_i32)['measurements']
    return torch.stack([m[k]['tensor'] for k in NAMES], 1)


def _meas_shares(meas, tgt):
    ok = torch.isfinite(tgt).all(1)
    rel = ((meas - tgt).abs() / tgt.abs())[ok]
    return {'height_1mm': float(((meas[:, 1] - tgt[:, 1]).abs()[ok] < 1e-3).float().mean()),
            'circ_0.5pct': float((rel[:, 2:] < 5e-3).all(1).float().mean()),
            'mass_1pct': float((rel[:, 0] < 1e-2).float().mean())}


# Shares of the 256 bodies after 50 LM iterations with exact rows, set just below the first run on an H100 80GB HBM3
# (700 W).  First run, exact / reference rows: betas to measurements height 0.116 / 0.112, circumferences 0.307 / 0.255,
# mass 0.853 / 0.661, median loss 1.16 / 6.47; keypoints + measurements keypoint RMS 0.043 / 0.027, height 0.091 /
# 0.067, circumferences 0.206 / 0.127, mass 0.849 / 0.694, median loss 9.27 / 10.77 (keypoints only: 0.395, 0.448,
# 0.393, 0.849).
BETAS_BARS = {'height_1mm': 0.11, 'circ_0.5pct': 0.29, 'mass_1pct': 0.83}
KP_BARS = {'kp_rms_1cm': 0.04, 'height_1mm': 0.085, 'circ_0.5pct': 0.19, 'mass_1pct': 0.83}


def _betas_targets(module, bm, B, seed=21):
    """test_gpu_fit_lm._targets: betas N(0, 1) clipped to +-2 (seed 21), their five measurements."""
    bstar = torch.randn(B, 10, generator=torch.Generator().manual_seed(seed)).clamp(-2, 2).cuda()
    m = _measure(module, bm, bstar)
    return {k: m[:, i].clone() for i, k in enumerate(NAMES)}


def test_betas_lm_exact_256_bodies(model):
    from shapy_b200.fit import fit_betas_to_measurements
    module, bm = model
    tg = _betas_targets(module, bm, 256)
    tgt = torch.stack([tg[k] for k in NAMES], 1)
    ok = torch.isfinite(tgt).all(1)
    fit = lambda **kw: fit_betas_to_measurements(module, bm, tg, **kw)  # noqa: E731
    ex = fit(method='lm', iterations=50, circumference_derivative='exact')
    ref = fit(method='lm', iterations=50)
    start = fit(method='lm', iterations=0, circumference_derivative='exact')['loss']
    adam = fit(iterations=400, circumference_derivative='exact')
    adam_ref = fit(iterations=400)
    med = {k: float(r['loss'][ok].median()) for k, r in (('lm_exact', ex), ('lm_reference', ref),
                                                          ('adam_exact', adam), ('adam_reference', adam_ref))}
    sh = {k: _meas_shares(r['measurements'], tgt) for k, r in (('lm_exact', ex), ('lm_reference', ref),
                                                               ('adam_exact', adam), ('adam_reference', adam_ref))}
    print('fit_betas_exact_256 median loss', med, 'shares', sh)
    fin = torch.isfinite(start)
    assert bool((ex['loss'][fin] <= start[fin]).all())
    assert med['lm_exact'] <= med['lm_reference']
    assert bool(torch.isfinite(adam['loss'][ok]).all())
    assert all(sh['lm_exact'][k] >= BETAS_BARS[k] for k in BETAS_BARS), sh['lm_exact']


def _kp_targets(module, bm, B, seed=31):
    """test_gpu_fit_lm_kp_meas._targets."""
    from shapy_b200 import ops
    gen = torch.Generator().manual_seed(seed)
    bstar = torch.randn(B, 10, generator=gen).clamp(-2, 2)
    raw = synth.mean_params()[:132] + 0.3 * torch.randn(B, 132, generator=gen)
    with torch.no_grad():
        rot = ops.decode_rot6d(raw.cuda())
        kp = module(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=bstar.cuda())['joints'][:].clone()
    m = _measure(module, bm, bstar.cuda())
    return kp, {k: m[:, i].clone() for i, k in enumerate(NAMES)}


def _init(B):
    mean = synth.mean_params().cuda()
    return {'global_rot': mean[:6].expand(B, 6), 'body_pose': mean[6:132].expand(B, 126)}


def _kp_fit(module, kp, init=None, **kw):
    from shapy_b200.fit import fit_body_to_keypoints
    return fit_body_to_keypoints(module, kp, init=init or _init(kp.shape[0]), **kw)


def test_keypoints_and_measurements_lm_exact_256_bodies(model):
    module, bm = model
    kp, tg = _kp_targets(module, bm, 256)
    tgt = torch.stack([tg[k] for k in NAMES], 1)
    kw = dict(body_measurements=bm, measurements=tg)
    ex = _kp_fit(module, kp, method='lm', circumference_derivative='exact', **kw)
    ref = _kp_fit(module, kp, method='lm', **kw)
    kpo = _kp_fit(module, kp, method='lm')
    start = _kp_fit(module, kp, method='lm', iterations=0, circumference_derivative='exact', **kw)['loss']
    adam = _kp_fit(module, kp, circumference_derivative='exact', **kw)
    adam_ref = _kp_fit(module, kp, **kw)
    res = {'lm_exact': ex, 'lm_reference': ref, 'lm_keypoints_only': kpo, 'adam_exact': adam, 'adam_reference': adam_ref}
    sh = {}
    for k, r in res.items():
        rms = (r['keypoints'] - kp).pow(2).sum(-1).mean(1).sqrt()
        sh[k] = dict(kp_rms_1cm=float((rms < 1e-2).float().mean()),
                     **_meas_shares(r['measurements'] if 'measurements' in r else _measure(module, bm, r['betas']), tgt))
    med = {k: float(r['loss'].median()) for k, r in res.items() if k != 'lm_keypoints_only'}
    print('fit_kp_meas_exact_256 median loss', med, 'shares', sh)
    fin = torch.isfinite(start)
    assert bool((ex['loss'][fin] <= start[fin]).all())
    assert med['lm_exact'] <= med['lm_reference']
    assert bool(torch.isfinite(adam['loss']).any())
    assert all(sh['lm_exact'][k] >= KP_BARS[k] for k in KP_BARS), sh['lm_exact']


def test_lm_loops_never_synchronise(model):
    from shapy_b200.fit import fit_betas_to_measurements
    module, bm = model
    kp, tg = _kp_targets(module, bm, 32)
    kw = dict(method='lm', body_measurements=bm, measurements=tg, betas_weight=0.01, circumference_derivative='exact',
              init=_init(32))                                 # on the device before the check: no copy in the loop
    _kp_fit(module, kp, iterations=1, **kw)                 # packs the model, builds the incidence table
    fit_betas_to_measurements(module, bm, tg, method='lm', iterations=1, circumference_derivative='exact')
    _, (res, res2) = harness.launches_without_sync(lambda: (
        _kp_fit(module, kp, iterations=3, **kw),
        fit_betas_to_measurements(module, bm, tg, method='lm', iterations=3, circumference_derivative='exact')))
    assert res['measurements'].shape == (32, 5) and res2['betas'].shape == (32, 10)


def test_same_launch_count_as_reference_rows(model):
    from shapy_b200 import _lib
    from shapy_b200.fit import fit_betas_to_measurements, measurement_jacobian
    module, bm = model
    kp, tg = _kp_targets(module, bm, 8)
    counts = {}
    for cd in ('reference', 'exact'):
        _kp_fit(module, kp, method='lm', iterations=1, body_measurements=bm, measurements=tg,
                circumference_derivative=cd)
        torch.cuda.synchronize()
        n0 = _lib.lib().shapy_launch_count()
        _kp_fit(module, kp, method='lm', iterations=4, body_measurements=bm, measurements=tg,
                circumference_derivative=cd)
        n1 = _lib.lib().shapy_launch_count()
        fit_betas_to_measurements(module, bm, tg, method='lm', iterations=4, circumference_derivative=cd)
        counts[cd] = (n1 - n0, _lib.lib().shapy_launch_count() - n1)
    assert counts['reference'] == counts['exact'], counts
    j = measurement_jacobian(module, bm, torch.zeros(2, 10, device='cuda'), circumference_derivative='exact')
    r = measurement_jacobian(module, bm, torch.zeros(2, 10, device='cuda'))
    assert torch.equal(j['measurements'], r['measurements']) and torch.equal(j['jacobian'][:, :2], r['jacobian'][:, :2])
    with pytest.raises(ValueError):
        measurement_jacobian(module, bm, torch.zeros(2, 10, device='cuda'), circumference_derivative='fd')


def test_cli_exact(tmp_path):
    import numpy as np
    from shapy_b200 import fit
    out = tmp_path / 'fit.npz'
    fit.main(['--synthetic', '--method', 'lm', '--iterations', '3', '--height', '1.7', '--chest', '0.95',
              '--circumference-derivative', 'exact', '--output', str(out)])
    d = np.load(out)
    assert d['betas'].shape == (1, 10) and np.isfinite(d['loss']).all()
