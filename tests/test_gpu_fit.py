"""GPU: the shape-blend backward (shapy_smplx_backward_shape), the chained betas -> measurements gradient, and the
batched fit of shapy_b200.fit."""
import numpy as np
import pytest
import torch

from shapy_b200 import synth

pytestmark = pytest.mark.gpu
NAMES = ('mass', 'height', 'chest', 'waist', 'hips')


@pytest.fixture(scope='module')
def model():
    from shapy_b200.body_measurements import BodyMeasurements
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    return SMPLX(data_struct=synth.make_smplx()).cuda(), BodyMeasurements({'landmarks': synth.load_landmarks()}).cuda()


def _generic(nb):
    d = dict(synth.make_smplx())
    rng = torch.Generator().manual_seed(nb)
    d['shapedirs'] = torch.randn(d['shapedirs'].shape[0], 3, nb, generator=rng) * 0.01
    return d


@pytest.mark.parametrize('nb', [10, 7])
@pytest.mark.parametrize('B', [1, 64, 4096])
def test_shape_backward_vs_float64(nb, B):
    from shapy_b200 import ops
    d = synth.make_smplx() if nb == 10 else _generic(nb)
    packed = ops.SmplxModel(dict(d), 'cuda')
    g = torch.randn(B, packed.V, 3, generator=torch.Generator().manual_seed(B)).cuda()
    out = ops.smplx_backward_shape(packed, g)
    S = d['shapedirs'].double().cuda()                       # (V, 3, NB)
    ref = torch.einsum('vcl,bvc->bl', S, g.double())
    scale = torch.einsum('vcl,bvc->bl', S.abs(), g.double().abs())
    assert ((out.double() - ref).abs() <= 1e-5 * scale + 1e-30).all()
    if B == 64:                                              # deterministic, a body alone equals it in the batch
        assert torch.equal(out, ops.smplx_backward_shape(packed, g))
        assert torch.equal(out[17:18], ops.smplx_backward_shape(packed, g[17:18].contiguous()))


def test_chain_gradient_vs_central_differences(model):
    """betas -> v_shaped -> (mass, height): smooth, and there the reference semantics are the true derivative."""
    smplx, bm = model
    betas = (torch.randn(4, 10, generator=torch.Generator().manual_seed(5)) * 0.5).cuda().requires_grad_(True)
    m = bm.forward_vertices(smplx.forward_shape(betas=betas)['v_shaped'], smplx.faces_i32)['measurements']
    (m['mass']['tensor'].sum() + 10.0 * m['height']['tensor'].sum()).backward()
    # float64 restatement of the forward for the differences
    from oracle import measure_oracle
    vt = smplx.v_template.double().cpu().numpy()
    S = smplx.shapedirs.double().cpu().numpy()
    faces = smplx.faces
    lm = synth.load_landmarks()

    def f(b):
        v = vt + S @ b
        t = v[faces]
        x, y, z = t[..., 0], t[..., 1], t[..., 2]
        vol = (-x[:, 2] * y[:, 1] * z[:, 0] + x[:, 1] * y[:, 2] * z[:, 0] + x[:, 2] * y[:, 0] * z[:, 1]
               - x[:, 0] * y[:, 2] * z[:, 1] - x[:, 1] * y[:, 0] * z[:, 2] + x[:, 0] * y[:, 1] * z[:, 2])
        mass = abs(vol.sum()) / 6 * measure_oracle.DENSITY
        hy = [(t[lm[k]['face_idx'], :, 1] * np.asarray(lm[k]['bc'])).sum() for k in ('head_top', 'left_heel')]
        return mass + 10.0 * abs(hy[0] - hy[1])
    bn = betas.detach().double().cpu().numpy()
    for i in range(4):
        fd = np.array([(f(bn[i] + 1e-4 * e) - f(bn[i] - 1e-4 * e)) / 2e-4 for e in np.eye(10)])
        got = betas.grad[i].double().cpu().numpy()
        assert np.abs(got - fd).max() <= 1e-3 * np.abs(fd).max(), (i, got, fd)


FIT = {}
# Fractions of the 256 bodies within the suggested bars (height < 1 mm, every circumference < 0.5 %, mass < 1 %),
# set from the first run on an H100 80GB HBM3 (700 W): 0.052, 0.143, 0.550 after 400 Adam iterations.  The seeded
# synthetic basis is white noise per vertex, so its measurements are far rougher functions of beta than a real
# SMPL-X model's; these bars guard against regressions, they do not claim the 95 % the real model may reach.
BARS = {'height_1mm': 0.04, 'circ_0.5pct': 0.12, 'mass_1pct': 0.5}


def _fit(model, B, seed=21, iterations=400):
    from shapy_b200.fit import fit_betas_to_measurements
    smplx, bm = model
    bstar = torch.randn(B, 10, generator=torch.Generator().manual_seed(seed)).clamp(-2, 2).cuda()
    with torch.no_grad():
        m = bm.forward_vertices(smplx.forward_shape(betas=bstar)['v_shaped'], smplx.faces_i32)['measurements']
        tg = {k: m[k]['tensor'].clone() for k in NAMES}
    return tg, fit_betas_to_measurements(smplx, bm, tg, iterations=iterations)


def test_fit_256_bodies(model):
    tg, res = _fit(model, 256)
    meas = res['measurements']
    tgt = torch.stack([tg[k] for k in NAMES], 1)
    ok = torch.isfinite(tgt).all(1)
    rel = ((meas - tgt).abs() / tgt.abs())[ok]
    height_err = (meas[:, 1] - tgt[:, 1]).abs()[ok]
    frac = {'height_1mm': float((height_err < 1e-3).float().mean()),
            'circ_0.5pct': float((rel[:, 2:] < 5e-3).all(1).float().mean()),
            'mass_1pct': float((rel[:, 0] < 1e-2).float().mean())}
    print('fit_256', frac, 'finite targets', int(ok.sum()))
    assert int(ok.sum()) >= 240
    FIT['res'] = res
    assert all(frac[k] >= BARS[k] for k in BARS), frac
    # the fit moves every body towards its targets: the median loss falls by > 10x from beta = 0
    start = _fit(model, 256, iterations=0)[1]['loss'][ok]
    assert float(res['loss'][ok].median()) < 0.1 * float(start.median())


def test_fit_8_bodies_alone_equal_their_batch_rows(model):
    from shapy_b200.fit import fit_betas_to_measurements
    if 'res' not in FIT:
        pytest.skip('needs test_fit_256_bodies')
    tg, _ = _fit(model, 256, iterations=0)
    rows = [3, 40, 77, 101, 150, 199, 230, 255]
    sub = {k: v[rows].contiguous() for k, v in tg.items()}
    res8 = fit_betas_to_measurements(model[0], model[1], sub, iterations=400)
    assert torch.equal(res8['betas'], FIT['res']['betas'][rows])
