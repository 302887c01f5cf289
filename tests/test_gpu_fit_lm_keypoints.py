"""GPU: the keypoint Jacobian (shapy_smplx_keypoint_jacobian) against the float64 closed form (tests/kp_lm_oracle.py,
itself pinned to central differences of the float64 forward by tests/test_fit_lm_keypoints_cpu.py), against the posed
backward and the forward; the keypoint Levenberg-Marquardt step (shapy_fit_lm_keypoints_step) against its NumPy
restatement; and fit_body_to_keypoints(method='lm') against Adam.

Bar of the Jacobian checks: per body and per column block (rotations, betas), max |J - J64| <= 1e-4 max |J64|."""
import numpy as np
import pytest
import torch

import kp_lm_oracle
import lm_harness as harness
from lm_harness import bits, rodrigues
from shapy_b200 import synth

pytestmark = pytest.mark.gpu
TOL = 1e-4
# Keypoints of the Jacobian launch (fp32 SIMT pose blend) against shapy_smplx_forward's joints + transl (split-fp16
# GEMM pose blend): max |difference| <= KP_TOL max |keypoint| per body.  First run on an H100 80GB HBM3 (700 W),
# 256 bodies: 9.2e-7.
KP_TOL = 2e-6


def _inputs(seed, B, n_rot):
    gen = torch.Generator().manual_seed(seed)
    rot = rodrigues(torch.randn(B, n_rot, 3, generator=gen, dtype=torch.float64) * 0.4).float()
    if n_rot > 15 and B > 1:                                 # necks turned past both ends of the contour LUT
        rot[0, 12] = rodrigues(torch.tensor([0.0, 1.2, 0.0])).float()
        rot[1, 12] = rodrigues(torch.tensor([0.0, -1.2, 0.0])).float()
    return rot, torch.randn(B, 10, generator=gen), torch.randn(B, 3, generator=gen) * 0.1


def _model(variant):
    m = dict(synth.make_smplx())
    if variant == 'no_contour_no_j14':
        for k in ('extra_joint_regressor', 'source_idxs', 'target_idxs'):
            m.pop(k)
        m['use_face_contour'] = False
    return m


def _blocks(n_rot):
    return (('rot', slice(0, 3 * n_rot)), ('betas', slice(3 * n_rot, 3 * n_rot + 10)))


@pytest.mark.parametrize('variant', ['full', 'no_contour_no_j14'])
@pytest.mark.parametrize('n_rot', [1, 22, 55])
@pytest.mark.parametrize('B', [1, 64])
def test_jacobian_vs_float64(B, n_rot, variant):
    from shapy_b200 import ops
    m = _model(variant)
    packed = ops.SmplxModel(dict(m), 'cuda')
    rot, betas, transl = _inputs(100 * n_rot + B, B, n_rot)
    kp, jac = ops.smplx_keypoint_jacobian(packed, betas.cuda(), rot.cuda(), transl.cuda())
    assert jac.shape == (B, 3 * packed.K, 3 * n_rot + 13) and kp.shape == (B, packed.K, 3)
    kp, jac = kp.double().cpu().numpy(), jac.double().cpu().numpy()
    for b in ([0] if B == 1 else [0, 1, 17, 63]):
        k64, j64 = kp_lm_oracle.keypoint_jacobian(m, betas[b], rot[b], transl[b],
                                                  use_face_contour=variant == 'full')
        assert np.abs(kp[b] - k64).max() <= 1e-5 * np.abs(k64).max(), b
        for name, cols in _blocks(n_rot):
            err = np.abs(jac[b][:, cols] - j64[:, cols]).max()
            assert err <= TOL * np.abs(j64[:, cols]).max(), (b, name, err)
        assert np.array_equal(jac[b][:, 3 * n_rot + 10:], np.tile(np.eye(3), (packed.K, 1)))


def test_jacobian_transpose_equals_backward():
    """B = 4096: J^T c for a random joints cotangent c against shapy_smplx_backward: the betas block equals grad_betas,
    each rotation block the tangent projection sum_e (dL/dR_j)_e (R_j [e_a]x)_e of grad_rot."""
    from shapy_b200 import ops
    B, n_rot = 4096, 22
    packed = ops.SmplxModel(dict(synth.make_smplx()), 'cuda')
    rot, betas, transl = _inputs(7, B, n_rot)
    rot, betas, transl = rot.cuda(), betas.cuda(), transl.cuda()
    c = torch.randn(B, packed.K, 3, generator=torch.Generator().manual_seed(8)).cuda()
    _, jac = ops.smplx_keypoint_jacobian(packed, betas, rot, transl)
    jtc = torch.einsum('brp,br->bp', jac.double(), c.double().reshape(B, -1))
    del jac
    g = ops.smplx_backward(packed, betas, rot, grad_joints=c, want=('betas', 'rot'))
    E = torch.zeros(3, 3, 3, dtype=torch.float64, device='cuda')   # [e_a]x
    for a in range(3):
        E[a, (a + 2) % 3, (a + 1) % 3], E[a, (a + 1) % 3, (a + 2) % 3] = 1.0, -1.0
    D = torch.einsum('bjrm,amc->bjarc', rot.double(), E)           # R_j [e_a]x
    proj = torch.einsum('bjrc,bjarc->bja', g['rot'].double(), D).reshape(B, -1)
    for name, got, ref in (('rot', jtc[:, :3 * n_rot], proj), ('betas', jtc[:, 3 * n_rot:3 * n_rot + 10],
                                                               g['betas'].double())):
        err = (got - ref).abs().amax(1)
        scale = ref.abs().amax(1)
        assert bool((err <= TOL * scale).all()), (name, float((err / scale).max()))


def test_keypoints_vs_forward():
    from shapy_b200 import ops
    B, n_rot = 256, 22
    packed = ops.SmplxModel(dict(synth.make_smplx()), 'cuda')
    rot, betas, transl = _inputs(9, B, n_rot)
    rot, betas, transl = rot.cuda(), betas.cuda(), transl.cuda()
    kp, _ = ops.smplx_keypoint_jacobian(packed, betas, rot, transl)
    want = ops.smplx_forward(packed, betas, rot, want_vertices=True, want_v_shaped=False)['joints'] + transl[:, None]
    rel = ((kp - want).abs().amax((1, 2)) / want.abs().amax((1, 2)))
    print('keypoints vs forward, max relative', float(rel.max()))
    assert float(rel.max()) <= KP_TOL


def test_jacobian_deterministic_and_batch_independent():
    from shapy_b200 import ops
    packed = ops.SmplxModel(dict(synth.make_smplx()), 'cuda')
    rot, betas, transl = _inputs(5, 64, 22)
    rot, betas, transl = rot.cuda(), betas.cuda(), transl.cuda()
    kp1, j1 = ops.smplx_keypoint_jacobian(packed, betas, rot, transl)
    kp2, j2 = ops.smplx_keypoint_jacobian(packed, betas, rot, transl)
    assert torch.equal(bits(kp1), bits(kp2)) and torch.equal(bits(j1), bits(j2))
    rows = [0, 1, 9, 20, 33, 41, 50, 63]
    kp8, j8 = ops.smplx_keypoint_jacobian(packed, betas[rows].contiguous(), rot[rows].contiguous(),
                                          transl[rows].contiguous())
    assert torch.equal(bits(kp8), bits(kp1[rows])) and torch.equal(bits(j8), bits(j1[rows]))


def _step_case():
    """Six bodies of the synthetic model: the state at one pose, the trial at a nearby one; body 0 targets the trial
    (accepted), body 1 the state (rejected), body 2 a NaN trial keypoint (rejected), body 3 the trial with a dropped
    keypoint whose keypoint and rows are NaN in state and trial (accepted), 4 and 5 random targets."""
    from shapy_b200 import ops
    packed = ops.SmplxModel(dict(synth.make_smplx()), 'cuda')
    B, K = 6, packed.K
    rot, betas, transl = _inputs(11, B, 22)
    gen = torch.Generator().manual_seed(12)
    trot = (rot.double() @ rodrigues(torch.randn(B, 22, 3, generator=gen, dtype=torch.float64) * 0.02)).float()
    tbetas = betas + 0.05 * torch.randn(B, 10, generator=gen)
    ttransl = transl + 0.01 * torch.randn(B, 3, generator=gen)
    c = lambda t: t.cuda().contiguous()  # noqa: E731
    kp, jac = [t.cpu() for t in ops.smplx_keypoint_jacobian(packed, c(betas), c(rot), c(transl))]
    tkp, tjac = [t.cpu() for t in ops.smplx_keypoint_jacobian(packed, c(tbetas), c(trot), c(ttransl))]
    tg = kp + 0.05 * torch.randn(B, K, 3, generator=gen)
    tg[0], tg[1], tg[3] = tkp[0], kp[1], tkp[3]
    tkp[2, 5, 1] = float('nan')
    w = torch.rand(B, K, generator=gen) + 0.5
    w[3, 70] = 0.0
    for t in (kp, tkp):
        t[3, 70] = float('nan')
    for t in (jac, tjac):
        t[3, 210:213] = float('nan')
    loss = torch.tensor([kp_lm_oracle.loss(tg[b].numpy(), w[b].numpy(), kp[b].numpy()) for b in range(B)]).float()
    lam = torch.rand(B, generator=gen) + 0.01
    return dict(rot=rot, betas=betas, transl=transl, kp=kp, jac=jac, loss=loss, lam=lam, trot=trot, tbetas=tbetas,
                ttransl=ttransl, tkp=tkp, tjac=tjac, tg=tg, w=w)


@pytest.mark.parametrize('first', [False, True])
def test_step_kernel_vs_oracle(first):
    c = _step_case()
    state, trial = harness.kp_device(c)
    harness.kp_step(c, state, trial, first)
    flags, _ = harness.kp_check(c, state, trial, first)
    if first:
        assert all(flags)
    else:
        assert flags[:4] == [True, False, False, True], flags


# ------------------------------------------------------------------------------------------------ fit
FITS = {}
# Fraction of the 256 bodies within 1 cm keypoint RMS after LM with its default 50 iterations, and its median loss,
# set just below / above the first run on an H100 80GB HBM3 (700 W): LM 0.395 and 0.420 (median RMS 0.058 m), against
# Adam(600)'s 0.035 and 3.98, from a median start of 61.9.
LM_FRAC_BAR = 0.37
LM_MEDIAN_LOSS_BAR = 0.45


def _targets(module, B, seed=31):
    """The recipe of test_gpu_smplx_grad._targets."""
    gen = torch.Generator().manual_seed(seed)
    bstar = torch.randn(B, 10, generator=gen).clamp(-2, 2)
    raw = synth.mean_params()[:132] + 0.3 * torch.randn(B, 132, generator=gen)
    from shapy_b200 import ops
    with torch.no_grad():
        rot = ops.decode_rot6d(raw.cuda())
        return module(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=bstar.cuda())['joints'][:].clone()


def _fit(module, kp, **kw):
    from shapy_b200.fit import fit_body_to_keypoints
    mean = synth.mean_params()
    B = kp.shape[0]
    init = {'global_rot': mean[:6].expand(B, 6), 'body_pose': mean[6:132].expand(B, 126)}
    return fit_body_to_keypoints(module, kp, init=init, **kw)


@pytest.fixture(scope='module')
def module():
    return harness.smplx_module()


def _rms(res, kp):
    return (res['keypoints'] - kp).pow(2).sum(-1).mean(1).sqrt()


def test_lm_fit_256_bodies_vs_adam(module):
    kp = _targets(module, 256)
    lm = _fit(module, kp, method='lm')
    adam = _fit(module, kp)
    start = _fit(module, kp, method='lm', iterations=0)['loss']
    FITS['lm'], FITS['kp'] = lm, kp
    frac = {k: float((_rms(r, kp) < 1e-2).float().mean()) for k, r in (('lm', lm), ('adam', adam))}
    med = {k: float(r['loss'].median()) for k, r in (('lm', lm), ('adam', adam))}
    print('fit_keypoints_lm_256', {'frac_rms_1cm': frac, 'median_loss': med, 'median_start': float(start.median()),
                                   'median_rms_lm': float(_rms(lm, kp).median())})
    assert bool((lm['loss'] <= start).all())
    assert frac['lm'] > frac['adam'] and med['lm'] < med['adam']
    assert frac['lm'] >= LM_FRAC_BAR and med['lm'] <= LM_MEDIAN_LOSS_BAR
    # the raw 6D outputs decode to the fitted rotations
    from shapy_b200 import ops
    dec = ops.decode_rot6d(torch.cat([lm['global_rot'], lm['body_pose']], 1))
    assert float((dec - torch.cat([lm['global_rot_mat'], lm['body_pose_mat']], 1)).abs().max()) < 1e-6


def test_lm_fit_8_bodies_alone_equal_their_batch_rows(module):
    if 'lm' not in FITS:
        pytest.skip('needs test_lm_fit_256_bodies_vs_adam')
    rows = [3, 40, 77, 101, 150, 199, 230, 255]
    res8 = _fit(module, FITS['kp'][rows].contiguous(), method='lm')
    for k in ('global_rot', 'body_pose', 'betas', 'transl'):
        assert torch.equal(bits(res8[k]), bits(FITS['lm'][k][rows])), k


def test_lm_loop_never_synchronises(module):
    from shapy_b200.fit import fit_body_to_keypoints
    kp = _targets(module, 32)
    mean = synth.mean_params().cuda()
    init = {'global_rot': mean[:6].expand(32, 6), 'body_pose': mean[6:132].expand(32, 126)}
    fit_body_to_keypoints(module, kp, init=init, method='lm', iterations=1)      # packs the model
    _, res = harness.launches_without_sync(lambda: fit_body_to_keypoints(module, kp, init=init, method='lm',
                                                                         iterations=3))
    assert res['betas'].shape == (32, 10)


def test_argument_errors_and_empty_batch():
    from shapy_b200 import _lib, ops
    L = _lib.lib()
    packed = ops.SmplxModel(dict(synth.make_smplx()), 'cuda')
    z = lambda *s: torch.zeros(*s, device='cuda')  # noqa: E731
    torch.cuda.synchronize()
    n0 = L.shapy_launch_count()
    for n_rot in (0, packed.J + 1):
        rc = L.shapy_smplx_keypoint_jacobian(packed.handle, _lib.ptr(z(1, 10)), _lib.ptr(z(1, 56, 9)), n_rot, None, 1,
                                             _lib.ptr(z(1, packed.K, 3)), _lib.ptr(z(1, 3 * packed.K, 200)), None)
        assert rc == -1
    rc = L.shapy_smplx_keypoint_jacobian(packed.handle, None, _lib.ptr(z(1, 22, 9)), 22, None, 1,
                                         _lib.ptr(z(1, packed.K, 3)), _lib.ptr(z(1, 3 * packed.K, 79)), None)
    assert rc == -1
    kp, jac = ops.smplx_keypoint_jacobian(packed, z(0, 10), z(0, 22, 3, 3))
    assert kp.shape == (0, packed.K, 3) and jac.shape == (0, 3 * packed.K, 79)

    def step(B, n_rot, nb, null=False):
        K, P = packed.K, 3 * n_rot + nb + 3
        st = {'rot': z(B, n_rot, 3, 3), 'betas': z(B, nb), 'transl': z(B, 3), 'keypoints': z(B, K, 3),
              'jac': z(B, 3 * K, P), 'loss': z(B), 'lambda': z(B), 'accepted': torch.zeros(B, dtype=torch.int32,
                                                                                             device='cuda')}
        tr = {'rot': z(B, n_rot, 3, 3), 'betas': z(B, nb), 'transl': z(B, 3)}
        p = [_lib.ptr(st[k]) for k in ('rot', 'betas', 'transl', 'keypoints', 'jac', 'loss', 'lambda', 'accepted')]
        if null:
            p[4] = None
        return L.shapy_fit_lm_keypoints_step(B, K, n_rot, nb, _lib.ptr(z(B, K, 3)), _lib.ptr(z(B, K)), 10.0, 3.0, 1,
                                             *p, _lib.ptr(tr['rot']), _lib.ptr(tr['betas']), _lib.ptr(tr['transl']),
                                             _lib.ptr(z(B, K, 3)), _lib.ptr(z(B, 3 * K, P)), None)
    assert step(2, 30, 10) == -3                    # P = 103 > 96
    assert step(2, 22, 10, null=True) == -1
    assert step(2, 0, 10) == -1
    K = packed.K
    st = {'rot': z(0, 22, 3, 3), 'betas': z(0, 10), 'transl': z(0, 3), 'keypoints': z(0, K, 3), 'jac': z(0, 3 * K, 79),
          'loss': z(0), 'lambda': z(0), 'accepted': torch.zeros(0, dtype=torch.int32, device='cuda')}
    ops.fit_lm_keypoints_step(st, {'rot': z(0, 22, 3, 3), 'betas': z(0, 10), 'transl': z(0, 3)}, z(0, K, 3), z(0, K),
                              10.0, 3.0, True, z(0, K, 3), z(0, 3 * K, 79))
    assert L.shapy_launch_count() == n0
