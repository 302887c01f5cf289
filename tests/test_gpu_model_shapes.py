"""GPU: the posed SMPL-X backward, the keypoint Jacobian, the keypoint LM steps and the keypoint LM fit on every model
shape they accept: the variants of tests/test_model_shapes_cpu.py (NB 1 to 27, NE 0 to 16, NC up to 32, J14 from 448
to 2 100 non-zeros, the keypoint Jacobian's cached and uncached entry paths), against the float64 restatements that
test_model_shapes_cpu.py pins at those shapes.

  * posed backward (shapy_smplx_backward) against float64 autograd: the generic shape adjoint at NB != 10 and with the
    expression gradient at NE != 10; bar of test_gpu_smplx_grad.check, max |g - g64| <= 1e-4 max |g64| per body and
    tensor
  * keypoint Jacobian against kp_lm_oracle: bar of test_gpu_fit_lm_keypoints, 1e-4 per body and column block
  * cached against uncached Jacobian entries (edge_2048 / edge_2049): the same bits
  * J^T c against the posed backward on the uncached NB = 27 model
  * both 3D LM step kernels against their restatements at P = 7, 54, 55 (the 48 KB opt-in boundary) and 96, K = 1 to
    127
  * every keypoint step entry launches at P = 96 and refuses P = 97 without a launch
  * the 2D measurement step and both grouped 2D steps on random Jacobians against kp2d_lm_oracle and kp2dg_lm_oracle at
    the same shapes, groups of 1 to 64 images in regular and irregular layouts; groups of one against the 2D step and
    dropped measurements against the plain grouped step at every shape; no write outside any output or past the
    workspace
  * fit_body_to_keypoints(method='lm') at NB = 27 (P = 96) and NB = 16 with height and mass, and
    fit_body_to_keypoints_2d(method='lm') on the same two, per image and with groups"""
import numpy as np
import pytest
import torch

import kp_lm_oracle
import lm_harness as harness
from lm_harness import KP_CACHE_ENTRIES, TOL, VARIANTS, bits, keypoint_entries, variant_model
from shapy_b200 import synth
from smplx_grad_ref import oracle_grads

pytestmark = pytest.mark.gpu
NAMES = list(VARIANTS)
CHANGED_KP = 15                   # the keypoint J14 row 13 overwrites (source_idxs[13]): edge_2049's added entry


def _check(name, got, ref, tol=TOL):
    """test_gpu_smplx_grad.check; returns the largest error over its bar."""
    got, ref = got.detach().double().cpu(), torch.as_tensor(ref).double().cpu()
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    worst = 0.0
    for b in range(ref.shape[0]):
        scale = float(ref[b].abs().max())
        err = float((got[b] - ref[b]).abs().max())
        assert err <= tol * scale + 1e-30, (name, b, err, scale)
        worst = max(worst, err / (tol * scale + 1e-30))
    return worst


@pytest.fixture(scope='module')
def packed():
    from shapy_b200 import ops
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = ops.SmplxModel(dict(variant_model(name), use_face_contour=True), 'cuda')
        return cache[name]
    return get


# ------------------------------------------------------------------------------------------------ posed backward
@pytest.mark.parametrize('kind', ['mixed', 'j14'])
@pytest.mark.parametrize('B', [1, 33])
@pytest.mark.parametrize('n_rot', [1, 22, 55])
@pytest.mark.parametrize('name', NAMES)
def test_backward_vs_float64(packed, name, n_rot, B, kind):
    """B = 33 is a multiple of neither the 8- or 4-body shape-adjoint tile nor the 32-body vertex tile: rows in the
    first, a middle and the partial last tile are checked.  The expression gradient is wanted wherever NE > 0."""
    from shapy_b200 import ops
    m, pk = variant_model(name), packed(name)
    NB, NE, _ = VARIANTS[name]
    x = harness.inputs(10000 * NB + 100 * n_rot + B, B, n_rot, NB, NE)
    gen = torch.Generator().manual_seed(NB + n_rot + B)
    if kind == 'mixed':
        cot = dict(vertices=torch.randn(B, pk.V, 3, generator=gen), joints=torch.randn(B, pk.K, 3, generator=gen),
                   v_shaped=torch.randn(B, pk.V, 3, generator=gen) * 0.5,
                   proj_joints=torch.randn(B, pk.K, 2, generator=gen))
    else:                         # a one-hot on the keypoint J14 row 0 overwrites
        cot = dict(joints=torch.zeros(B, pk.K, 3))
        cot['joints'][:, int(m['source_idxs'][0]), 1] = 1.0
    c = lambda t: None if t is None else t.cuda()  # noqa: E731
    got = ops.smplx_backward(pk, c(x['betas']), c(x['rot']), expr=c(x['expression']), camera=c(x['camera']),
                             grad_vertices=c(cot.get('vertices')), grad_v_shaped=c(cot.get('v_shaped')),
                             grad_joints=c(cot.get('joints')), grad_proj_joints=c(cot.get('proj_joints')))
    assert (got['expr'] is None) == (NE == 0)
    rows = [0] if B == 1 else [0, 7, 8, 31, 32]
    sub = lambda t: None if t is None else t[rows]  # noqa: E731
    ref, _ = oracle_grads(m, {k: sub(v) for k, v in cot.items()}, sub(x['betas']), sub(x['rot']),
                          expression=sub(x['expression']), camera=sub(x['camera']))
    worst = max(_check('betas', got['betas'][rows], ref['betas']), _check('rot', got['rot'][rows], ref['rot']),
                _check('camera', got['camera'][rows], ref['camera']))
    if NE:
        worst = max(worst, _check('expression', got['expr'][rows], ref['expression']))
    print(f'[model-shapes] backward {name} n_rot={n_rot} B={B} {kind}: worst error / bar {worst:.3f}')


def test_module_autograd_with_expression():
    """SMPLX.forward through autograd on nb16_ne16 (NC = 32): betas, expression, the rotations, transl."""
    name = 'nb16_ne16'
    module = harness.smplx_module(name)
    NB, NE, _ = VARIANTS[name]
    B = 9
    x = harness.inputs(16, B, 22, NB, NE)
    leaf = {k: x[k].cuda().requires_grad_(True) for k in ('betas', 'expression', 'transl')}
    leaf['rot'] = x['rot'].cuda().requires_grad_(True)
    out = module(global_rot=leaf['rot'][:, :1], body_pose=leaf['rot'][:, 1:], betas=leaf['betas'],
                 expression=leaf['expression'], transl=leaf['transl'])
    gen = torch.Generator().manual_seed(17)
    V = module.get_num_verts()
    cot = dict(vertices=torch.randn(B, V, 3, generator=gen), joints=torch.randn(B, 123, 3, generator=gen),
               v_shaped=torch.randn(B, V, 3, generator=gen) * 0.5)
    loss = sum((out[k][:] * cot[k].cuda()).sum() for k in cot)
    loss.backward()
    ref, _ = oracle_grads(variant_model(name), cot, x['betas'], x['rot'], expression=x['expression'],
                          transl=x['transl'])
    worst = max(_check(k, leaf[k].grad, ref[k]) for k in ('betas', 'expression', 'rot', 'transl'))
    print(f'[model-shapes] module autograd {name}: worst error / bar {worst:.3f}')


# ------------------------------------------------------------------------------------------------ keypoint Jacobian
def _blocks(n_rot, NB):
    return (('rot', slice(0, 3 * n_rot)), ('betas', slice(3 * n_rot, 3 * n_rot + NB)))


@pytest.mark.parametrize('with_transl', [False, True])
@pytest.mark.parametrize('n_rot', [1, 22, 55])
@pytest.mark.parametrize('name', NAMES)
def test_jacobian_vs_float64(packed, name, n_rot, with_transl):
    from shapy_b200 import ops
    m, pk = variant_model(name), packed(name)
    NB = VARIANTS[name][0]
    B = 2
    x = harness.inputs(1000 * NB + 10 * n_rot + with_transl, B, n_rot, NB)
    transl = x['transl'] if with_transl else None
    kp, jac = ops.smplx_keypoint_jacobian(pk, x['betas'].cuda(), x['rot'].cuda(),
                                          None if transl is None else transl.cuda())
    P = 3 * n_rot + NB + 3
    assert jac.shape == (B, 3 * pk.K, P) and kp.shape == (B, pk.K, 3)
    kp, jac = kp.double().cpu().numpy(), jac.double().cpu().numpy()
    worst = 0.0
    for b in range(B):
        k64, j64 = kp_lm_oracle.keypoint_jacobian(m, x['betas'][b], x['rot'][b], None if transl is None else transl[b])
        assert np.abs(kp[b] - k64).max() <= 1e-5 * np.abs(k64).max(), b
        for block, cols in _blocks(n_rot, NB):
            err, scale = np.abs(jac[b][:, cols] - j64[:, cols]).max(), np.abs(j64[:, cols]).max()
            assert err <= TOL * scale, (b, block, err, scale)
            worst = max(worst, err / (TOL * scale))
        assert np.array_equal(jac[b][:, 3 * n_rot + NB:], np.tile(np.eye(3), (pk.K, 1)))
    print(f'[model-shapes] jacobian {name} n_rot={n_rot} transl={with_transl}: worst error / bar {worst:.3f}')


@pytest.mark.parametrize('n_rot', [1, 22, 55])
def test_cached_and_uncached_entries_give_the_same_bits(packed, n_rot):
    """edge_2048 caches its 2 048 keypoint entries in shared memory, edge_2049 (one more J14 non-zero, in the row of
    keypoint 15) recomputes each entry's vertex state where it is used.  Every other keypoint row, and every keypoint,
    must be bit-identical."""
    from shapy_b200 import ops
    a, b = variant_model('edge_2048'), variant_model('edge_2049')
    assert keypoint_entries(a) == KP_CACHE_ENTRIES < keypoint_entries(b)
    B = 64
    x = harness.inputs(2048 + n_rot, B, n_rot, 10)
    args = (x['betas'].cuda(), x['rot'].cuda(), x['transl'].cuda())
    kp_a, jac_a = ops.smplx_keypoint_jacobian(packed('edge_2048'), *args)
    kp_b, jac_b = ops.smplx_keypoint_jacobian(packed('edge_2049'), *args)
    K = kp_a.shape[1]
    keep = torch.tensor([k for k in range(K) if k != CHANGED_KP], device='cuda')
    rows = (3 * keep[:, None] + torch.arange(3, device='cuda')).reshape(-1)
    assert torch.equal(bits(kp_a[:, keep]), bits(kp_b[:, keep]))
    assert torch.equal(bits(jac_a[:, rows]), bits(jac_b[:, rows]))
    # the added entry does reach keypoint 15 (the two models differ there)
    assert not torch.equal(kp_a[:, CHANGED_KP], kp_b[:, CHANGED_KP])


def test_jacobian_transpose_equals_backward(packed):
    """nb27_ne5_dense at B = 256: J^T c for a random joints cotangent c against shapy_smplx_backward (whose betas
    gradient comes from the generic shape adjoint over 27 rows): the betas block equals grad_betas, each rotation block
    the tangent projection sum_e (dL/dR_j)_e (R_j [e_a]x)_e of grad_rot."""
    from shapy_b200 import ops
    name = 'nb27_ne5_dense'
    pk, NB = packed(name), VARIANTS[name][0]
    B, n_rot = 256, 22
    x = harness.inputs(7, B, n_rot, NB)
    rot, betas, transl = x['rot'].cuda(), x['betas'].cuda(), x['transl'].cuda()
    c = torch.randn(B, pk.K, 3, generator=torch.Generator().manual_seed(8)).cuda()
    _, jac = ops.smplx_keypoint_jacobian(pk, betas, rot, transl)
    jtc = torch.einsum('brp,br->bp', jac.double(), c.double().reshape(B, -1))
    del jac
    g = ops.smplx_backward(pk, betas, rot, grad_joints=c, want=('betas', 'rot'))
    E = torch.zeros(3, 3, 3, dtype=torch.float64, device='cuda')   # [e_a]x
    for a in range(3):
        E[a, (a + 2) % 3, (a + 1) % 3], E[a, (a + 1) % 3, (a + 2) % 3] = 1.0, -1.0
    D = torch.einsum('bjrm,amc->bjarc', rot.double(), E)           # R_j [e_a]x
    proj = torch.einsum('bjrc,bjarc->bja', g['rot'].double(), D).reshape(B, -1)
    worst = 0.0
    for block, got, ref in (('rot', jtc[:, :3 * n_rot], proj),
                            ('betas', jtc[:, 3 * n_rot:3 * n_rot + NB], g['betas'].double())):
        err = (got - ref).abs().amax(1)
        scale = ref.abs().amax(1)
        assert bool((err <= TOL * scale).all()), (block, float((err / scale).max()))
        worst = max(worst, float((err / (TOL * scale)).max()))
    print(f'[model-shapes] J^T c vs backward {name}: worst error / bar {worst:.3f}')


# ------------------------------------------------------------------------------------------------ LM steps
# (n_rot, nb): P = 3 n_rot + nb + 3 = 7, 54 (the largest P under 48 KB of shared memory without opting in), 55 (the
# smallest that opts in, twice: nb 16 and 1), 96 (kLmKpMaxP)
STEP_SHAPES = [(1, 1), (8, 27), (12, 16), (17, 1), (22, 27)]
STEP_K = [1, 5, 6, 127]           # 3K < 16 rows; K = 6 has a dropped keypoint 5 whose rows 15-17 straddle row 16


def _kp_step_vs_oracle(n_rot, nb, K, first, rho=None):
    """lm_harness.kp_random_case stepped once (rho None: the keypoint step) and checked against kp_lm_oracle; returns
    the largest trial error over its bar."""
    c = harness.kp_random_case(n_rot, nb, K, rho is not None, rho or 0.0)
    state, trial = harness.kp_device(c, rho)
    harness.kp_step(c, state, trial, first, rho)
    flags, worst = harness.kp_check(c, state, trial, first, rho)
    if first:
        assert all(flags)
    else:
        assert flags[:3] == [True, False, False] and (rho is None or not flags[3]), flags
    return worst


@pytest.mark.parametrize('first', [False, True])
@pytest.mark.parametrize('K', STEP_K)
@pytest.mark.parametrize('n_rot,nb', STEP_SHAPES)
def test_keypoint_step_vs_oracle(n_rot, nb, K, first):
    worst = _kp_step_vs_oracle(n_rot, nb, K, first)
    print(f'[model-shapes] kp step P={3 * n_rot + nb + 3} nb={nb} K={K} first={first}: trial error / bar {worst:.3f}')


@pytest.mark.parametrize('rho', [0.0, 0.05])
@pytest.mark.parametrize('first', [False, True])
@pytest.mark.parametrize('K', STEP_K)
@pytest.mark.parametrize('n_rot,nb', STEP_SHAPES)
def test_keypoint_measurement_step_vs_oracle(n_rot, nb, K, first, rho):
    worst = _kp_step_vs_oracle(n_rot, nb, K, first, rho)
    print(f'[model-shapes] kpm step P={3 * n_rot + nb + 3} nb={nb} K={K} first={first} rho={rho}: '
          f'trial error / bar {worst:.3f}')


def _call_every_step(n_rot, nb):
    """Each keypoint LM step entry once on zero inputs at (n_rot, nb), two bodies (two groups of one), first step: 3D,
    3D + measurements, 2D, 2D + measurements, grouped 2D, grouped 2D + measurements.  Returns their return codes."""
    from shapy_b200 import _lib
    L = _lib.lib()
    keep = []                                        # every tensor lives until the launches are done

    def z(*s, dtype=torch.float32):
        keep.append(torch.zeros(*s, dtype=dtype, device='cuda'))
        return _lib.ptr(keep[-1])
    B, G, K = 2, 2, 6
    P = 3 * n_rot + nb + 3
    off = torch.tensor([0, 1, 2], dtype=torch.int32)
    ws = z(L.shapy_fit_lm_groups_workspace_bytes(B, G, n_rot, nb) // 4 + 1)
    st = lambda: [z(B, n_rot, 3, 3), z(B, nb), z(B, 3), z(B, K, 3), z(B, 3 * K, P)]  # noqa: E731
    tr = lambda: [z(B, n_rot, 3, 3), z(B, nb), z(B, 3), z(B, K, 3), z(B, 3 * K, P)]  # noqa: E731
    head2d = lambda: [z(B, K, 2), z(B, K), z(B, n_rot, 3, 3), 1.0, 0.5, 0.1]  # noqa: E731
    counters = lambda: [z(B), z(B), z(B, dtype=torch.int32)]  # noqa: E731
    ms = lambda: [z(B, 5), z(B, 5, nb)]  # noqa: E731
    gst = lambda: [z(B, n_rot, 3, 3), z(G, nb), z(B, 3), z(B, K, 3), z(B, 3 * K, P)]  # noqa: E731
    gtr = lambda: [z(B, n_rot, 3, 3), z(G, nb), z(B, nb), z(B, 3), z(B, K, 3), z(B, 3 * K, P)]  # noqa: E731
    rc = [L.shapy_fit_lm_keypoints_step(B, K, n_rot, nb, z(B, K, 3), z(B, K), 10.0, 3.0, 1, *st(), *counters(), *tr(),
                                        None),
          L.shapy_fit_lm_keypoints_measurements_step(B, K, n_rot, nb, z(B, K, 3), z(B, K), z(B, 5), z(B, 5), 0.0, 10.0,
                                                     3.0, 1, *st(), *ms(), *counters(), *tr(), *ms(), None),
          L.shapy_fit_lm_keypoints_2d_step(B, K, n_rot, nb, *head2d(), 10.0, 3.0, 1, *st(), *counters(), *tr(), None),
          L.shapy_fit_lm_keypoints_2d_measurements_step(B, K, n_rot, nb, *head2d(), z(B, 5), z(B, 5), 10.0, 3.0, 1,
                                                        *st(), *ms(), *counters(), *tr(), *ms(), None),
          L.shapy_fit_lm_keypoints_2d_groups_step(B, G, off.data_ptr(), K, n_rot, nb, *head2d(), 10.0, 3.0, 1, *gst(),
                                                  *counters(), *gtr(), ws, None),
          L.shapy_fit_lm_keypoints_2d_groups_measurements_step(B, G, off.data_ptr(), K, n_rot, nb, *head2d(), z(G, 5),
                                                               z(G, 5), 10.0, 3.0, 1, *gst(), *ms(), *counters(),
                                                               *gtr(), *ms(), ws, None)]
    torch.cuda.synchronize()
    return rc


def test_steps_refuse_97_parameters_without_a_launch():
    """P = 96 (n_rot 22, nb 27) launches every keypoint step (one launch each, three for the grouped ones); P = 97, as
    (22, 28) and as (31, 1), is SHAPY_ERR_UNSUPPORTED from each, with nothing launched."""
    from shapy_b200 import _lib
    L = _lib.lib()
    torch.cuda.synchronize()
    n0 = L.shapy_launch_count()
    assert _call_every_step(22, 27) == [0] * 6
    assert L.shapy_launch_count() == n0 + 10
    for n_rot, nb in ((22, 28), (31, 1)):
        assert 3 * n_rot + nb + 3 == 97
        n0 = L.shapy_launch_count()
        assert _call_every_step(n_rot, nb) == [-3] * 6, (n_rot, nb)        # SHAPY_ERR_UNSUPPORTED
        assert L.shapy_launch_count() == n0, (n_rot, nb)


# ------------------------------------------------------------------------------------------------ 2D LM steps
# the 2D steps on random Jacobians at STEP_SHAPES, against kp2d_lm_oracle and kp2dg_lm_oracle (which
# test_model_shapes_cpu.py pins at these shapes); K: 2K = 2, 16 (one full staging tile), 18 and 254 rows
STEP_K_2D = [1, 8, 9, 127]
GROUP_K = [1, 9, 127]
LAYOUTS = {'1-2-3-5': (1, 2, 3, 5), '1-7-1-33-2': (1, 7, 1, 33, 2), '64': (64,)}
TERMS = harness.KP2D_TERMS['weak']


@pytest.mark.parametrize('terms', TERMS, ids=['lsq', 'robust_priors'])
@pytest.mark.parametrize('first', [False, True])
@pytest.mark.parametrize('K', STEP_K_2D)
@pytest.mark.parametrize('n_rot,nb', STEP_SHAPES + [(22, 10), (22, 11)])   # and P = 79 / 80, its 48 KB opt-in boundary
def test_keypoint_2d_measurement_step_vs_oracle(n_rot, nb, K, first, terms):
    worst = harness.kp2d_run(first, n_rot=n_rot, nb=nb, K=K, terms=terms, meas=True)
    print(f'[model-shapes] kp2dm step P={3 * n_rot + nb + 3} nb={nb} K={K} first={first} terms={terms}: '
          f'trial error / bar {worst:.3f}')


@pytest.mark.parametrize('with_meas', [False, True], ids=['kp2dg', 'kp2dgm'])
@pytest.mark.parametrize('layout', list(LAYOUTS))
@pytest.mark.parametrize('terms', TERMS, ids=['lsq', 'robust_priors'])
@pytest.mark.parametrize('first', [False, True])
@pytest.mark.parametrize('K', GROUP_K)
@pytest.mark.parametrize('n_rot,nb', STEP_SHAPES)
def test_groups_step_vs_oracle(n_rot, nb, K, first, terms, layout, with_meas):
    """Both grouped entries against kp2dg_lm_oracle: groups (1, 2, 3, 5), an irregular layout whose image kernel finds
    the groups of 1, 7, 1, 33 and 2 images by its binary search, and one group of 64 images."""
    c = harness.random_group_case(n_rot, nb, K, terms, LAYOUTS[layout])
    state, trial, _, G = harness.groups_device(c, with_meas)
    s0 = {k: v.cpu().numpy() for k, v in state.items()}
    harness.groups_step(c, state, trial, first, with_meas)
    flags, worst = harness.check_groups_vs_oracle(c, s0, state, trial, first, with_meas)
    if first:
        assert all(flags)
    else:
        assert flags[:3] == [True, False, True][:G], flags
    print(f'[model-shapes] {"kp2dgm" if with_meas else "kp2dg"} step P={3 * n_rot + nb + 3} nb={nb} K={K} '
          f'layout={layout} first={first} terms={terms}: trial error / bar {worst:.3f}')


@pytest.mark.parametrize('terms', TERMS, ids=['lsq', 'robust_priors'])
@pytest.mark.parametrize('first', [False, True])
@pytest.mark.parametrize('n_rot,nb', STEP_SHAPES)
def test_groups_of_one_equal_the_2d_step(n_rot, nb, first, terms):
    harness.check_groups_of_one(harness.random_group_case(n_rot, nb, 9, terms, (1,) * 6), first)


@pytest.mark.parametrize('terms', TERMS, ids=['lsq', 'robust_priors'])
@pytest.mark.parametrize('first', [False, True])
@pytest.mark.parametrize('n_rot,nb', STEP_SHAPES)
def test_dropped_measurements_equal_the_plain_groups_step(n_rot, nb, first, terms):
    harness.check_dropped_measurements(harness.random_group_case(n_rot, nb, 9, terms, (1, 2, 3, 5)), first)


GUARD = 64                        # sentinel elements on each side of a guarded output: 256 bytes, the alignment kept
SENTINEL = 0x7FA5A5A5


def _guarded(t):
    """A copy of t inside a larger int32 buffer with GUARD sentinel elements on each side; returns (copy, buffer)."""
    n = t.numel()
    buf = torch.full((n + 2 * GUARD,), SENTINEL, dtype=torch.int32, device='cuda')
    v = buf[GUARD:GUARD + n].view(t.dtype).view(t.shape)
    v.copy_(t)
    return v, buf


@pytest.mark.parametrize('entry', ['kp2dm', 'kp2dg', 'kp2dgm'])
@pytest.mark.parametrize('n_rot,nb', STEP_SHAPES)
def test_steps_write_nothing_outside_their_outputs(n_rot, nb, entry):
    """A first and a second step with every output (state, trial, image_betas, meas, meas_jac) a slice between
    sentinel guards and the workspace followed by sentinel bytes: the guards, the bytes past
    shapy_fit_lm_groups_workspace_bytes and every input keep their bits, and the outputs equal those of unguarded
    tensors bit for bit."""
    from shapy_b200 import _lib
    terms, K = TERMS[1], 9
    keys = ['tg', 'w', 'anchor', 'tkp', 'tjac'] + ([] if entry == 'kp2dg' else ['mt', 'mw', 'tmeas', 'tmjac'])
    if entry == 'kp2dm':
        c = harness.kp2d_case(n_rot, nb, K, terms, meas=True)
        state, trial = harness.kp2d_device(c)
    else:
        c = harness.random_group_case(n_rot, nb, K, terms, (1, 2, 3, 5))
        state, trial, B, G = harness.groups_device(c, entry == 'kp2dgm')
        need = _lib.lib().shapy_fit_lm_groups_workspace_bytes(B, G, n_rot, nb)
        wbuf = torch.full((need // 4 + 1 + GUARD,), SENTINEL, dtype=torch.int32, device='cuda')
        ws = wbuf.view(torch.uint8)[:need]
        tail = wbuf.view(torch.uint8)[need:].clone()
    cd = dict(c, **{k: c[k].cuda().contiguous() for k in keys})       # the inputs on the device, read in place
    inputs = {k: cd[k].clone() for k in keys}
    g_state = {k: _guarded(v) for k, v in state.items()}
    g_trial = {k: _guarded(v) for k, v in trial.items()}
    for first in (True, False):
        a_st, a_tr = {k: v[0] for k, v in g_state.items()}, {k: v[0] for k, v in g_trial.items()}
        if entry == 'kp2dm':
            harness.kp2d_step(cd, a_st, a_tr, first)
            harness.kp2d_step(cd, state, trial, first)
        else:
            harness.groups_step(cd, a_st, a_tr, first, entry == 'kp2dgm', ws)
            harness.groups_step(cd, state, trial, first, entry == 'kp2dgm')
    torch.cuda.synchronize()
    for what, gd, ref in (('state', g_state, state), ('trial', g_trial, trial)):
        for k, (v, buf) in gd.items():
            n = v.numel()
            assert bool((buf[:GUARD] == SENTINEL).all()) and bool((buf[GUARD + n:] == SENTINEL).all()), (what, k)
            assert torch.equal(bits(v), bits(ref[k])), (what, k)
    for k in keys:
        assert torch.equal(bits(cd[k]), bits(inputs[k])), k
    if entry != 'kp2dm':
        assert torch.equal(wbuf.view(torch.uint8)[need:], tail)


# ------------------------------------------------------------------------------------------------ fits
FIT_CASES = {'nb27_ne5_dense': None, 'nb16_ne16': ('height', 'mass')}


def _fit_targets(module, NB, B, bm=None, seed=31):
    """The recipe of test_gpu_fit_lm_keypoints._targets at the model's NB, plus the measurements of the generating
    betas."""
    from shapy_b200 import ops
    gen = torch.Generator().manual_seed(seed)
    bstar = torch.randn(B, NB, generator=gen).clamp(-2, 2).cuda()
    raw = synth.mean_params()[:132] + 0.3 * torch.randn(B, 132, generator=gen)
    with torch.no_grad():
        rot = ops.decode_rot6d(raw.cuda())
        kp = module(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=bstar)['joints'][:].clone()
        meas = None
        if bm is not None:
            m = bm.forward_vertices(module.forward_shape(betas=bstar)['v_shaped'], module.faces_i32)['measurements']
            meas = {k: m[k]['tensor'].clone() for k in m}
    return kp, meas


@pytest.mark.parametrize('name', list(FIT_CASES))
def test_lm_fit(packed, name):
    """fit_body_to_keypoints(method='lm') on 32 bodies: nb27_ne5_dense (P = 96, the uncached Jacobian) and nb16_ne16
    with height and mass (the four-launch stacked loop at NB = 16).  Every body's loss is at most its start, 8 bodies
    fitted alone equal their batch rows, the loop never synchronises, and the Jacobian and the backward repeat their
    bits."""
    from shapy_b200 import ops
    from shapy_b200.fit import fit_body_to_keypoints
    NB, NE, _ = VARIANTS[name]
    module = harness.smplx_module(name)
    bm, kw = None, {}
    if FIT_CASES[name]:
        from shapy_b200.body_measurements import BodyMeasurements
        bm = BodyMeasurements({'landmarks': synth.load_landmarks()}).cuda()
    B = 32
    kp, meas = _fit_targets(module, NB, B, bm)
    if bm is not None:
        kw = dict(body_measurements=bm, measurements={k: meas[k] for k in FIT_CASES[name]})
    mean = synth.mean_params().cuda()              # a CPU init would be copied to the device inside the fit

    def fit(kp, kw, iterations=None):
        n = kp.shape[0]
        init = {'global_rot': mean[:6].expand(n, 6), 'body_pose': mean[6:132].expand(n, 126)}
        return fit_body_to_keypoints(module, kp, init=init, method='lm', iterations=iterations, **kw)

    res = fit(kp, kw)
    start = fit(kp, kw, iterations=0)['loss']
    assert res['betas'].shape == (B, NB)
    fin = torch.isfinite(start)
    assert int(fin.sum()) >= B - 2
    assert bool((res['loss'][fin] <= start[fin]).all()), (res['loss'], start)
    print(f'[model-shapes] lm fit {name}: median loss {float(res["loss"].median()):.4g} from '
          f'{float(start[fin].median()):.4g}')
    rows = [3, 4, 9, 15, 16, 22, 30, 31]
    kw8 = dict(kw)
    if bm is not None:
        kw8['measurements'] = {k: v[rows].contiguous() for k, v in kw['measurements'].items()}
    res8 = fit(kp[rows].contiguous(), kw8)
    keys = ('global_rot', 'body_pose', 'betas', 'transl') + (('measurements',) if bm is not None else ())
    for k in keys:
        assert torch.equal(bits(res8[k]), bits(res[k][rows])), k
    harness.launches_without_sync(lambda: fit(kp, kw, iterations=3))
    # the Jacobian and the backward twice on the same inputs
    pk = packed(name)
    x = harness.inputs(99, B, 22, NB, NE)
    c = lambda t: None if t is None else t.cuda()  # noqa: E731
    j1, j2 = (ops.smplx_keypoint_jacobian(pk, c(x['betas']), c(x['rot']), c(x['transl'])) for _ in range(2))
    assert all(torch.equal(bits(a), bits(b)) for a, b in zip(j1, j2))
    gen = torch.Generator().manual_seed(100)
    cot = dict(grad_vertices=torch.randn(B, pk.V, 3, generator=gen).cuda(),
               grad_joints=torch.randn(B, pk.K, 3, generator=gen).cuda(),
               grad_v_shaped=torch.randn(B, pk.V, 3, generator=gen).cuda())
    g1, g2 = (ops.smplx_backward(pk, c(x['betas']), c(x['rot']), expr=c(x['expression']), **cot) for _ in range(2))
    for k in ('betas', 'rot', 'expr'):
        assert torch.equal(bits(g1[k]), bits(g2[k])), k


def _fit_problem_2d(module, NB, G, views, bm=None, seed=33):
    """G identities seen in `views` images each, image b of identity b % G (the labels are not sorted): betas* per
    identity, a raw pose (mean + 0.3 N) and camera per image; the targets their projected keypoints, with bm the
    identities' measurements; a start camera near the true one."""
    from shapy_b200 import ops
    gen = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=gen)  # noqa: E731
    B = G * views
    labels = torch.arange(B) % G
    bstar = rn(G, NB).clamp(-2, 2).cuda()
    raw = synth.mean_params()[:132] + 0.3 * rn(B, 132)
    cam = torch.stack([1.0 + 0.2 * rn(B), 0.1 * rn(B), 0.1 * rn(B)], 1)
    meas = None
    with torch.no_grad():
        rot = ops.decode_rot6d(raw.cuda())
        x = module(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=bstar[labels.cuda()],
                   camera=cam.cuda())['proj_joints'].clone()
        if bm is not None:
            m = bm.forward_vertices(module.forward_shape(betas=bstar)['v_shaped'], module.faces_i32)['measurements']
            meas = {k: m[k]['tensor'].clone() for k in m}
    return x, labels, (cam + 0.05 * rn(B, 3)).cuda(), meas


@pytest.mark.parametrize('grouped', [False, True], ids=['per_image', 'groups_8x4'])
@pytest.mark.parametrize('name', list(FIT_CASES))
def test_lm_fit_2d(name, grouped):
    """fit_body_to_keypoints_2d(method='lm') on 32 images of nb27_ne5_dense (P = 96) and of nb16_ne16 with height and
    mass, per image and as 8 identities x 4 views: every body's (group's) loss is at most its start, betas is (G, NB),
    a sub-batch of whole groups gives the batch's rows bit for bit, and the loop never synchronises."""
    from shapy_b200.fit import fit_body_to_keypoints_2d
    NB = VARIANTS[name][0]
    module = harness.smplx_module(name)
    bm = None
    if FIT_CASES[name]:
        from shapy_b200.body_measurements import BodyMeasurements
        bm = BodyMeasurements({'landmarks': synth.load_landmarks()}).cuda()
    G = 8 if grouped else 32
    x, labels, cam0, meas = _fit_problem_2d(module, NB, G, 32 // G, bm)
    mean = synth.mean_params().cuda()

    def args(ids):
        """The arguments of the fit of the identities `ids` (sorted), relabelled 0 .. len(ids) - 1 in their order, on
        the device (a copy from the host would synchronise), and their images' rows."""
        ids = torch.tensor(ids)
        rows = torch.isin(labels, ids).nonzero()[:, 0].cuda()
        n = len(rows)
        kw = dict(init={'global_rot': mean[:6].expand(n, 6), 'body_pose': mean[6:132].expand(n, 126),
                        'camera': cam0[rows].contiguous()},
                  method='lm', robust_sigma=0.1, pose_prior_weight=0.5, betas_weight=0.01)
        if grouped:
            kw['groups'] = torch.searchsorted(ids, labels[rows.cpu()])  # on the host: group_plan reads no device
        if bm is not None:
            kw.update(body_measurements=bm,
                      measurements={k: meas[k][ids.cuda()].contiguous() for k in FIT_CASES[name]})
        return x[rows].contiguous(), kw, rows

    def fit(a, iterations=None):
        return fit_body_to_keypoints_2d(module, a[0], iterations=iterations, **a[1])

    every = args(range(G))
    res = fit(every)
    start = fit(every, iterations=0)['loss']
    assert res['betas'].shape == (G, NB) and res['loss'].shape == (G,)
    fin = torch.isfinite(start)
    assert int(fin.sum()) >= G - 2
    assert bool((res['loss'][fin] <= start[fin]).all()), (res['loss'], start)
    print(f'[model-shapes] lm fit 2d {name} grouped={grouped}: median loss {float(res["loss"].median()):.4g} from '
          f'{float(start[fin].median()):.4g}')
    ids = [1, 4, 6] if grouped else [3, 4, 9, 15, 16, 22, 30, 31]
    a = args(ids)
    sub, rows = fit(a), a[2]
    for k in ('global_rot', 'body_pose', 'camera'):
        assert torch.equal(bits(sub[k]), bits(res[k][rows])), k
    for k in ('betas',) + (('measurements',) if bm is not None else ()) + (('loss',) if grouped else ()):
        assert torch.equal(bits(sub[k]), bits(res[k][ids])), k
    harness.launches_without_sync(lambda: fit(every, iterations=3))
