"""GPU: the sequence 2D keypoint Levenberg-Marquardt step (shapy_fit_lm_keypoints_2d_sequence_step) against its NumPy
restatement (tests/kp2d_sequence_lm_oracle.py, pinned by tests/test_fit_lm_kp2d_sequence_cpu.py) at P = 7 to 96 with
sequences of 1 to 33 frames, one-frame sequences against the perspective step, argument errors, and
fit_body_to_sequence end to end on the synthetic SMPL-X: launches per iteration, no host synchronisation, monotone
losses, determinism, batch independence, time reversal, a start behind the camera, Adam, the command line, and the
quality of per-frame, sequence and smoothed sequence fits of 32 synthetic videos."""
import math
import time

import numpy as np
import pytest
import torch

import kp2d_lm_oracle as o2
import kp2d_sequence_lm_oracle as osq
import lm_harness as harness
from lm_harness import bits, rodrigues
from shapy_b200 import synth

pytestmark = pytest.mark.gpu

F, PP = 1000.0, (500.0, 500.0)
STEP_SHAPES = [(1, 1), (8, 27), (22, 10), (22, 27)]
STEP_K = [1, 9, 127]
# (robust_sigma, pose_prior_weight, betas_weight, smooth_rot_weight, smooth_transl_weight), in pixels
TERMS = [(math.inf, 0.0, 0.0, 0.0, 0.0), (20.0, 500.0, 100.0, 3e3, 3e4)]
LENS = (1, 2, 5, 3)


# ------------------------------------------------------------------------------------------------ step kernels
def _step_case(n_rot, nb, K, terms, lens=LENS, seed=0):
    """Sequences of `lens` frames with random Jacobians, keypoints about 3-4 m in front of the camera.  Sequence 0's
    trial hits its targets, the others' targets are the state's projections plus noise; the last sequence's middle
    frame has a weighted trial keypoint behind the camera (rejected; NaN on a first step).  With K >= 8 keypoint 7 has
    weight 0 and NaN targets, keypoints and rows."""
    S, B, P = len(lens), sum(lens), 3 * n_rot + nb + 3
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    gidx = torch.repeat_interleave(torch.arange(S), torch.tensor(lens))
    gen = torch.Generator().manual_seed(5000 * n_rot + 10 * nb + K + seed + (3 if terms[1] else 0))
    rn = lambda *s: torch.randn(*s, generator=gen)  # noqa: E731
    rot = rodrigues(rn(B, n_rot, 3).double() * 0.5).float()
    trot = (rot.double() @ rodrigues(rn(B, n_rot, 3).double() * 0.05)).float()
    anchor = (rot.double() @ rodrigues(rn(B, n_rot, 3).double() * 0.1)).float()
    betas = rn(S, nb)
    tr = torch.cat([0.3 * rn(B, 2), 3.0 + torch.rand(B, 1, generator=gen)], 1)
    tbetas, ttr = betas + 0.05 * rn(S, nb), tr + 0.02 * rn(B, 3)
    kp, jac = 0.4 * rn(B, K, 3), 0.3 * rn(B, 3 * K, P)
    tkp, tjac = kp + 0.01 * rn(B, K, 3), jac + 0.03 * rn(B, 3 * K, P)
    intr = torch.tensor([F, *PP]).repeat(B, 1)
    intr[:, 0] *= 0.8 + 0.4 * torch.rand(B, generator=gen)
    proj = lambda k, t, b: torch.from_numpy(o2.project(k.numpy(), t.numpy(), intr[b].numpy())).float()  # noqa: E731
    tg = torch.stack([proj(kp[b], tr[b], b) for b in range(B)]) + 5.0 * rn(B, K, 2)
    for b in range(off[0], off[1]):
        tg[b], anchor[b] = proj(tkp[b], ttr[b], b), trot[b]
    bad = int(off[-2] + (off[-1] - off[-2]) // 2)
    tkp[bad, 0, 2] = -ttr[bad, 2] - 0.5                 # Y_z = -0.5
    w = torch.rand(B, K, generator=gen) + 0.5
    if K >= 8:
        w[:, 7] = 0.0
        tg[:, 7] = float('nan')
        for t in (kp, tkp):
            t[:, 7] = float('nan')
        for t in (jac, tjac):
            t[:, 21:24] = float('nan')
    return dict(off=off, gidx=gidx, rot=rot, betas=betas, tr=tr, kp=kp, jac=jac, trot=trot, tbetas=tbetas, ttr=ttr,
                tkp=tkp, tjac=tjac, tg=tg, w=w, intr=intr, anchor=anchor, lam=torch.rand(S, generator=gen) + 0.01,
                terms=terms)


def _n(t):
    return t.numpy()


def _frames(c, s):
    return [{'targets': _n(c['tg'][i]), 'weights': _n(c['w'][i]), 'intr': _n(c['intr'][i]),
             'anchor': _n(c['anchor'][i]), 'trial_kp': _n(c['tkp'][i]), 'trial_jac': _n(c['tjac'][i])}
            for i in range(c['off'][s], c['off'][s + 1])]


def _state_loss(c, s):
    """The loss of sequence s at its state, as the kernels compute it."""
    sigma, pw, bw, srw, stw = c['terms']
    r = range(c['off'][s], c['off'][s + 1])
    L = 0.0
    for i in r:
        L += o2.loss(_n(c['tg'][i]), _n(c['w'][i]), _n(c['kp'][i]), _n(c['tr'][i]), sigma, _n(c['rot'][i]),
                     _n(c['anchor'][i]), pw, intr=_n(c['intr'][i]))
        if i + 1 in r:
            L += osq.smooth_loss(_n(c['rot'][i]), _n(c['rot'][i + 1]), _n(c['tr'][i]), _n(c['tr'][i + 1]), srw, stw)
    if bw > 0:
        L += float(np.float32(bw)) * float(np.sum(_n(c['betas'][s]).astype(np.float64) ** 2))
    return L


def _device(c):
    S = len(c['off']) - 1
    cu = lambda t: t.cuda().contiguous()  # noqa: E731
    loss = torch.tensor([_state_loss(c, s) for s in range(S)]).float()
    state = {'rot': cu(c['rot']), 'betas': cu(c['betas']), 'transl': cu(c['tr']), 'keypoints': cu(c['kp']),
             'jac': cu(c['jac']), 'loss': cu(loss), 'lambda': cu(c['lam']),
             'accepted': torch.zeros(S, dtype=torch.int32, device='cuda')}
    trial = {'rot': cu(c['trot']), 'betas': cu(c['tbetas']), 'image_betas': cu(c['tbetas'][c['gidx']]),
             'transl': cu(c['ttr'])}
    return state, trial


def _step(c, state, trial, first):
    from shapy_b200 import ops
    cu = lambda t: t.cuda().contiguous()  # noqa: E731
    B, S = c['rot'].shape[0], len(c['off']) - 1
    ws = ops.fit_lm_sequence_workspace(B, S, c['rot'].shape[1], c['betas'].shape[1], 'cuda')
    sigma, pw, bw, srw, stw = c['terms']
    ops.fit_lm_keypoints_2d_sequence_step(state, trial, cu(c['tg']), cu(c['w']), cu(c['intr']), sigma, pw, bw, srw,
                                          stw, 10.0, 3.0, first, cu(c['tkp']), cu(c['tjac']),
                                          torch.from_numpy(c['off']), ws, pose_anchor=cu(c['anchor']))


def _check_vs_oracle(c, s0, state, trial, first):
    """The stepped device state and next trial against kp2d_sequence_lm_oracle sequence by sequence: loss and lambda to
    fp32 rounding, the state bit for bit, the next trial within 2e-6 max(1, |x|) (lm_harness.check_step), each frame's
    trial betas its sequence's.  Returns (the sequences' accepted flags, the largest trial error over its bar)."""
    S = len(c['off']) - 1
    sigma, pw, bw, srw, stw = c['terms']
    oracle = []
    for s in range(S):
        r = range(c['off'][s], c['off'][s + 1])
        st = {'rot': [s0['rot'][i] for i in r], 'transl': [s0['transl'][i] for i in r],
              'keypoints': [s0['keypoints'][i] for i in r], 'jac': [s0['jac'][i] for i in r],
              'betas': s0['betas'][s], 'loss': s0['loss'][s], 'lambda': s0['lambda'][s], 'accepted': 0}
        tr = {'rot': [_n(c['trot'][i]) for i in r], 'transl': [_n(c['ttr'][i]) for i in r],
              'betas': _n(c['tbetas'][s])}
        oracle.append(osq.lm_sequence_step(st, _frames(c, s), 10.0, 3.0, first, tr, sigma, pw, bw, srw, stw))
    got, nxt = harness.numpy_of(state), harness.numpy_of(trial)
    for s in range(S):
        for i in range(c['off'][s], c['off'][s + 1]):
            assert np.array_equal(nxt['image_betas'][i], nxt['betas'][s]), (s, i)
    image = ('rot', 'transl', 'keypoints', 'jac')
    gs, xs = harness.group_rows(c, got, nxt, S, image, ())
    return harness.check_step(gs, xs, oracle, image + ('betas',), ('rot', 'transl', 'betas'), exact=False)


@pytest.mark.parametrize('terms', TERMS, ids=['lsq', 'robust_priors_smooth'])
@pytest.mark.parametrize('first', [False, True])
@pytest.mark.parametrize('K', STEP_K)
@pytest.mark.parametrize('n_rot,nb', STEP_SHAPES)
def test_step_kernels_vs_oracle(n_rot, nb, K, first, terms):
    c = _step_case(n_rot, nb, K, terms)
    state, trial = _device(c)
    s0 = {k: v.cpu().numpy() for k, v in state.items()}
    _step(c, state, trial, first)
    flags, worst = _check_vs_oracle(c, s0, state, trial, first)
    assert flags[0] and not (flags[-1] and not first), flags
    if first:
        assert math.isnan(float(state['loss'][-1])) and torch.equal(trial['transl'][-3:].cpu(), c['ttr'][-3:])
    print(f'[kp2d sequence] step P={3 * n_rot + nb + 3} K={K} first={first} terms={terms}: accepted {flags}, trial '
          f'error / bar {worst:.3f}')


@pytest.mark.parametrize('first', [False, True])
def test_a_33_frame_sequence_vs_oracle(first):
    c = _step_case(22, 10, 127, TERMS[1], lens=(33, 2), seed=1)
    state, trial = _device(c)
    s0 = {k: v.cpu().numpy() for k, v in state.items()}
    _step(c, state, trial, first)
    flags, worst = _check_vs_oracle(c, s0, state, trial, first)
    print(f'[kp2d sequence] 33 frames first={first}: accepted {flags}, trial error / bar {worst:.3f}')


@pytest.mark.parametrize('terms', TERMS, ids=['lsq', 'robust_priors_smooth'])
@pytest.mark.parametrize('first', [False, True])
def test_one_frame_sequences_are_the_perspective_step(first, terms):
    """Eight sequences of one frame: loss, lambda, accepted and the state bit for bit as
    shapy_fit_lm_keypoints_2d_perspective_step; the next trial within 4e-6 max(1, |x|) (the CPU oracle test bounds
    the two eliminations' fp64 difference by 1e-12; what is left is the fp32 rounding of the result)."""
    from shapy_b200 import ops
    c = _step_case(22, 10, 127, terms, lens=(1,) * 8)
    c['tkp'][-1, 0, 2] = c['kp'][-1, 0, 2]          # no frame behind the camera: every loss finite
    state, trial = _device(c)
    b_state = {k: v.clone() for k, v in state.items()}
    b_trial = {k: v.clone() for k, v in trial.items() if k != 'image_betas'}
    _step(c, state, trial, first)
    cu = lambda t: t.cuda().contiguous()  # noqa: E731
    sigma, pw, bw, _, _ = terms
    ops.fit_lm_keypoints_2d_perspective_step(b_state, b_trial, cu(c['tg']), cu(c['w']), cu(c['intr']), sigma, pw, bw,
                                             10.0, 3.0, first, cu(c['tkp']), cu(c['tjac']),
                                             pose_anchor=cu(c['anchor']))
    for k in ('rot', 'betas', 'transl', 'keypoints', 'jac', 'loss', 'lambda', 'accepted'):
        assert torch.equal(bits(state[k]), bits(b_state[k])), k
    for k in ('rot', 'betas', 'transl'):
        err = (trial[k] - b_trial[k]).abs().max()
        assert float(err) <= 4e-6 * max(1.0, float(b_trial[k].abs().max())), (k, float(err))


def test_argument_offset_and_workspace_errors_and_the_empty_batch():
    from shapy_b200 import _lib, ops
    L = _lib.lib()
    z = lambda *s: torch.zeros(*s, device='cuda')  # noqa: E731
    K = 5
    torch.cuda.synchronize()
    n0 = L.shapy_launch_count()

    def step(B=3, off=(0, 1, 3), n_rot=22, nb=10, null=None, sigma=1.0, srw=1.0, stw=1.0):
        S = len(off) - 1
        P = 3 * n_rot + nb + 3
        ws = z(max(1, L.shapy_fit_lm_sequence_workspace_bytes(B, max(S, 0), max(n_rot, 1), nb) // 4 + 1))
        o = torch.tensor(off, dtype=torch.int32)
        head = [B, S, None if null == 'offsets' else o.data_ptr(), K, n_rot, nb, _lib.ptr(z(B, K, 2)),
                _lib.ptr(z(B, K)), None if null == 'intr' else _lib.ptr(z(B, 3)),
                None if null == 'anchor' else _lib.ptr(z(B, max(n_rot, 1), 3, 3)),
                sigma, 1.0 if null == 'anchor' else 0.0, 0.0, srw, stw, 10.0, 3.0, 1]
        st = [_lib.ptr(t) for t in (z(B, max(n_rot, 1), 3, 3), z(S, nb), z(B, 3), z(B, K, 3), z(B, 3 * K, P), z(S),
                                    z(S), torch.zeros(S, dtype=torch.int32, device='cuda'))]
        tr = [_lib.ptr(t) for t in (z(B, max(n_rot, 1), 3, 3), z(S, nb), z(B, nb), z(B, 3), z(B, K, 3),
                                    z(B, 3 * K, P))]
        return L.shapy_fit_lm_keypoints_2d_sequence_step(*head, *st, *tr, None if null == 'workspace' else
                                                         _lib.ptr(ws), None)
    assert step(n_rot=30) == -3                                 # P = 103 > 96
    assert step(nb=28) == -3                                    # P = 97
    for kw in (dict(null='offsets'), dict(null='intr'), dict(null='workspace'), dict(null='anchor'),
               dict(off=(0, 1, 2)), dict(off=(1, 3)), dict(off=(0, 3, 3)), dict(off=(0, 2, 1, 3)), dict(n_rot=0),
               dict(sigma=0.0), dict(sigma=float('nan')), dict(srw=-1.0), dict(stw=-1.0), dict(srw=float('nan')),
               dict(stw=float('inf'))):
        assert step(**kw) == -1, kw
    assert L.shapy_launch_count() == n0                       # nothing launched by a refused call
    for nb in (1, 27):                                          # P = 96 at nb = 27 launches
        assert step(nb=nb) == 0, nb
    torch.cuda.synchronize()
    assert L.shapy_launch_count() == n0 + 6
    assert L.shapy_fit_lm_sequence_workspace_bytes(-1, 0, 22, 10) == 0
    per = L.shapy_fit_lm_sequence_workspace_bytes(2, 1, 22, 10) - L.shapy_fit_lm_sequence_workspace_bytes(1, 1, 22, 10)
    assert L.shapy_fit_lm_sequence_workspace_bytes(100, 1, 22, 10) == \
        L.shapy_fit_lm_sequence_workspace_bytes(1, 1, 22, 10) + 99 * per
    n0 = L.shapy_launch_count()
    st = {'rot': z(0, 22, 3, 3), 'betas': z(0, 10), 'transl': z(0, 3), 'keypoints': z(0, K, 3), 'jac': z(0, 3 * K, 79),
          'loss': z(0), 'lambda': z(0), 'accepted': torch.zeros(0, dtype=torch.int32, device='cuda')}
    tr = {'rot': z(0, 22, 3, 3), 'betas': z(0, 10), 'image_betas': z(0, 10), 'transl': z(0, 3)}
    ops.fit_lm_keypoints_2d_sequence_step(st, tr, z(0, K, 2), z(0, K), z(0, 3), None, 0.0, 0.0, 0.0, 0.0, 10.0, 3.0,
                                          True, z(0, K, 3), z(0, 3 * K, 79), torch.zeros(1, dtype=torch.int32),
                                          ops.fit_lm_sequence_workspace(0, 0, 22, 10, 'cuda'))
    assert L.shapy_launch_count() == n0
    c = _step_case(22, 10, 9, TERMS[1])
    state, trial = _device(c)
    cu = lambda t: t.cuda().contiguous()  # noqa: E731
    args = (state, trial, cu(c['tg']), cu(c['w']), cu(c['intr']), None, 0.0, 0.0, 1.0, 1.0, 10.0, 3.0, True,
            cu(c['tkp']), cu(c['tjac']))
    with pytest.raises(RuntimeError, match='workspace'):
        ops.fit_lm_keypoints_2d_sequence_step(*args, torch.from_numpy(c['off']),
                                              torch.empty(0, device='cuda', dtype=torch.uint8))
    with pytest.raises(ValueError, match='sequence_offsets'):
        ops.fit_lm_keypoints_2d_sequence_step(*args, torch.tensor([0, 1, 1, 11], dtype=torch.int32),
                                              ops.fit_lm_sequence_workspace(11, 3, 22, 10, 'cuda'))
    with pytest.raises(ValueError, match='smoothness'):
        ops.fit_lm_keypoints_2d_sequence_step(*args[:8], -1.0, *args[9:], torch.from_numpy(c['off']),
                                              ops.fit_lm_sequence_workspace(11, 4, 22, 10, 'cuda'))
    assert L.shapy_launch_count() == n0


# ------------------------------------------------------------------------------------------------ fit
def _slerp(R0, R1, s):
    """R0 Exp(s Log(R0^T R1)) per joint, float64 (via scipy)."""
    from scipy.spatial.transform import Rotation
    d = Rotation.from_matrix((R0.transpose(-1, -2) @ R1).reshape(-1, 3, 3).numpy()).as_rotvec()
    E = torch.from_numpy(Rotation.from_rotvec(d * s).as_matrix()).reshape(R0.shape)
    return R0 @ E


def _video(module, S, T, seed=81, noise_px=3.0, drop=0.05, fps=30.0):
    """S synthetic videos of T frames: betas* per video; the body pose slerped between two keyframes of the 2D recipe
    (raw 6D = mean + 0.3 N(0, 1)); the global rotation turning 60 degrees about the vertical over the clip; the root
    walking sideways at 1 m/s at a depth t_z in [2, 4] m; f = 1000 px, pp = (500, 500).  Detections: the exact
    projections plus noise_px Gaussian noise, a fraction `drop` of the keypoints dropped (weight 0, NaN).  Start: the
    2D recipe's perturbation drawn per frame (raw pose + 0.1 N, betas + 0.5 N) and t* + (5, 5, 30) cm N(0, 1)."""
    from shapy_b200 import ops
    from shapy_b200.fit import _project
    gen = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=gen)  # noqa: E731
    B = S * T
    bstar = rn(S, module.num_betas).clamp(-2, 2)
    raw0 = synth.mean_params()[:132] + 0.3 * rn(S, 132)
    raw1 = synth.mean_params()[:132] + 0.3 * rn(S, 132)
    k0, k1 = ops.decode_rot6d(raw0.cuda()).cpu().double(), ops.decode_rot6d(raw1.cuda()).cpu().double()
    s = torch.linspace(0.0, 1.0, T, dtype=torch.float64)
    rot = torch.stack([torch.stack([_slerp(k0[i], k1[i], float(s[t])) for t in range(T)]) for i in range(S)])
    ang = math.radians(60.0) * s
    Ry = torch.zeros(T, 3, 3, dtype=torch.float64)
    Ry[:, 0, 0], Ry[:, 0, 2], Ry[:, 1, 1], Ry[:, 2, 0], Ry[:, 2, 2] = ang.cos(), ang.sin(), 1.0, -ang.sin(), ang.cos()
    rot[:, :, 0] = Ry[None] @ k0[:, None, 0]
    rot = rot.reshape(B, 22, 3, 3).float()
    tz = 2.0 + 2.0 * torch.rand(S, generator=gen)
    t = torch.arange(T, dtype=torch.float32)
    tstar = torch.stack([(-0.5 + t[None] / fps).expand(S, T), (0.2 * rn(S))[:, None].expand(S, T),
                         tz[:, None].expand(S, T)], -1).reshape(B, 3)
    seq = torch.arange(B) // T
    intr = torch.tensor([F, *PP]).repeat(B, 1).cuda()
    with torch.no_grad():
        out = module(global_rot=rot[:, :1].cuda(), body_pose=rot[:, 1:].cuda(), betas=bstar[seq].cuda(),
                     transl=tstar.cuda())
        joints = out['joints'][:].clone()
        exact = _project(joints, intr)
    K = exact.shape[1]
    x = exact + noise_px * rn(B, K, 2).cuda()
    w = (torch.rand(B, K, generator=gen) >= drop).float().cuda()
    x = torch.where(w[..., None] > 0, x, torch.full_like(x, float('nan')))
    raw = rot[..., :2].reshape(B, 132)
    init = {'global_rot': (raw[:, :6] + 0.1 * rn(B, 6)).cuda(), 'body_pose': (raw[:, 6:] + 0.1 * rn(B, 126)).cuda(),
            'betas': (bstar[seq] + 0.5 * rn(B, module.num_betas)).cuda(),
            'transl': (tstar + torch.tensor([0.05, 0.05, 0.3]) * rn(B, 3)).cuda()}
    return dict(x=x.contiguous(), w=w, exact=exact, joints=joints, init=init, tstar=tstar.cuda(), bstar=bstar.cuda(),
                seq=seq, S=S, T=T)


def _fit(module, v, **kw):
    from shapy_b200.fit import fit_body_to_sequence
    kw.setdefault('init', v['init'])
    kw.setdefault('sequences', v['seq'])
    return fit_body_to_sequence(module, v['x'], F, PP, weights=v['w'], **kw)


SMOOTH = dict(smooth_rot_weight=3e3, smooth_transl_weight=1e4)


def test_lm_launches_no_synchronisation_and_monotone_losses():
    module = harness.smplx_module()
    v = _video(module, 4, 8, seed=82)
    kw = dict(method='lm', robust_sigma=10.0, pose_prior_weight=100.0, **SMOOTH)
    _fit(module, v, iterations=1, **kw)
    for init in (v['init'], {}):                                # and the default start
        counts = []
        for its in (3, 4):
            n, res = harness.launches_without_sync(lambda: _fit(module, v, iterations=its, init=init, **kw))
            counts.append(n)
        assert counts[1] - counts[0] == 4, counts
    assert res['transl'].shape == (32, 3) and res['betas'].shape == (4, 10) and res['loss'].shape == (4,)
    assert res['proj_joints'].shape == v['x'].shape
    prev = None
    for its in (0, 2, 5, 10, 20):
        r = _fit(module, v, iterations=its, **kw)
        assert bool(torch.isfinite(r['loss']).all())
        if prev is not None:
            assert bool((r['loss'] <= prev).all()), (its, r['loss'], prev)
        prev = r['loss']
    assert float(prev.median()) < 0.5 * float(_fit(module, v, iterations=0, **kw)['loss'].median())


def test_lm_deterministic_batch_independent_and_reversible():
    """Bitwise determinism; a sequence alone gives its bits in the batch; the labels need not be sorted; and every
    sequence's frames reversed give the reversed fit to tolerance (C_t against C_t^T)."""
    module = harness.smplx_module()
    v = _video(module, 6, 8, seed=83)
    kw = dict(method='lm', iterations=12, robust_sigma=10.0, pose_prior_weight=100.0, **SMOOTH)
    r1, r2 = _fit(module, v, **kw), _fit(module, v, **kw)
    for k in r1:
        assert torch.equal(bits(r1[k]), bits(r2[k])), k
    s = 3
    rows = torch.arange(s * 8, (s + 1) * 8)
    one = _fit(module, dict(v, x=v['x'][rows], w=v['w'][rows]), sequences=None,
               init={k: t[rows] for k, t in v['init'].items()}, **kw)
    for k in ('global_rot', 'body_pose', 'transl'):
        assert torch.equal(bits(one[k]), bits(r1[k][rows])), k
    for k in ('betas', 'loss'):
        assert torch.equal(bits(one[k][0]), bits(r1[k][s])), k
    # interleaved labels: the same sequences in another batch order
    perm = torch.arange(48).reshape(6, 8).t().reshape(-1)
    mixed = _fit(module, dict(v, x=v['x'][perm], w=v['w'][perm], seq=v['seq'][perm]),
                 init={k: t[perm] for k, t in v['init'].items()}, **kw)
    for k in ('global_rot', 'transl'):
        assert torch.equal(bits(mixed[k]), bits(r1[k][perm])), k
    assert torch.equal(bits(mixed['betas']), bits(r1['betas']))
    rev = torch.arange(48).reshape(6, 8).flip(1).reshape(-1)
    back = _fit(module, dict(v, x=v['x'][rev], w=v['w'][rev]), init={k: t[rev] for k, t in v['init'].items()},
                iterations=3, **{k: a for k, a in kw.items() if k != 'iterations'})
    fwd = _fit(module, v, iterations=3, **{k: a for k, a in kw.items() if k != 'iterations'})
    err_t = float((back['transl'] - fwd['transl'][rev]).abs().max())
    err_b = float((back['betas'] - fwd['betas']).abs().max())
    err_l = float(((back['loss'] - fwd['loss']).abs() / fwd['loss']).max())
    print(f'[kp2d sequence] reversed frames: transl {err_t:.2e} m, betas {err_b:.2e}, loss {err_l:.2e}')
    assert err_t <= 1e-4 and err_b <= 1e-3 and err_l <= 1e-4


def test_start_behind_the_camera_reports_inf_and_does_not_move():
    module = harness.smplx_module()
    v = _video(module, 3, 5, seed=84)
    init = {k: t.clone() for k, t in v['init'].items()}
    init['transl'][7, 2] = -3.0                                 # frame 2 of sequence 1
    res = _fit(module, v, init=init, method='lm', iterations=5, **SMOOTH)
    assert res['loss'][1] == float('inf') and torch.isfinite(res['loss'][[0, 2]]).all()
    assert torch.equal(bits(res['transl'][5:10]), bits(init['transl'][5:10]))
    ref = _fit(module, v, method='lm', iterations=5, **SMOOTH)
    for k in ('betas', 'loss'):
        assert torch.equal(bits(res[k][[0, 2]]), bits(ref[k][[0, 2]])), k


def test_adam_lowers_the_loss():
    module = harness.smplx_module()
    v = _video(module, 4, 6, seed=85)
    r0 = _fit(module, v, method='adam', iterations=0, **SMOOTH)
    r = _fit(module, v, method='adam', iterations=150, lr=0.01, **SMOOTH)
    ratio = float(r['loss'].median() / r0['loss'].median())
    print(f'[kp2d sequence] Adam(150): median loss / start {ratio:.3f}')
    assert ratio < 0.5 and r['proj_joints'].shape == v['x'].shape and r['betas'].shape == (4, 10)


def test_cli_on_a_written_npz(tmp_path):
    from shapy_b200 import fit
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    module = harness.smplx_module()
    v = _video(module, 2, 5, seed=86)
    K = SMPLX(data_struct=synth.make_smplx()).cuda().packed().K          # the command line's model: its keypoints lead
    n = lambda t: t.detach().cpu().numpy()  # noqa: E731
    seq = np.array([1, 0] * 5)                                  # interleaved: video 0 the odd rows
    order = np.argsort(seq, kind='stable')
    x = np.empty((10, K, 2), np.float32)
    w = np.empty((10, K), np.float32)
    x[order], w[order] = n(v['x'][:, :K]), n(v['w'][:, :K])
    np.savez(tmp_path / 'kp.npz', keypoints=x, weights=w, focal_length=np.float32(F),
             principal_point=np.array(PP, np.float32), sequences=seq)
    out = {}
    for its in (0, 10):
        path = tmp_path / f'fit{its}.npz'
        fit.main(['--synthetic', '--keypoints-2d', str(tmp_path / 'kp.npz'), '--sequence', '--method', 'lm',
                  '--iterations', str(its), '--robust-sigma', '10', '--smooth-rot', '1000', '--smooth-transl', '1e4',
                  '--output', str(path)])
        out[its] = np.load(path)
    r = out[10]
    assert r['transl'].shape == (10, 3) and r['betas'].shape[0] == 2 and r['loss'].shape == (2,)
    assert np.array_equal(r['sequences'], seq) and np.isfinite(r['loss']).all()
    assert (r['loss'] < out[0]['loss']).all()


# Quality, 32 videos x 32 frames at 30 fps, 50 LM iterations each: (a) per-frame perspective fits, (b) the sequence
# fit without smoothness, (c) the sequence fit with SMOOTH.  First run on an H100 80GB HBM3 (700 W): median root-aligned
# joint error 0.170 / 0.184 / 0.180 m, acceleration error 417 / 387 / 343 mm / frame^2, median |beta - beta*| 1.345 /
# 0.869 / 1.132, median |t_z - t_z*| / t_z* 6.2 / 10.0 / 10.9 %, frames under 5 px RMS 38.5 / 30.5 / 31.0 % (README.md).
# Bars just past (b) and (c).
BARS = {'seq': {'mpjpe': 0.19, 'accel': 400.0, 'beta': 0.9, 'tz_rel': 0.105},
        'smooth': {'mpjpe': 0.185, 'accel': 355.0, 'beta': 1.17, 'tz_rel': 0.115}}


def video_quality(module, v, res, per_frame_betas=False):
    """The report of one fit: median root-aligned joint error (m), mean acceleration error of the camera-frame joints
    (mm / frame^2), median |beta - beta*| per sequence (per frame for per-frame fits), median |t_z - t_z*| / t_z*, the
    share of frames under 5 px 2D RMS against the detections."""
    from shapy_b200.metrics import PointError, build_alignment
    pe = PointError(build_alignment('root'))
    pe(res['keypoints'].contiguous(), v['joints'])
    S, T = v['S'], v['T']
    j, js = res['keypoints'].reshape(S, T, -1, 3), v['joints'].reshape(S, T, -1, 3)
    acc = lambda a: a[:, 2:] - 2 * a[:, 1:-1] + a[:, :-2]  # noqa: E731
    accel = float((acc(j) - acc(js)).norm(dim=-1).mean()) * 1e3
    bstar = v['bstar'][v['seq'].cuda()] if per_frame_betas else v['bstar']
    w = v['w']
    d = torch.where(w[..., None] > 0, res['proj_joints'] - v['x'], torch.zeros_like(v['x']))
    rms = (d.pow(2).sum(-1).sum(1) / w.sum(1)).sqrt()
    return dict(mpjpe=float(pe.last_mean.median()), accel=accel,
                beta=float((res['betas'] - bstar).norm(dim=1).median()),
                tz_rel=float(((res['transl'][:, 2] - v['tstar'][:, 2]).abs() / v['tstar'][:, 2]).median()),
                rms_5px=float((rms < 5.0).float().mean()))


def quality_runs(module, v, iterations=50):
    """The three fits of the quality test, each timed after a warm-up: {arm: report + seconds}."""
    from shapy_b200.fit import fit_body_to_keypoints_2d
    arms = {'per_frame': lambda its: fit_body_to_keypoints_2d(module, v['x'], v['w'], init=v['init'], method='lm',
                                                              iterations=its, focal_length=F, principal_point=PP),
            'seq': lambda its: _fit(module, v, method='lm', iterations=its),
            'smooth': lambda its: _fit(module, v, method='lm', iterations=its, **SMOOTH)}
    out = {}
    for name, run in arms.items():
        run(2)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = run(iterations)
        torch.cuda.synchronize()
        sec = time.perf_counter() - t0
        q = video_quality(module, v, res, name == 'per_frame')
        out[name] = {**{k: round(x, 5) for k, x in q.items()}, 'seconds': round(sec, 3)}
    return out


def test_quality_32_videos():
    module = harness.smplx_module()
    v = _video(module, 32, 32)
    rep = quality_runs(module, v)
    print('fit_kp2d_sequence_32x32', rep)
    for arm, bars in BARS.items():
        for m, bar in bars.items():
            assert rep[arm][m] <= bar, (arm, m, rep[arm][m], bar)
    assert rep['seq']['beta'] < rep['per_frame']['beta']          # one betas per video sees it better
    assert rep['smooth']['accel'] < min(rep['seq']['accel'], rep['per_frame']['accel'])
