"""GPU: the vertex Jacobian, the scan LM step against tests/scan_lm_oracle.py, and fit_body_to_scan(method='lm') on
the recipe of test_gpu_fit_scan.py."""
import json
import math
import os

import numpy as np
import pytest
import torch

import lm_harness as H
import scan_lm_oracle as so
import test_gpu_fit_scan as ts
from shapy_b200 import ops, synth

pytestmark = pytest.mark.gpu


def _module():
    return H.smplx_module()


def _start(B, seed, nb):
    g = torch.Generator().manual_seed(seed)
    rot = H.rodrigues(torch.randn(B, 22, 3, generator=g, dtype=torch.float64) * 0.3).float()
    return rot, torch.randn(B, nb, generator=g) * 0.5, torch.randn(B, 3, generator=g) * 0.1


@pytest.mark.parametrize('variant', ['full', 'nb1_ne0', 'nb16_ne16'])
def test_vertex_jacobian_matches_oracle_and_keypoint_rows(variant):
    m = H.smplx_module(variant)
    md = H.variant_model(variant) if variant in H.VARIANTS else synth.make_smplx()
    rot, betas, transl = _start(2, 3, m.num_betas)
    packed = m.packed()
    v, jac = ops.smplx_vertex_jacobian(packed, betas.cuda(), rot.cuda(), transl.cuda())
    kp, kjac = ops.smplx_keypoint_jacobian(packed, betas.cuda(), rot.cuda(), transl.cuda())
    nb = m.num_betas
    for b in range(2):
        x64, j64 = so.vertex_jacobian(md, betas[b], rot[b], transl[b])
        assert np.abs(v[b].double().cpu().numpy() - x64).max() < 2e-5
        jb = jac[b].double().cpu().numpy()
        for lo, hi in ((0, 66), (66, 66 + nb), (66 + nb, 69 + nb)):
            ref = j64[..., lo:hi]
            assert np.abs(jb[..., lo:hi] - ref).max() <= H.TOL * max(1.0, np.abs(ref).max()), (b, lo)
        # the static landmarks: the barycentric mix of their face's vertex rows is the keypoint Jacobian's row
        faces = md['faces_tensor'].long()
        J = packed.J
        for li, (f, bc) in enumerate(zip(md['lmk_faces_idx'].long(), md['lmk_bary_coords'].float())):
            vi = faces[f]
            mix = sum(float(bc[k]) * jac[b, int(vi[k])].double() for k in range(3))
            row = kjac[b, 3 * (J + li):3 * (J + li) + 3].double()
            assert float((mix - row).abs().max()) <= 1e-5 * max(1.0, float(row.abs().max())), li


def _scan_case(B, N, seed, nan_dropped=True):
    """Scans of B bodies near the synthetic model's posed surface, about a fifth of the points dropped (NaN)."""
    m = _module()
    rot, betas, transl = _start(B, seed, m.num_betas)
    with torch.no_grad():
        out = m(global_rot=rot[:, :1].cuda(), body_pose=rot[:, 1:].cuda(), betas=betas.cuda(), transl=transl.cuda(),
                return_shaped=False)
    g = torch.Generator().manual_seed(seed + 1)
    idx = torch.randint(0, out['vertices'].shape[1], (B, N), generator=g)
    pts = torch.gather(out['vertices'].cpu(), 1, idx[..., None].expand(-1, -1, 3)) + 0.01 * torch.randn(B, N, 3,
                                                                                                          generator=g)
    w = torch.rand(B, N, generator=g) + 0.5
    drop = torch.rand(B, N, generator=g) < 0.2
    w[drop] = 0.0
    if nan_dropped:
        pts[drop] = float('nan')
    trial = {'rot': (rot.double() @ H.rodrigues(torch.randn(B, 22, 3, generator=g, dtype=torch.float64) * 0.05)).float(),
             'betas': betas + 0.2 * torch.randn(B, m.num_betas, generator=g),
             'transl': transl + 0.02 * torch.randn(B, 3, generator=g)}
    return m, pts.cuda().contiguous(), w.cuda().contiguous(), {k: v.cuda().contiguous() for k, v in trial.items()}


def _state(B, P, nb, device='cuda'):
    mk = lambda *s: torch.zeros(*s, dtype=torch.float32, device=device)  # noqa: E731
    return {'rot': mk(B, 22, 3, 3), 'betas': mk(B, nb), 'transl': mk(B, 3),
            'A': torch.zeros(B, P, P, dtype=torch.float64, device=device),
            'g': torch.zeros(B, P, dtype=torch.float64, device=device), 'loss': mk(B), 'lambda': mk(B),
            'accepted': torch.zeros(B, dtype=torch.int32, device=device)}


def _evaluate(m, trial, pts, w, m2s):
    v, jac = ops.smplx_vertex_jacobian(m.packed(), trial['betas'], trial['rot'], trial['transl'])
    face, bary, _ = ops.closest_points(v, m.faces_i32, pts, w)
    nearest = ops.nearest_points(v, pts, w)[0] if m2s > 0 else None
    return v, jac, face, bary, nearest


def _step(m, state, trial, pts, w, ev, terms, first, meas=None, anchor=None):
    sigma, s2m, m2s, pw, bw = terms
    B, N = pts.shape[:2]
    P = 66 + m.num_betas + 3
    ws = ops.fit_lm_scan_workspace(B, N, m.packed().V, P, 'cuda')
    ops.fit_lm_scan_step(state, trial, pts, w, m.faces_i32, sigma, s2m, m2s, pw, bw, 10.0, 3.0, first, *ev, ws,
                         pose_anchor=anchor, meas=meas)


def _meas_block(m, trial, seed):
    """(targets, weights, trial_meas, trial_meas_jac) of the trial betas: the measurements and their Jacobian (the
    circumferences' exact derivative, so that a Gauss-Newton step from the state lowers the loss), targets about 1 %
    off them, fit_betas_to_measurements' default weights with body 1's chest dropped."""
    from shapy_b200.fit import DEFAULT_WEIGHTS, NAMES, measurement_jacobian
    _, bm = H.smplx_and_measurements()
    r = measurement_jacobian(m, bm, trial['betas'], circumference_derivative='exact')
    tm, tmj = r['measurements'].contiguous(), r['jacobian'].contiguous()
    B = tm.shape[0]
    g = torch.Generator().manual_seed(seed)
    tgt = (tm.cpu() * (1 + 0.01 * torch.randn(B, 5, generator=g))).cuda().contiguous()
    wt = torch.tensor([DEFAULT_WEIGHTS[k] for k in NAMES]).repeat(B, 1)
    wt[1, 2] = 0.0
    return tgt, wt.cuda().contiguous(), tm, tmj


def _oracle(m, s0, trial0, pts, w, ev, terms, first, anchor, meas=None):
    sigma, s2m, m2s, pw, bw = terms
    v, jac, face, bary, nearest = [None if t is None else t.cpu().numpy() for t in ev]
    faces = m.faces_tensor.cpu().numpy()
    B, N = pts.shape[:2]
    P, V = 66 + m.num_betas + 3, v.shape[1]
    ns = math.ceil(N / so.CHUNK)
    out = []
    for b in range(B):
        chunks = so.rows(v[b], jac[b], pts[b].cpu().numpy(), w[b].cpu().numpy(), faces, face[b], bary[b],
                         None if nearest is None else nearest[b], math.inf if sigma is None else sigma, P)
        st = {k: t[b].cpu().numpy() for k, t in s0.items()}
        st['accepted'] = 0
        tr = {k: t[b].cpu().numpy() for k, t in trial0.items()}
        mk = {} if meas is None else dict(meas=(meas[0][b].cpu().numpy(), meas[1][b].cpu().numpy()),
                                          trial_meas=(meas[2][b].cpu().numpy(), meas[3][b].cpu().numpy()))
        out.append(so.lm_scan_step(st, tr, chunks, ns, w[b].cpu().numpy(), V, s2m, m2s, 10.0, 3.0, first,
                                   None if anchor is None else anchor[b].cpu().numpy(), pw, bw, **mk))
    return out


def _check(state, trial, oracle):
    got, nxt = H.numpy_of(state), H.numpy_of(trial)
    flags = []
    for b, (new, want, acc) in enumerate(oracle):
        flags.append(acc)
        assert got['accepted'][b] == new['accepted'], b
        assert np.isclose(got['loss'][b], new['loss'], rtol=3e-7, atol=0, equal_nan=True), (b, got['loss'][b], new['loss'])
        assert np.isclose(got['lambda'][b], new['lambda'], rtol=3e-7, atol=0), b
        for k in ('rot', 'betas', 'transl') + (('meas', 'meas_jac') if 'meas' in new else ()):
            assert np.array_equal(got[k][b], new[k], equal_nan=True), (b, k)
        for k in ('A', 'g'):
            ref = np.asarray(new[k])
            assert np.abs(got[k][b] - ref).max() <= 1e-9 * max(1.0, np.abs(ref).max()), (b, k)
        for k in ('rot', 'betas', 'transl'):
            assert np.abs(nxt[k][b] - want[k]).max() <= 2e-6 * max(1.0, np.abs(want[k]).max()), (b, k)
    return flags


# (robust_sigma, s2m, m2s, pose_prior_weight, betas_weight), with measurements or not
TERMS = [((None, 1.0, 1.0, 0.0, 0.0), False), ((0.01, 1.0, 1.0, 0.5, 0.1), False), ((None, 1.0, 0.0, 0.0, 0.0), False),
         ((None, 1.0, 1.0, 0.0, 0.0), True), ((0.01, 1.0, 1.0, 0.5, 0.1), True)]


@pytest.mark.parametrize('terms,with_meas', TERMS)
def test_step_matches_oracle_first_accept_reject(terms, with_meas):
    B, N = 2, 1500
    m, pts, w, trial = _scan_case(B, N, 11)
    P, nb = 66 + m.num_betas + 3, m.num_betas
    anchor = trial['rot'].clone() if terms[3] > 0 else None
    state = _state(B, P, nb)
    if with_meas:
        state.update(meas=torch.zeros(B, 5, device='cuda'), meas_jac=torch.zeros(B, 5, nb, device='cuda'))
    # first step: the trial becomes the state
    t0 = {k: v.clone() for k, v in trial.items()}
    s0 = {k: v.clone() for k, v in state.items()}
    ev = _evaluate(m, trial, pts, w, terms[2])
    meas = _meas_block(m, trial, 12) if with_meas else None
    _step(m, state, trial, pts, w, ev, terms, True, anchor=anchor, meas=meas)
    assert all(_check(state, trial, _oracle(m, s0, t0, pts, w, ev, terms, True, anchor, meas)))
    # the next trials, each step checked against the oracle: body 1's first one pushed far away with betas far from the
    # state's (rejected: under Geman-McClure a far trial alone can lower the loss, the betas prior or least squares
    # cannot), body 0's own (a Gauss-Newton step that overshoots is rejected and retried at a larger lambda, so body 0
    # must accept within four steps)
    trial['transl'][1] += 0.3
    trial['betas'][1] = 4.0 * state['betas'][1] + 1.0
    flags = []
    for _ in range(4):
        t0 = {k: v.clone() for k, v in trial.items()}
        s0 = {k: v.clone() for k, v in state.items()}
        ev = _evaluate(m, trial, pts, w, terms[2])
        if with_meas:                   # the same targets and weights, the new trial's measurements
            meas = meas[:2] + _meas_block(m, trial, 12)[2:]
        _step(m, state, trial, pts, w, ev, terms, False, anchor=anchor, meas=meas)
        flags.append(_check(state, trial, _oracle(m, s0, t0, pts, w, ev, terms, False, anchor, meas)))
        if flags[-1][0]:
            break
    assert not flags[0][1] and flags[-1][0], flags


def test_fit_with_measurements_end_to_end():
    """fit_body_to_scan(method='lm') with known height and mass: every body's loss non-increasing, the returned
    measurements those of the fitted betas, and the height nearer its target than without the measurements."""
    from shapy_b200.fit import fit_body_to_scan
    m, bm = H.smplx_and_measurements()
    B, N = 4, 2048
    _, pts, w, _ = _scan_case(B, N, 51, nan_dropped=False)
    _, betas, _ = _start(B, 51, m.num_betas)
    truth = H.measure(m, bm, betas.cuda())
    known = {'height': truth[:, 1] + 0.02, 'mass': truth[:, 0]}     # a known height 2 cm off what the scan shows
    kw = dict(method='lm', body_measurements=bm, measurements=known, robust_sigma=0.02)
    start = fit_body_to_scan(m, pts, w, iterations=0, **kw)
    res = fit_body_to_scan(m, pts, w, iterations=15, **kw)
    plain = fit_body_to_scan(m, pts, w, iterations=15, method='lm', body_measurements=bm, robust_sigma=0.02)
    assert bool((res['loss'] <= start['loss'] * (1 + 1e-5) + 1e-9).all())
    assert float((res['measurements'] - H.measure(m, bm, res['betas'])).abs().max()) < 1e-5
    err = lambda r: (r['measurements'][:, 1] - known['height']).abs()  # noqa: E731
    assert bool((err(res) < err(plain)).all()), (err(res), err(plain))


def test_dropped_measurements_and_nan_points_change_nothing():
    """Every measurement weight <= 0 (NaN values and rows): the bits of the step without measurements; a dropped
    point's coordinates are never read."""
    B, N = 2, 1500
    m, pts, w, trial = _scan_case(B, N, 21)
    P, nb = 66 + m.num_betas + 3, m.num_betas
    terms = (0.01, 1.0, 1.0, 0.0, 0.1)
    ev = _evaluate(m, trial, pts, w, 1.0)
    runs = []
    for variant in ('plain', 'meas', 'finite'):
        state, tr = _state(B, P, nb), {k: v.clone() for k, v in trial.items()}
        p, meas = pts, None
        if variant == 'meas':
            nan = torch.full((B, 5), float('nan'), device='cuda')
            state.update(meas=nan.clone(), meas_jac=torch.full((B, 5, nb), float('nan'), device='cuda'))
            wt = torch.zeros(B, 5, device='cuda')
            wt[:, 1] = -1.0
            meas = (nan.clone(), wt, nan.clone(), torch.full((B, 5, nb), float('nan'), device='cuda'))
        if variant == 'finite':
            p = torch.where(torch.isnan(pts), torch.full_like(pts, 7.0), pts)
        for first in (True, False):
            _step(m, state, tr, p, w, ev, terms, first, meas=meas)
        runs.append((state, tr))
    for k in ('rot', 'betas', 'transl', 'A', 'g', 'loss', 'lambda', 'accepted'):
        for s, _ in runs[1:]:
            assert torch.equal(runs[0][0][k].view(torch.uint8), s[k].view(torch.uint8)), k
    for k in ('rot', 'betas', 'transl'):
        for _, t in runs[1:]:
            assert torch.equal(H.bits(runs[0][1][k]), H.bits(t[k])), k
    assert torch.isfinite(runs[0][0]['loss']).all()


def test_bits_run_to_run_and_alone_in_a_batch():
    B, N = 3, 1200
    m, pts, w, trial = _scan_case(B, N, 31)
    P, nb = 66 + m.num_betas + 3, m.num_betas
    terms = (0.01, 1.0, 1.0, 0.0, 0.0)
    res = []
    for rows in (slice(0, B), slice(0, B), slice(1, 2)):
        tr = {k: v[rows].clone().contiguous() for k, v in trial.items()}
        n = tr['rot'].shape[0]
        state = _state(n, P, nb)
        p, ww = pts[rows].contiguous(), w[rows].contiguous()
        for first in (True, False, False):
            _step(m, state, tr, p, ww, _evaluate(m, tr, p, ww, 1.0), terms, first)
        res.append((state, tr))
    for k in ('rot', 'betas', 'transl', 'A', 'g', 'loss', 'lambda', 'accepted'):
        a, b, c = res[0][0][k], res[1][0][k], res[2][0][k]
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), k
        assert torch.equal(a[1:2].contiguous().view(torch.uint8), c.view(torch.uint8)), k


def test_iteration_without_host_sync():
    B, N = 2, 1000
    m, pts, w, trial = _scan_case(B, N, 41, nan_dropped=False)
    P, nb = 66 + m.num_betas + 3, m.num_betas
    state = _state(B, P, nb)
    ws = ops.fit_lm_scan_workspace(B, N, m.packed().V, P, 'cuda')
    tree = ops.ScanTree()
    ops.closest_points(*_evaluate(m, trial, pts, w, 1.0)[:1], m.faces_i32, pts, w, tree)   # builds the tree

    def it():
        v, jac = ops.smplx_vertex_jacobian(m.packed(), trial['betas'], trial['rot'], trial['transl'])
        face, bary, _ = ops.closest_points(v, m.faces_i32, pts, w, tree)
        nearest = ops.nearest_points(v, pts, w)[0]
        ops.fit_lm_scan_step(state, trial, pts, w, m.faces_i32, None, 1.0, 1.0, 0.0, 0.0, 10.0, 3.0, True, v, jac, face,
                             bary, nearest, ws)
    n, _ = H.launches_without_sync(it)
    assert n >= 4


# ---------------------------------------------------------------------------------------------------------- quality
def _lm_row(c, name, **kw):
    from shapy_b200.fit import fit_body_to_scan
    start = fit_body_to_scan(c['model'], c['points'], init=c['init'], method='lm', iterations=0, **kw)
    res, seconds = ts._timed(lambda: fit_body_to_scan(c['model'], c['points'], init=c['init'], method='lm', **kw))
    # every body's loss is non-increasing: the final forward (split-fp16 pose blend) may differ from the step's
    # vertices (fp32 posedirs) in the last bits
    assert bool((res['loss'] <= start['loss'] * (1 + 1e-5) + 1e-9).all()), name
    row = ts._row(c, res, seconds)
    row['start_loss'], row['final_loss'] = float(start['loss'].median()), float(res['loss'].median())
    return row


def test_scan_lm_quality():
    c = ts._setup()
    rows = {'b_both_terms': _lm_row(c, 'b')}
    partial = c['facing'].float()
    rows['d_partial_m2s0'] = _lm_row(c, 'd', weights=partial, model_to_scan_weight=0.0)
    B, N = c['points'].shape[:2]
    gen = torch.Generator().manual_seed(63)         # test_gpu_fit_scan.py's 5 % outliers, 0.1 - 0.3 m off
    out = (torch.rand(B, N, generator=gen) < 0.05).cuda()
    d = torch.randn(B, N, 3, generator=gen).cuda()
    d = d / d.norm(dim=-1, keepdim=True) * (0.1 + 0.2 * torch.rand(B, N, 1, generator=gen).cuda())
    c5 = dict(c, points=torch.where(out[..., None], c['points'] + d, c['points']))
    rows['e_outliers_ls'] = _lm_row(c5, 'e_ls')
    rows['e_outliers_gm_1cm'] = _lm_row(c5, 'e_gm', robust_sigma=0.01)
    print(json.dumps(rows))
    d = os.environ.get('SHAPY_TEST_OUT')
    if d:
        with open(os.path.join(d, 'scan_lm_quality.json'), 'w') as f:
            json.dump(rows, f, indent=1)
    # bars just past the values measured on an H100 80GB HBM3 at 700 W (README): posed v2v, T-pose v2v [mm], |beta -
    # beta*|; the posed v2v of b is well above Adam's 14.4 mm: 50 iterations stop short of convergence (README)
    bars = {'b_both_terms': (66.0, 11.5, 1.45), 'd_partial_m2s0': (240.0, 165.0, 20.5),
            'e_outliers_ls': (71.0, 23.5, 3.0), 'e_outliers_gm_1cm': (245.0, 76.0, 9.6)}
    for name, (v2v, tpose, beta) in bars.items():
        r = rows[name]
        assert r['posed_v2v_mm'] < v2v and r['tpose_v2v_mm'] < tpose and r['betas_err'] < beta, (name, r)
        assert r['final_loss'] < r['start_loss'], name
