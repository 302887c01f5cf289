"""GPU: fit_body_to_scan on the synthetic model (real SMPL-X topology and T-pose): 64 bodies of the 2D recipe's ground
truth, scans of 8192 area-weighted samples of the true posed surface with 2 mm noise, from the recipe's perturbed start,
against the 3D keypoint LM fit on the exact keypoints of the same bodies."""
import time

import numpy as np
import pytest
import torch

import scan_oracle as so
from shapy_b200 import ops, synth

pytestmark = pytest.mark.gpu

B, N = 64, 8192
_CACHE = {}


def _setup():
    if _CACHE:
        return _CACHE
    from shapy_b200.body_measurements import BodyMeasurements
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    m = SMPLX(data_struct=synth.make_smplx(), use_face_contour=True).cuda()
    bm = BodyMeasurements({'landmarks': synth.load_landmarks()}).cuda()
    gen = torch.Generator().manual_seed(61)
    rn = lambda *s: torch.randn(*s, generator=gen)  # noqa: E731
    bstar = rn(B, m.num_betas).clamp(-2, 2)
    raw = synth.mean_params()[:132] + 0.3 * rn(B, 132)
    transl = 0.3 * rn(B, 3)
    with torch.no_grad():
        rot = ops.decode_rot6d(raw.cuda())
        out = m(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=bstar.cuda(), transl=transl.cuda())
    init = {'global_rot': (raw[:, :6] + 0.1 * rn(B, 6)).cuda(), 'body_pose': (raw[:, 6:] + 0.1 * rn(B, 126)).cuda(),
            'betas': (bstar + 0.5 * rn(B, m.num_betas)).cuda(), 'transl': (transl + 0.05 * rn(B, 3)).cuda()}
    faces = m.faces_tensor.cpu().numpy()
    rng = np.random.default_rng(62)
    pts, facing = [], []
    for v in out['vertices'].double().cpu().numpy():
        p, f, _ = so.sample_surface(v, faces, N, rng)
        tri = v[faces[f]]
        nz = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])[:, 2]
        pts.append(p + rng.normal(size=p.shape) * 2e-3)
        facing.append(nz > 0)                              # seen by a camera on +z looking down -z
    _CACHE.update(model=m, bm=bm, bstar=bstar.cuda(), verts=out['vertices'].clone(), joints=out['joints'][:].clone(),
                  vshaped=out['v_shaped'].clone(), init=init,
                  points=torch.tensor(np.stack(pts), dtype=torch.float32).cuda(),
                  facing=torch.tensor(np.stack(facing)).cuda(), rng=rng)
    return _CACHE


def _measure(bm, m, betas):
    with torch.no_grad():
        vs = m.forward_shape(betas=betas)['v_shaped']
        meas = bm.forward_vertices(vs, m.faces_i32)['measurements']
    return vs, meas['height']['tensor'], meas['mass']['tensor']


def _row(c, res, seconds):
    m, bm = c['model'], c['bm']
    with torch.no_grad():
        rot = torch.cat([res['global_rot_mat'], res['body_pose_mat']], 1)
        v = m(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=res['betas'], transl=res['transl'],
              return_shaped=False)['vertices']
    vs, h, mass = _measure(bm, m, res['betas'])
    vs0, h0, mass0 = _measure(bm, m, c['bstar'])
    center = lambda x: x - x.mean(1, keepdim=True)  # noqa: E731
    return {'posed_v2v_mm': 1e3 * float((v - c['verts']).norm(dim=-1).mean(1).median()),
            'tpose_v2v_mm': 1e3 * float((center(vs) - center(vs0)).norm(dim=-1).mean(1).median()),
            'betas_err': float((res['betas'] - c['bstar']).norm(dim=1).median()),
            'height_1mm': float(((h - h0).abs() < 1e-3).float().mean()),
            'mass_1pct': float(((mass - mass0).abs() < 0.01 * mass0).float().mean()),
            'seconds': round(seconds, 2)}


def _timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = fn()
    torch.cuda.synchronize()
    return res, time.perf_counter() - t0


ROWS = {}


def _rows():
    if ROWS:
        return ROWS
    from shapy_b200.fit import fit_body_to_keypoints, fit_body_to_scan
    c = _setup()
    m, init, pts = c['model'], c['init'], c['points']
    fit_body_to_scan(m, pts[:2], init={k: v[:2] for k, v in init.items()}, iterations=2)       # warm-up
    fit_body_to_keypoints(m, c['joints'][:2], init={k: v[:2] for k, v in init.items()}, method='lm', iterations=2)
    res, s = _timed(lambda: fit_body_to_keypoints(m, c['joints'], init=init, method='lm'))
    ROWS['a_keypoints_lm'] = _row(c, res, s)
    res, s = _timed(lambda: fit_body_to_scan(m, pts, init=init))
    ROWS['b_scan_both'] = _row(c, res, s)
    res, s = _timed(lambda: fit_body_to_scan(m, pts, init=init, model_to_scan_weight=0.0))
    ROWS['c_scan_to_model'] = _row(c, res, s)
    w = c['facing'].float()
    res, s = _timed(lambda: fit_body_to_scan(m, pts, w, init=init, model_to_scan_weight=0.0))
    ROWS['d_partial'] = _row(c, res, s)
    gen = torch.Generator().manual_seed(63)
    out = (torch.rand(B, N, generator=gen) < 0.05).cuda()
    d = torch.randn(B, N, 3, generator=gen).cuda()
    d = d / d.norm(dim=-1, keepdim=True) * (0.1 + 0.2 * torch.rand(B, N, 1, generator=gen).cuda())
    po = torch.where(out[..., None], pts + d, pts)
    res, s = _timed(lambda: fit_body_to_scan(m, po, init=init))
    ROWS['e_outliers_lsq'] = _row(c, res, s)
    res, s = _timed(lambda: fit_body_to_scan(m, po, init=init, robust_sigma=0.01))
    ROWS['e_outliers_robust'] = _row(c, res, s)
    print('fit_body_to_scan_64', ROWS)
    return ROWS


# Bars just past the first run on an H100 80GB HBM3 (700 W) (README.md): the median posed per-vertex error (mm), the
# median translation-aligned T-pose v2v (mm) and the median |betas - betas*|.  The scan -> model term alone, the partial
# scan and the robust fit from this start do not converge; their bars only pin what the first run measured.
BARS = {
    'a_keypoints_lm': {'posed_v2v_mm': 24.5, 'tpose_v2v_mm': 11.0, 'betas_err': 1.37},   # 23.8, 10.6, 1.33
    'b_scan_both': {'posed_v2v_mm': 15.0, 'tpose_v2v_mm': 10.0, 'betas_err': 1.25},      # 14.4, 9.55, 1.21
    'c_scan_to_model': {'posed_v2v_mm': 170.0},                                           # 160
    'd_partial': {'posed_v2v_mm': 145.0},                                                 # 135
    'e_outliers_lsq': {'posed_v2v_mm': 17.0, 'betas_err': 1.6},                           # 16.0, 1.52
    'e_outliers_robust': {'posed_v2v_mm': 400.0},                                         # 385
}


def test_scan_fit_quality_against_the_keypoint_lm_fit():
    rows = _rows()
    for name, bars in BARS.items():
        for k, bar in bars.items():
            assert rows[name][k] <= bar, (name, k, rows[name][k], bar)
    # the dense surface beats the exact keypoints on the posed surface and the shape
    b, a = rows['b_scan_both'], rows['a_keypoints_lm']
    assert b['posed_v2v_mm'] < a['posed_v2v_mm'] and b['betas_err'] < a['betas_err']


def test_scan_fit_result_and_loss():
    """The returned vertices are SMPLX.forward of the returned parameters, and the loss is the definition's."""
    from shapy_b200.fit import fit_body_to_scan
    c = _setup()
    m, pts = c['model'], c['points'][:8].contiguous()
    init = {k: v[:8] for k, v in c['init'].items()}
    res = fit_body_to_scan(m, pts, init=init, iterations=5, robust_sigma=0.02, pose_prior_weight=0.1,
                           betas_weight=0.01, body_measurements=c['bm'])
    with torch.no_grad():
        v = m(global_rot=res['global_rot_mat'], body_pose=res['body_pose_mat'], betas=res['betas'],
              transl=res['transl'], return_shaped=False)['vertices']
    assert torch.equal(v, res['vertices'])
    assert res['measurements'].shape == (8, 5)
    f, b, d2 = ops.closest_points(v, m.faces_i32, pts)
    idx, e2 = ops.nearest_points(v, pts)
    s2 = 0.02 ** 2
    rho = lambda e: s2 * e / (s2 + e)  # noqa: E731
    rot0 = ops.decode_rot6d(torch.cat([init['global_rot'], init['body_pose']], 1))
    want = rho(d2).mean(1) + rho(e2).mean(1) + 0.05 * (res['body_pose_mat'] - rot0[:, 1:]).pow(2).sum((1, 2, 3)) + \
        0.01 * res['betas'].pow(2).sum(1)
    assert torch.allclose(res['loss'], want, rtol=1e-4, atol=1e-9)


def test_scan_fit_deterministic():
    from shapy_b200.fit import fit_body_to_scan
    c = _setup()
    m, pts, init = c['model'], c['points'][:16].contiguous(), {k: v[:16] for k, v in c['init'].items()}
    kw = dict(iterations=20, robust_sigma=0.02)
    r1 = fit_body_to_scan(m, pts, init=init, **kw)
    r2 = fit_body_to_scan(m, pts, init=init, **kw)
    for k in ('global_rot', 'body_pose', 'betas', 'transl', 'loss', 'vertices'):
        assert torch.equal(r1[k], r2[k]), k


def test_default_start_centres_the_body_on_the_scan():
    from shapy_b200.fit import fit_body_to_scan
    c = _setup()
    m, pts = c['model'], c['points'][:4].contiguous()
    res = fit_body_to_scan(m, pts, iterations=0)
    gap = (res['vertices'].mean(1) - pts.mean(1)).norm(dim=1)
    assert float(gap.max()) < 1e-5
