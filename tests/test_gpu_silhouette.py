"""GPU: the silhouette kernels (include/shapy_b200.h, shapy_silhouette_*, shapy_render_silhouette) against
tests/silhouette_oracle.py: the distance transform and contour bit for bit, the rasteriser at every unambiguous pixel,
shapy_closest_points on the flat projected mesh against float64 brute force, the term and its gradient, determinism
and batch independence, and the fit without silhouettes unchanged with every argument error raised before any
launch."""
import numpy as np
import pytest
import torch
from scipy import ndimage

import lm_harness as harness
import silhouette_oracle as so
from lm_harness import bits
from shapy_b200 import _lib, ops
from shapy_b200.autograd import SilhouetteFunction

pytestmark = pytest.mark.gpu

F, PP = harness.F, harness.PP


def _blobs(H, W, seed, n=1):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        field = ndimage.gaussian_filter(rng.standard_normal((H, W)), max(1.0, min(H, W) / 20))
        out.append((field > np.quantile(field, 0.7)).astype(np.uint8))
    return np.stack(out)


def _special(H=48, W=64):
    one = np.zeros((H, W), np.uint8)
    one[17, 23] = 1
    border = np.zeros((H, W), np.uint8)
    border[:5, 10:30] = 1            # top
    border[-3:, :7] = 1              # bottom-left corner
    border[20:30, -4:] = 1           # right
    border[35:40, :2] = 1            # left
    return np.stack([one, np.ones((H, W), np.uint8), np.zeros((H, W), np.uint8), border])


def _check_prepare(masks, max_points):
    m = torch.from_numpy(masks).cuda()
    dist, contour, cw, count = ops.silhouette_prepare(m, max_points)
    dist, contour, cw, count = (t.cpu().numpy() for t in (dist, contour, cw, count))
    for b in range(masks.shape[0]):
        want = so.dist_f32(masks[b])
        assert (dist[b].view(np.uint32) == want.view(np.uint32)).all(), b
        pts, w, n = so.kept_contour(masks[b], max_points)
        assert count[b] == n and (contour[b] == pts).all() and (cw[b] == w).all(), (b, count[b], n)
    return count


@pytest.mark.parametrize('case', ['blobs512', 'blobs1000x750', 'one_by_one', 'special'])
def test_edt_and_contour_match_the_oracle(case):
    masks = {'blobs512': lambda: _blobs(512, 512, 0, 3), 'blobs1000x750': lambda: _blobs(1000, 750, 1, 2),
             'one_by_one': lambda: np.array([[[0]], [[1]]], np.uint8), 'special': _special}[case]()
    count = _check_prepare(masks, ops.MAX_SCAN_POINTS)
    small = max(1, int(count.max()) // 7)
    _check_prepare(masks, small)                          # past max_points: every k-th in raster order
    # bool masks are the same masks
    a = ops.silhouette_prepare(torch.from_numpy(masks).cuda(), 64)
    b = ops.silhouette_prepare(torch.from_numpy(masks != 0).cuda(), 64)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def _bodies(B, seed, tz=None):
    from test_gpu_fit_lm_kp2d_persp import _problem
    module = harness.smplx_module()
    _, _, init, tstar, bstar = _problem(module, B, seed=seed)
    if tz is not None:
        tstar = tstar.clone()
        tstar[:, 2] = tz
    with torch.no_grad():
        rot = ops.decode_rot6d(torch.cat([init['global_rot'], init['body_pose']], 1))
        v = module(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=bstar, transl=tstar,
                   return_shaped=False)['vertices'].contiguous()
    return module, v


def _intr(B, f=F, pp=PP):
    return torch.tensor([f, *pp]).repeat(B, 1).cuda()


def _compare_render(v, faces, intr, H, W):
    got = ops.render_silhouette(v, faces, intr, H, W).cpu().numpy()
    bad = 0
    for b in range(v.shape[0]):
        want, amb = so.rasterise(v[b].cpu().numpy(), faces.cpu().numpy(), intr[b].cpu().numpy(), H, W)
        bad += int(((got[b] != want) & ~amb).sum())
    return got, bad


def test_render_random_triangles_and_behind_the_camera():
    rng = np.random.default_rng(3)
    V, Fn, H, W = 60, 40, 90, 130
    Y = np.stack([rng.uniform(-1, 1, V), rng.uniform(-1, 1, V), rng.uniform(-0.5, 2.0, V)], 1).astype(np.float32)
    faces = torch.from_numpy(rng.integers(0, V, (Fn, 3)).astype(np.int32)).cuda()
    v = torch.from_numpy(Y).cuda()[None].repeat(2, 1, 1).contiguous()
    v[1, :, 2] += 1.0
    got, bad = _compare_render(v, faces, _intr(2, 60.0, (65.0, 45.0)), H, W)
    assert bad == 0 and got.any()
    assert (Y[:, 2] <= 0).sum() > 5           # some triangles are behind the camera


def test_render_bodies_far_and_near():
    module, v = _bodies(2, 11)
    faces = module.faces_i32
    got, bad = _compare_render(v, faces, _intr(2), 1000, 1000)
    assert bad == 0 and got.sum() > 10000
    # near the camera: triangles hundreds of pixels across, and vertices behind the camera
    _, v = _bodies(1, 12, tz=0.15)
    H = W = 400
    intr = _intr(1, 400.0, (200.0, 200.0))
    got, bad = _compare_render(v, faces, intr, H, W)
    uv = so.project_f32(v[0].cpu().numpy(), intr[0].cpu().numpy(), z_near=False)
    front = (v[0, :, 2].cpu().numpy() > 0)[faces.cpu().numpy()].all(1)
    ext = np.ptp(uv[faces.cpu().numpy()[front]], axis=1).max(1)
    print(f'[silhouette] near body: largest drawn triangle {ext.max():.0f} px, {int((~front).sum())} faces behind')
    assert bad == 0 and ext.max() > 100 and (~front).any()


def _case(B=2, seed=21, max_points=512):
    """Bodies, masks rendered from the bodies moved 2 cm, and the prepared masks."""
    module, v = _bodies(B, seed)
    intr = _intr(B)
    masks = ops.render_silhouette(v + torch.tensor([0.02, -0.02, 0.0], device='cuda'), module.faces_i32, intr, 1000,
                                  1000)
    return module, v, intr, masks, ops.silhouette_prepare(masks, max_points)


def test_closest_points_on_the_flat_projected_mesh():
    module, v, intr, masks, (dist, contour, cw, _) = _case()
    faces = module.faces_i32
    proj, _ = ops.silhouette_forward(v, intr, dist)
    face, bary, d2 = ops.closest_points(proj, faces, contour, cw)
    tree = ops.ScanTree()
    ops.closest_points(proj + 3.0, faces, contour, cw, tree=tree)
    refit = ops.closest_points(proj, faces, contour, cw, tree=tree)
    for x, y in zip((face, bary, d2), refit):
        assert torch.equal(bits(x) if x.dtype == torch.float32 else x, bits(y) if y.dtype == torch.float32 else y)
    worst, covered_max, n_cov = 0.0, 0.0, 0
    fc = faces.cpu().numpy()
    for b in range(v.shape[0]):
        keep = cw[b].cpu().numpy() > 0
        pts = contour[b].cpu().numpy()[keep, :2]
        uv = proj[b].cpu().numpy()[:, :2]
        dmin, all_d2 = so.closest_2d(pts, uv[fc])
        d = np.sqrt(d2[b].cpu().numpy()[keep].astype(np.float64))
        worst = max(worst, float(np.abs(d - np.sqrt(dmin)).max()))
        fi = face[b].cpu().numpy()[keep]
        assert (np.sqrt(all_d2[np.arange(len(fi)), fi]) <= np.sqrt(dmin) + 1e-4).all()
        cov, amb = so.rasterise(v[b].cpu().numpy(), fc, intr[b].cpu().numpy(), 1000, 1000)
        inside = cov[pts[:, 1].astype(int), pts[:, 0].astype(int)]
        n_cov += int(inside.sum())
        if inside.any():
            covered_max = max(covered_max, float(d[inside].max()))
    print(f'[silhouette] flat-mesh closest points: max |d - d64| {worst:.2e} px; {n_cov} covered contour pixels, '
          f'largest distance {covered_max:.2e} px')
    assert worst <= 1e-4 and n_cov > 0 and covered_max <= 1e-4


def test_term_and_gradient_match_the_oracle():
    module, v, intr, masks, (dist, contour, cw, _) = _case()
    faces = module.faces_i32
    n = cw.sum(1)
    inv = torch.where(n > 0, 1.0 / n.clamp(min=1.0), torch.zeros_like(n))
    vg = v.clone().requires_grad_(True)
    s = SilhouetteFunction.apply(vg, intr, faces, dist, contour, cw, inv, None)
    g_out = torch.tensor([1.0, 0.5], device='cuda')
    (s * g_out).sum().backward()
    proj, _ = ops.silhouette_forward(v, intr, dist)
    face, bary, _ = ops.closest_points(proj, faces, contour, cw)
    fc = faces.cpu().numpy()
    for b in range(v.shape[0]):
        args = (v[b].cpu().numpy(), intr[b].cpu().numpy(), dist[b].cpu().numpy())
        want = so.term(*args, contour[b].cpu().numpy(), cw[b].cpu().numpy(), fc)
        rel = abs(float(s[b]) - want) / want
        gw = so.gradient(*args, float(g_out[b]), contour[b].cpu().numpy(), cw[b].cpu().numpy(), fc,
                         face[b].cpu().numpy(), bary[b].cpu().numpy().astype(np.float64))
        gg = vg.grad[b].cpu().numpy().astype(np.float64)
        gerr = float(np.abs(gg - gw).max() / np.abs(gw).max())
        print(f'[silhouette] body {b}: term {float(s[b]):.4f} px^2, relative error {rel:.2e}; gradient error / max '
              f'{gerr:.2e}')
        assert rel <= 1e-5 and gerr <= 1e-4
        # directional derivatives of the model -> mask half against float64 central differences
        gm = so.gradient(*args, 1.0)
        rng = np.random.default_rng(b)
        checked = 0
        for _ in range(6):
            dirn = rng.standard_normal(args[0].shape)
            h = 1e-5
            # move only the vertices whose steps stay inside their bilinear cell
            cells = lambda y: so.cell_of(dist.shape[1:], *so.project_f32(y, args[1]).T)  # noqa: E731
            dirn[(cells(args[0] + h * dirn) != cells(args[0] - h * dirn)).any(1)] = 0
            a, c = args[0] + h * dirn, args[0] - h * dirn
            if not (cells(a) == cells(c)).all() or not dirn.any():
                continue
            fd = (so.model_to_mask_f64(a, args[1], args[2]) - so.model_to_mask_f64(c, args[1], args[2])) / (2 * h)
            np.testing.assert_allclose((gm * dirn).sum(), fd, rtol=2e-3, atol=1e-6)
            checked += 1
        assert checked >= 3


def test_deterministic_and_batch_independent():
    module, v8 = _bodies(8, 31)
    faces, intr = module.faces_i32, _intr(8)
    masks = ops.render_silhouette(v8 * 1.01, faces, intr, 600, 500)

    def run(v, m, it):
        prep = ops.silhouette_prepare(m, 1000)
        dist, contour, cw, _ = prep
        n = cw.sum(1)
        inv = torch.where(n > 0, 1.0 / n.clamp(min=1.0), torch.zeros_like(n))
        vg = v.clone().requires_grad_(True)
        s = SilhouetteFunction.apply(vg, it, faces, dist, contour, cw, inv, None)
        s.sum().backward()
        return list(prep) + [ops.render_silhouette(v, faces, it, 600, 500), s.detach(), vg.grad]

    r1, r2 = run(v8, masks, intr), run(v8, masks, intr)
    for x, y in zip(r1, r2):
        assert torch.equal(x, y)
    one = run(v8[5:6].contiguous(), masks[5:6].contiguous(), intr[5:6].contiguous())
    for x, y in zip(one, r1):
        x, y = x.contiguous(), y[5:6].contiguous()
        assert torch.equal(x.view(torch.uint8) if x.dtype != torch.bool else x,
                           y.view(torch.uint8) if y.dtype != torch.bool else y)


def test_fit_without_silhouettes_is_unchanged_and_errors_raise_before_any_launch():
    from shapy_b200.fit import fit_body_to_keypoints_2d
    from test_gpu_fit_lm_kp2d_persp import _problem
    module = harness.smplx_module()
    x, _, init, _, _ = _problem(module, 4, seed=41)
    kw = dict(focal_length=F, principal_point=PP, iterations=3)
    L = _lib.lib()
    torch.cuda.synchronize()
    n0 = L.shapy_launch_count()
    a = fit_body_to_keypoints_2d(module, x, init=dict(init), **kw)
    n1 = L.shapy_launch_count()
    b = fit_body_to_keypoints_2d(module, x, init=dict(init), silhouettes=None, silhouette_weight=5.0, **kw)
    n2 = L.shapy_launch_count()
    assert n1 - n0 == n2 - n1 and a.keys() == b.keys() and 'silhouette' not in a
    for k in a:
        if torch.is_tensor(a[k]):
            assert torch.equal(a[k], b[k]), k
    m = torch.zeros(4, 50, 60, dtype=torch.uint8)
    n0 = L.shapy_launch_count()
    bad = [dict(kw, silhouettes=m, method='lm'),
           dict(iterations=3, silhouettes=m),                                   # weak perspective
           dict(kw, silhouettes=m, groups=torch.tensor([0, 0, 1, 1])),
           dict(kw, silhouettes=m[:3]),
           dict(kw, silhouettes=m[0]),
           dict(kw, silhouettes=m.float()),
           dict(kw, silhouettes=torch.zeros(4, 5000, 10, dtype=torch.uint8)),
           dict(kw, silhouettes=m, max_silhouette_points=0),
           dict(kw, silhouettes=m, max_silhouette_points=ops.MAX_SCAN_POINTS + 1),
           dict(kw, silhouettes=m, silhouette_weight=-1.0),
           dict(kw, silhouettes=m, silhouette_weight=float('inf'))]
    for k in bad:
        with pytest.raises(ValueError):
            fit_body_to_keypoints_2d(module, x, init=dict(init), **k)
    with pytest.raises(ValueError):
        fit_body_to_keypoints_2d(module, x, init=dict(init), share_pose=True, groups=torch.tensor([0, 0, 1, 1]),
                                 silhouettes=m)
    mc = m.cuda()
    with pytest.raises(ValueError):
        ops.silhouette_prepare(torch.zeros(1, 4097, 3, dtype=torch.uint8, device='cuda'), 10)
    with pytest.raises(ValueError):
        ops.silhouette_prepare(mc, ops.MAX_SCAN_POINTS + 1)
    with pytest.raises(ValueError):
        ops.render_silhouette(torch.zeros(1, 3, 3, device='cuda'), module.faces_i32, _intr(1), 10, 4097)
    with pytest.raises(ValueError):
        ops.silhouette_forward(torch.zeros(1, 3, 3, device='cuda'), _intr(2), torch.zeros(1, 5, 5, device='cuda'))
    z = lambda *s: torch.zeros(*s, device='cuda')  # noqa: E731
    p = _lib.ptr
    ws = z(64)
    assert L.shapy_silhouette_prepare(p(mc), 4, 50, 4097, 10, *[p(ws)] * 5, 256, None) == -3
    assert L.shapy_silhouette_prepare(p(mc), 4, 50, 60, 32769, *[p(ws)] * 5, 256, None) == -3
    assert L.shapy_silhouette_prepare(p(mc), 4, 50, 60, 0, *[p(ws)] * 5, 256, None) == -1
    assert L.shapy_silhouette_prepare(p(mc), 4, 50, 60, 10, *[p(ws)] * 5, 4, None) == -1     # small workspace
    assert L.shapy_silhouette_prepare(None, 4, 50, 60, 10, *[p(ws)] * 5, 256, None) == -1
    assert L.shapy_silhouette_forward(p(ws), p(ws), p(ws), 1, 3, 4097, 5, p(ws), p(ws), None) == -3
    assert L.shapy_silhouette_forward(p(ws), None, p(ws), 1, 3, 5, 5, p(ws), p(ws), None) == -1
    assert L.shapy_silhouette_backward(p(ws), p(ws), p(ws), 1, 3, 5, 0, p(ws), None, p(ws), None) == -1
    assert L.shapy_silhouette_backward(p(ws), p(ws), p(ws), 1, 3, 5, 5, None, None, p(ws), None) == -1
    assert L.shapy_render_silhouette(p(ws), None, p(ws), 1, 3, 1, 5, 5, p(ws), None) == -1
    assert L.shapy_render_silhouette(p(ws), p(ws), p(ws), 1, 3, 1, 4097, 5, p(ws), None) == -3
    assert L.shapy_launch_count() == n0


def test_fit_reports_the_term_and_the_cli_writes_it(tmp_path):
    """The fit's 'silhouette' is the term at its final parameters, +inf (with the loss) for a body behind the camera;
    python -m shapy_b200.fit --silhouettes writes silhouette and silhouette_iou."""
    from shapy_b200 import fit
    from test_gpu_fit_lm_kp2d_persp import _problem
    module = harness.smplx_module()
    x, _, init, _, _ = _problem(module, 3, seed=43)
    intr = _intr(3)
    with torch.no_grad():
        rot = ops.decode_rot6d(torch.cat([init['global_rot'], init['body_pose']], 1))
        v = module(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=init['betas'], transl=init['transl'],
                   return_shaped=False)['vertices']
    masks = ops.render_silhouette(v * 1.02, module.faces_i32, intr, 700, 900)
    init['transl'][1, 2] = -3.0
    r = fit.fit_body_to_keypoints_2d(module, x, init=dict(init), iterations=5, focal_length=F, principal_point=PP,
                                     silhouettes=masks.cpu().numpy(), silhouette_weight=3.0)
    assert r['silhouette'][1] == float('inf') and r['loss'][1] == float('inf')
    dist, contour, cw, _ = ops.silhouette_prepare(masks, 4096)
    n = cw.sum(1)
    with torch.no_grad():
        vf = module(global_rot=r['global_rot_mat'], body_pose=r['body_pose_mat'], betas=r['betas'],
                    transl=r['transl'], return_shaped=False)['vertices'].contiguous()
        s = SilhouetteFunction.apply(vf, intr, module.faces_i32, dist, contour, cw, 1.0 / n, None)
        iou = [so.iou(a, b) for a, b in zip(ops.render_silhouette(vf, module.faces_i32, intr, 700, 900).cpu().numpy(),
                                              masks.cpu().numpy())]
    for b in (0, 2):
        assert float(r['silhouette'][b]) == pytest.approx(float(s[b]), rel=1e-6) and 0 < float(r['silhouette_iou'][b]) <= 1
        assert float(r['silhouette_iou'][b]) == pytest.approx(iou[b], rel=1e-6)
    from shapy_b200 import synth
    from shapy_b200.fit import _project
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    cli_model = SMPLX(data_struct=synth.make_smplx()).cuda()        # the command line's --synthetic model
    with torch.no_grad():
        j = cli_model(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=init['betas'], transl=init['transl'] * 0 +
                      torch.tensor([0.0, 0.0, 3.0], device='cuda'), return_shaped=False)['joints'][:]
        x = _project(j, intr)
    np.savez(tmp_path / 'kp.npz', keypoints=x.cpu().numpy(), focal_length=np.float32(F),
             principal_point=np.array(PP, np.float32))
    np.savez(tmp_path / 'masks.npz', masks=masks.cpu().numpy())
    out = tmp_path / 'fit.npz'
    fit.main(['--synthetic', '--keypoints-2d', str(tmp_path / 'kp.npz'), '--silhouettes', str(tmp_path / 'masks.npz'),
              '--silhouette-weight', '3', '--iterations', '4', '--output', str(out)])
    res = np.load(out)
    assert res['silhouette'].shape == (3,) and res['silhouette_iou'].shape == (3,)
    assert np.isfinite(res['silhouette']).all() and (res['silhouette_iou'] > 0).all()
