"""The measurement kernels on constructed slices (tests/measure_slices.py), through both entries: vertices + faces
(measure_smem_kernel, or measure_kernel beyond its shared memory) and triangles (measure_kernel).

  point sets     bit for bit the float C oracle's, face 0 excluded
  circumference  vs the exact hull's float64 perimeter of the kernel's own points (isolates hull + sum), and vs
                 qhull on the oracle's points
  mass           vs a float64 sum of the same per-face terms, bar c * 2^-24 * sum |products|; height exact
  capacity       1 024 points and 8 192 candidates per body in every entry; NaN + status past them
  degenerate     fewer than 3 points, collinear or coincident in xz: NaN
  determinism    64 copies give identical rows; permuted faces give bit-identical circumferences
The largest error of each family is printed by test_zz_report (pytest -s)."""
import numpy as np
import pytest
import torch
from scipy.spatial import ConvexHull

import measure_slices as ms
from oracle import hull_exact

pytestmark = pytest.mark.gpu

BAR_HULL = 2e-6         # kernel vs exact hull of its own points, and vs qhull on the oracle's points
BAR_V1V2 = 2e-6         # the two kernels: same hull, different fp32 summation order
# measure_kernel sums a plane's k hull edges in one fp32 running sum (measure_smem_kernel in 8 chains of about k / 8),
# whose worst-case relative error grows as k * 2^-24 (6.1e-5 at k = 1 024).  Rounding errors of that many terms add
# up far below the worst case: 3.7e-6 measured at k = 1 024 (H100).  The bar is an eighth of the worst case, twice the
# measurement, and 2e-6 up to k = 268 (which covers every plane but the 333-, 500- and 1 024-vertex ones).
MASS_C = 2.0            # |mass - ref| <= MASS_C * 2^-24 * sum|products| (+ the final division's rounding); measured 0.21
MAXP = 1100
WORST = {}


def _note(key, val):
    WORST[key] = max(WORST.get(key, 0.0), float(val))


@pytest.fixture(scope='module')
def ops():
    from shapy_b200 import ops
    return ops


def _families():
    return ms.value_families() + [ms.exact_count(1025), ms.overhang(1400)]


FAMILIES = {m.meta['family']: m for m in _families()}


def _run(ops, meshes, entry, max_points=MAXP):
    """meshes share faces and landmarks; returns out (B,5), pts, cnt, status as numpy."""
    m0 = meshes[0]
    lm = ops.make_landmarks(m0.lm)
    if entry == 'vertices':
        v = torch.from_numpy(np.stack([m.verts for m in meshes])).cuda()
        r = ops.measure(lm, v_shaped=v, faces_i32=torch.from_numpy(m0.faces).cuda(), return_points=True,
                        max_points=max_points)
    else:
        t = torch.from_numpy(np.stack([m.tris for m in meshes])).cuda()
        r = ops.measure(lm, triangles=t, return_points=True, max_points=max_points)
    out, pts, cnt, st = r
    return out.cpu().numpy(), pts.cpu().numpy(), cnt.cpu().numpy(), int(st.item())


def _bits_sorted(p):
    return np.sort(np.ascontiguousarray(p, np.float32).view(np.int32).view([('x', np.int32), ('y', np.int32),
                                                                            ('z', np.int32)]).ravel())


def _scipy_perimeter(p):
    h = ConvexHull(p[:, [0, 2]].astype(np.float64))
    seg = p[h.simplices.reshape(-1)].reshape(-1, 2, 3).astype(np.float64)
    return float(np.sqrt(((seg[:, 1] - seg[:, 0]) ** 2).sum(-1)).sum())


def _mass_ref(mesh):
    t = mesh.tris.astype(np.float64)
    x, y, z = t[..., 0], t[..., 1], t[..., 2]
    prods = np.stack([-x[:, 2] * y[:, 1] * z[:, 0], x[:, 1] * y[:, 2] * z[:, 0], x[:, 2] * y[:, 0] * z[:, 1],
                      -x[:, 0] * y[:, 2] * z[:, 1], -x[:, 1] * y[:, 0] * z[:, 2], x[:, 0] * y[:, 1] * z[:, 2]])
    return abs(prods.sum()) / 6 * 985, np.abs(prods).sum() / 6 * 985


def _height_ref(mesh):
    t = mesh.tris
    ys = []
    for k in ('head_top', 'left_heel'):
        bc = np.asarray(mesh.lm[k]['bc'], np.float32)
        y = t[mesh.lm[k]['face_idx'], :, 1]
        ys.append(np.float32(np.float32(y[0] * bc[0] + y[1] * bc[1]) + y[2] * bc[2]))
    return np.float32(abs(np.float32(ys[0] - ys[1])))


def _sum_bar(bar, pts):
    h = hull_exact.hull_indices(pts)
    return max(bar, (0 if h is None else len(h)) * 2 ** -27)


def _check_mass_height(fam, mesh, row):
    ref, scale = _mass_ref(mesh)
    err = abs(float(row[0]) - ref)
    _note(f'mass c [{fam}]', (err - 4 * 2 ** -24 * ref) / (2 ** -24 * scale))
    assert err <= MASS_C * 2 ** -24 * scale + 4 * 2 ** -24 * ref, (fam, row[0], ref, scale)
    assert row[1] == _height_ref(mesh), (fam, row[1])


def _rows(mesh):
    return [mesh, mesh.translated((0.0, 0.25, 0.0))]


@pytest.mark.parametrize('entry', ['vertices', 'triangles'])
@pytest.mark.parametrize('fam', list(FAMILIES))
def test_family_vs_oracle_and_exact_hull(ops, fam, entry):
    meshes = _rows(FAMILIES[fam])
    out, pts, cnt, st = _run(ops, meshes, entry)
    cand_over = ms.candidate_count(meshes[0]) > ms.CAP_CAND
    any_over = cand_over
    for b, mesh in enumerate(meshes):
        _check_mass_height(fam, mesh, out[b])
        for p in range(3):
            ref = ms.oracle_points(mesh, p)
            n = len(ref)
            val = float(out[b, 2 + p])
            if cand_over:
                assert np.isnan(val), (fam, entry, b, p, val)
                continue
            if n > ms.CAP_POINTS:
                any_over = True
                assert np.isnan(val) and cnt[b, p] == ms.CAP_POINTS, (fam, entry, b, p, val, cnt[b, p])
                continue
            assert cnt[b, p] == n, (fam, entry, b, p, cnt[b, p], n)
            mine = pts[b, p, :n]
            assert np.array_equal(_bits_sorted(mine), _bits_sorted(ref)), (fam, entry, b, p)
            exact = hull_exact.perimeter(mine)
            if np.isnan(exact):
                assert np.isnan(val), (fam, entry, b, p, n, val)
                continue
            err = abs(val - exact) / exact
            bar = BAR_HULL if entry == 'vertices' else _sum_bar(BAR_HULL, mine)
            _note(f'hull vs exact [{fam}, {entry}] (bar {bar:.2g})', err)
            assert err <= bar, (fam, entry, b, p, val, exact, bar)
            sp = _scipy_perimeter(ref)
            _note(f'hull vs qhull [{fam}, {entry}] (bar {bar:.2g})', abs(val - sp) / sp)
            assert abs(val - sp) <= bar * sp, (fam, entry, b, p, val, sp, bar)
    assert (st != 0) == any_over, (fam, entry, st)


@pytest.mark.parametrize('fam', list(FAMILIES))
def test_v1_vs_v2(ops, fam):
    meshes = _rows(FAMILIES[fam])
    a = _run(ops, meshes, 'vertices')
    b = _run(ops, meshes, 'triangles')
    assert np.array_equal(np.isnan(a[0]), np.isnan(b[0])) and a[3] == b[3]
    for r in range(len(meshes)):
        for p in range(3):
            if np.isnan(a[0][r, 2 + p]):
                continue
            rel = abs(a[0][r, 2 + p] - b[0][r, 2 + p]) / abs(b[0][r, 2 + p])
            bar = _sum_bar(BAR_V1V2, b[1][r, p, :b[2][r, p]])
            _note(f'v1 vs v2 [{fam}] (bar {bar:.2g})', rel)
            assert rel <= bar, (fam, r, p, rel, bar)
    if ms.candidate_count(meshes[0]) > ms.CAP_CAND:
        return                                        # truncated candidate queues: which points were kept is open
    assert np.array_equal(a[2], b[2])
    for r in range(len(meshes)):
        for p in range(3):
            n = int(a[2][r, p])
            if len(ms.oracle_points(meshes[r], p)) > ms.CAP_POINTS:
                continue
            assert np.array_equal(_bits_sorted(a[1][r, p, :n]), _bits_sorted(b[1][r, p, :n])), (fam, r, p)


def test_capacity_1024_everywhere(ops):
    """1 024 points on a plane (with 4 696 candidates): a value and status 0 from the vertices entry, the triangles
    entry, and the vertices entry at V = 20 000 (measure_kernel, as the triangles entry)."""
    m = FAMILIES['count1024']
    runs = {e: _run(ops, [m], e) for e in ('vertices', 'triangles')}
    runs['vertices_v1'] = _run(ops, [m.padded()], 'vertices')
    for e, (out, _, cnt, st) in runs.items():
        assert st == 0 and not np.isnan(out).any() and list(cnt[0]) == [1024, 1024, 300], (e, out, cnt)
    assert np.array_equal(runs['vertices_v1'][0], runs['triangles'][0])
    for p in range(3):
        n = runs['triangles'][2][0, p]
        assert np.array_equal(_bits_sorted(runs['vertices_v1'][1][0, p, :n]), _bits_sorted(runs['triangles'][1][0, p, :n]))


@pytest.mark.parametrize('entry', ['vertices', 'triangles', 'vertices_v1'])
def test_capacity_overflow(ops, entry):
    """1 025 points: NaN on that plane only, status set.  More than 8 192 candidates: NaN on all three planes."""
    pad = entry == 'vertices_v1'
    e = 'vertices' if pad else entry
    m = FAMILIES['count1025']
    out, _, cnt, st = _run(ops, [m.padded() if pad else m], e)
    assert st == 1 and np.isnan(out[0, 2]) and not np.isnan(out[0, [0, 1, 3, 4]]).any(), out
    assert list(cnt[0]) == [1024, 1024, 300]
    m = FAMILIES['overhang1400']
    out, _, _, st = _run(ops, [m.padded() if pad else m], e)
    assert st == 1 and np.isnan(out[0, 2:]).all() and not np.isnan(out[0, :2]).any(), out


@pytest.mark.parametrize('entry', ['vertices', 'triangles'])
def test_max_points_truncates_returned_points_only(ops, entry):
    m = FAMILIES['ngon64']
    full = _run(ops, [m], entry)
    out, pts, cnt, st = _run(ops, [m], entry, max_points=16)
    assert st == 1 and np.array_equal(out, full[0]) and np.array_equal(cnt, full[2])
    for p in range(3):
        ref = set(_bits_sorted(ms.oracle_points(m, p)).tolist())
        got = _bits_sorted(pts[0, p]).tolist()
        assert len(got) == 16 and all(g in ref for g in got)


@pytest.mark.parametrize('entry', ['vertices', 'triangles'])
def test_degenerate_slices(ops, entry):
    """n < 3, collinear and coincident slices are NaN (qhull raises on them); 3 points give the triangle."""
    out = _run(ops, [FAMILIES['degenerate']], entry)[0][0]
    assert np.isnan(out[2]) and np.isnan(out[3]) and not np.isnan(out[4]), out
    m = FAMILIES['small_counts']
    out = _run(ops, [m], entry)[0][0]
    assert np.isnan(out[3]) and np.isnan(out[4]), out
    p = ms.oracle_points(m, 0).astype(np.float64)
    tri = sum(np.linalg.norm(p[i] - p[(i + 1) % 3]) for i in range(3))
    assert abs(out[2] - tri) <= 1e-6 * tri, (out[2], tri)
    out = _run(ops, [FAMILIES['obtuse']], entry)[0][0]
    for k in range(3):
        p = ms.oracle_points(FAMILIES['obtuse'], k).astype(np.float64)
        tri = sum(np.linalg.norm(p[i] - p[(i + 1) % 3]) for i in range(3))
        assert abs(out[2 + k] - tri) <= 1e-6 * tri, (k, out[2 + k], tri)


@pytest.mark.parametrize('entry', ['vertices', 'triangles'])
@pytest.mark.parametrize('fam', ['identical_xz', 'arc_cluster', 'subdivided_square', 'ngon333'])
def test_determinism(ops, fam, entry):
    """64 copies in one batch give bit-identical rows; permuted faces give bit-identical circumferences and height
    (the mass is a sum in face order: within its bar)."""
    m = FAMILIES[fam]
    out = _run(ops, [m] * 64, entry)[0]
    assert (out.view(np.int32) == out[:1].view(np.int32)).all(), fam
    for seed in (1, 2, 3):
        q = m.permuted(seed)
        o = _run(ops, [q], entry)[0]
        assert np.array_equal(o[0, 1:].view(np.int32), out[0, 1:].view(np.int32)), (fam, seed, o[0], out[0])
        _check_mass_height(fam, q, o[0])


def test_mass_far_from_origin(ops):
    """A body 2.5 m from the origin, triangles entry: the fp32 sum of the signed volumes cancels heavily."""
    for fam in ('ngon500', 'count1024'):
        m = FAMILIES[fam].translated((2.5, 0.0, 0.0))
        out = _run(ops, [m], 'triangles')[0][0]
        _check_mass_height(fam + '@2.5m', m, out)


def test_zz_report(capsys):
    with capsys.disabled():
        print(f'\nlargest measured errors (mass: c, bar {MASS_C:g}):')
        for k in sorted(WORST):
            print(f'  {k:60s} {WORST[k]:.3g}')
