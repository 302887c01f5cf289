"""The measurement kernel on constructed slices (tests/measure_slices.py), through its entries: vertices + faces
(staged in shared memory), triangles, and vertices + faces too many to stage (V = 20 000, gathered from global memory).

  point sets     bit for bit the float C oracle's, face 0 excluded
  circumference  vs the exact hull's float64 perimeter of the kernel's own points (isolates hull + sum), and vs
                 qhull on the oracle's points
  mass           vs a float64 sum of the same per-face terms, bar c * 2^-24 * sum |products|; height exact
  capacity       1 024 points and 8 192 candidates per body in every entry; NaN + status past them
  entries        the same rows, status, counts and point sets from every entry, bit for bit
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
MASS_C = 2.0            # |mass - ref| <= MASS_C * 2^-24 * sum|products| (+ the final division's rounding); measured 0.21
MAXP = 1100
ENTRIES = ('vertices', 'triangles', 'vertices_global')
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
    """meshes share faces and landmarks; returns out (B,5), pts, cnt, status as numpy.  'vertices_global' pads the
    meshes with unused vertices past what the kernel stages in shared memory."""
    if entry == 'vertices_global':
        meshes, entry = [m.padded() for m in meshes], 'vertices'
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
            _note(f'hull vs exact [{fam}, {entry}]', err)
            assert err <= BAR_HULL, (fam, entry, b, p, val, exact)
            sp = _scipy_perimeter(ref)
            _note(f'hull vs qhull [{fam}, {entry}]', abs(val - sp) / sp)
            assert abs(val - sp) <= BAR_HULL * sp, (fam, entry, b, p, val, sp)
    assert (st != 0) == any_over, (fam, entry, st)


@pytest.mark.parametrize('fam', list(FAMILIES))
def test_entries_bit_identical(ops, fam):
    """Every entry runs the same phases on the same triangles: equal rows as bits (NaN included), status and counts,
    and equal point sets wherever nothing was truncated."""
    meshes = _rows(FAMILIES[fam])
    runs = {e: _run(ops, meshes, e) for e in ENTRIES}
    out, pts, cnt, st = runs['vertices']
    cand_over = ms.candidate_count(meshes[0]) > ms.CAP_CAND
    for e in ENTRIES[1:]:
        o, p, c, s = runs[e]
        assert np.array_equal(o.view(np.int32), out.view(np.int32)), (fam, e, o, out)
        assert s == st, (fam, e, s, st)
        if cand_over:
            continue                                  # truncated candidate queues: which points were kept is open
        assert np.array_equal(c, cnt), (fam, e, c, cnt)
        for r, mesh in enumerate(meshes):
            for q in range(3):
                if len(ms.oracle_points(mesh, q)) > ms.CAP_POINTS:
                    continue
                n = int(cnt[r, q])
                assert np.array_equal(_bits_sorted(p[r, q, :n]), _bits_sorted(pts[r, q, :n])), (fam, e, r, q)


def test_capacity_1024_everywhere(ops):
    """1 024 points on a plane (with 4 696 candidates): a value and status 0 from every entry, the same bits from
    all of them."""
    m = FAMILIES['count1024']
    runs = {e: _run(ops, [m], e) for e in ENTRIES}
    for e, (out, _, cnt, st) in runs.items():
        assert st == 0 and not np.isnan(out).any() and list(cnt[0]) == [1024, 1024, 300], (e, out, cnt)
    out, pts, cnt, _ = runs['vertices']
    for e in ENTRIES[1:]:
        assert np.array_equal(runs[e][0].view(np.int32), out.view(np.int32)), (e, runs[e][0], out)
        for p in range(3):
            n = cnt[0, p]
            assert np.array_equal(_bits_sorted(runs[e][1][0, p, :n]), _bits_sorted(pts[0, p, :n])), (e, p)


@pytest.mark.parametrize('entry', ENTRIES)
def test_capacity_overflow(ops, entry):
    """1 025 points: NaN on that plane only, status set.  More than 8 192 candidates: NaN on all three planes."""
    out, _, cnt, st = _run(ops, [FAMILIES['count1025']], entry)
    assert st == 1 and np.isnan(out[0, 2]) and not np.isnan(out[0, [0, 1, 3, 4]]).any(), out
    assert list(cnt[0]) == [1024, 1024, 300]
    out, _, _, st = _run(ops, [FAMILIES['overhang1400']], entry)
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
