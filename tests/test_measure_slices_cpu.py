"""The constructed slices of tests/measure_slices.py reach the edge cases they are named for, on the float C oracle
(bit-exact with the kernels' predicates: both are compiled without FMA contraction); and the exact hull of
oracle/hull_exact.py agrees with qhull where qhull gives an answer.  No GPU."""
import numpy as np
import pytest
from scipy.spatial import ConvexHull

import measure_slices as ms
from oracle import hull_exact


@pytest.fixture(scope='module')
def fam():
    out = {m.meta['family']: m for m in ms.value_families() + [ms.exact_count(1025), ms.overhang(1400)]}
    return out


@pytest.fixture(scope='module')
def pts(fam):
    return {k: [ms.oracle_points(m, p) for p in range(3)] for k, m in fam.items()}


def _scipy_perimeter(p):
    h = ConvexHull(p[:, [0, 2]].astype(np.float64))
    seg = p[h.simplices.reshape(-1)].reshape(-1, 2, 3).astype(np.float64)
    return float(np.sqrt(((seg[:, 1] - seg[:, 0]) ** 2).sum(-1)).sum())


def test_point_counts(pts):
    n = {k: [len(p) for p in v] for k, v in pts.items()}
    assert n['small_counts'] == [3, 2, 0]
    assert n['obtuse'] == [3, 3, 3]
    assert n['degenerate'][:2] == [5, 3]
    assert n['count1024'] == [1024, 1024, 300]
    assert n['count1025'] == [1025, 1024, 300]
    assert n['arc_cluster'][0] > ms.CHAIN_CAP and n['arc_cluster'][0] <= ms.CAP_POINTS
    for k, v in n.items():
        if k != 'count1025':
            assert max(v) <= ms.CAP_POINTS, (k, v)
    assert n['clipped'][1] > 0


def test_hull_exact_matches_scipy(pts):
    rng = np.random.default_rng(0)
    sets = [rng.normal(size=(n, 3)).astype(np.float32) for n in (3, 4, 10, 100, 1000)]
    sets += [p for v in pts.values() for p in v if len(p) >= 3 and hull_exact.hull_indices(p) is not None]
    assert len(sets) > 40
    for p in sets:
        mine, ref = hull_exact.perimeter(p), _scipy_perimeter(p)
        assert abs(mine - ref) <= 1e-12 * ref, (mine, ref)


def test_zero_area_sets(pts):
    """Collinear and coincident sets: the exact hull reports zero area, and qhull raises on them."""
    from scipy.spatial import QhullError
    collinear, coincident = pts['degenerate'][0], pts['degenerate'][1]
    assert np.all(collinear[:, 2] == 0) and len(np.unique(collinear[:, 0])) == 5
    assert len(np.unique(coincident, axis=0)) == 1
    for p in (collinear, coincident, pts['small_counts'][1]):
        assert hull_exact.hull_indices(p) is None and np.isnan(hull_exact.perimeter(p))
    for p in (collinear, coincident):
        with pytest.raises(QhullError):
            ConvexHull(p[:, [0, 2]].astype(np.float64))
    assert not np.isnan(hull_exact.perimeter(pts['small_counts'][0]))


def test_chain_over_640_outer_points(pts):
    """arc_cluster: one chord of the 8-extreme split has more than 640 points on its outer side, so that chain's
    candidate list overflows and the kernel scans every point.  The chain's 16 hull vertices each carry more than
    2e-6 of the perimeter, so a scan that missed any of them fails the 2e-6 hull bar of the GPU tests."""
    for p in (pts['arc_cluster'][0], pts['arc_cluster'][2]):
        assert len(p) == 1000 and max(ms.chain_sizes(p)) > ms.CHAIN_CAP
        h = hull_exact.hull_indices(p)
        full = hull_exact.perimeter(p)
        arc = [i for i in h if p[i, 0] > 0.6]          # the arc needles (the anchors are at x <= 0.2)
        assert len(arc) == 16
        for i in arc[1:-1]:                            # the two ends are the chain's extremes
            short = hull_exact.perimeter(np.delete(p, i, axis=0))
            assert (full - short) / full > 2e-6, (i, (full - short) / full)


def test_hull_vertex_not_extreme(pts):
    """obtuse: the obtuse vertex is a hull vertex, but extreme in none of the 8 directions."""
    p = pts['obtuse'][0]
    e = set(ms.extremes(p))
    assert len(e) == 2 and len(hull_exact.hull_indices(p)) == 3
    assert max(ms.chain_sizes(p)) == 3


def test_exact_ties_and_collinear_points(pts):
    """subdivided_square: each side holds its subdivision points exactly on the hull edge, and the keys of the axis
    directions tie exactly (a whole side shares x or z), so the tie-break picks the extreme."""
    for p in pts['subdivided_square']:
        xs = p[:, 0]
        assert (xs == xs.max()).sum() > 10 and (xs == xs.min()).sum() > 10
        for k in (0, 2, 4, 6):                      # the axis directions: a whole side ties
            keys = [ms._key(a[0], a[2], k)[0] for a in p]
            assert sum(1 for x in keys if x == max(keys)) >= 2, k
        assert len(hull_exact.hull_indices(p)) == 4


def test_identical_xz_pair(pts):
    for p in (pts['identical_xz'][0], pts['identical_xz'][2]):
        at = p[(p[:, 0] == np.float32(0.5)) & (p[:, 2] == 0)]
        assert len(at) == 2 and at[0, 1] != at[1, 1]
        assert any(p[i, 0] == np.float32(0.5) for i in hull_exact.hull_indices(p))


def test_plane_through_vertices_and_face0(fam, pts):
    m = fam['through_vertices']
    ys = m.verts[:, 1]
    for p in (0, 1):
        assert (ys == m.heights()[p]).sum() >= 16
    m = fam['face0_crossing']
    t0 = m.tris[0]
    assert t0[:, 1].min() < m.heights()[0] < t0[:, 1].max() and np.abs(t0[:, [0, 2]]).max() < 1
    # the oracle with face 0 admitted would add its points
    from oracle import measure_oracle
    f, _ = measure_oracle.mesh_to_mesh_forward(measure_oracle.plane_quad(m.heights()[0])[None], m.tris[None], 4096)
    assert (f[0] == 0).any()


def test_candidate_counts(fam, pts):
    """overhang1400 passes 8192 candidates with every plane at 1024 points or fewer; count1024 and overhang700 sit
    between 4096 and 8192."""
    assert ms.candidate_count(fam['overhang1400']) > ms.CAP_CAND
    assert max(len(p) for p in pts['overhang1400']) <= ms.CAP_POINTS
    for k in ('count1024', 'overhang700'):
        assert 4096 < ms.candidate_count(fam[k]) <= ms.CAP_CAND, k


def test_padded_mesh_leaves_shared_memory():
    """V = 20 000: staging the vertices would take more than the 220 KB of shared memory the kernel may use, so the
    vertices entry gathers them from global memory."""
    V = ms.GLOBAL_VERTS_V
    assert ((V * 12 + 15) & ~15) + 3 * 1024 * 12 + 8192 * 4 > 220 * 1024
    m = ms.exact_count(ms.CAP_POINTS).padded()
    assert m.verts.shape == (V, 3) and m.faces.max() < V


def test_permutation_keeps_slices(fam):
    m = fam['identical_xz']
    q = m.permuted(1)
    assert q.heights() == m.heights() and not np.array_equal(q.faces, m.faces)
    for p in range(3):
        a, b = ms.oracle_points(m, p), ms.oracle_points(q, p)
        assert np.array_equal(np.sort(a.view(np.int32), 0), np.sort(b.view(np.int32), 0))
