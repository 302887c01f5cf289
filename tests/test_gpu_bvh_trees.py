"""GPU: the LBVH queries of shapy_b200/csrc/bvh.cu on trees built to break them, against restatements of the same
operations.  Closest and nearest points equal the float32 restatement of tests/bvh_f32_oracle.py bit for bit (the
lexicographic minimum of (float32 d2, index) over every primitive), on a fresh tree and on a tree built on scrambled
vertex positions and then refit; the backward matches tests/scan_oracle.py; self-collisions match
tests/penetration_oracle.py pair for pair; mesh_to_mesh_forward matches the plain-C oracles.

The scenes: tree sizes around powers of two up to the 32768 limit (u16 ids), all primitives identical (one Morton
code), coplanar and collinear scenes (a zero extent in the Morton normalisation), a 1000 m outlier that collapses the
body into one Morton cell, the synthetic SMPL-X body 3 m from the origin with queries 1 um to 1 cm from its shared
vertices and edges, the same body with every face listed twice, the flat projected mesh in pixels, far queries, NaN
and zero weights.  Every call runs two or more bodies with different scenes."""
import numpy as np
import pytest
import torch

import bvh_f32_oracle as bo
import penetration_oracle as po
import scan_oracle as so
from oracle import measure_oracle, mmi_oracle_f64
from shapy_b200 import ops

pytestmark = pytest.mark.gpu

GRAD_BAR = 5e-7          # tests/test_gpu_scan.py's bar on the backward, relative to its largest entry


def _bits(x):
    return np.ascontiguousarray(x).view(np.uint32)


def _cuda(x, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(x)).to('cuda', dtype)


def _closest(v, faces, p, w=None, tree=None):
    """faces: a CUDA int32 tensor (a tree refits only for the same faces tensor) or an array."""
    faces = faces if torch.is_tensor(faces) else _cuda(faces, torch.int32)
    out = ops.closest_points(_cuda(v), faces, _cuda(p), None if w is None else _cuda(w), tree=tree)
    return [t.cpu().numpy() for t in out]


def check_closest(v, faces, p, w=None, scramble=True, seed=0):
    """v (B, V, 3), p (B, N, 3): ops.closest_points equals the restatement bit for bit on a fresh tree and on a tree
    built on a permutation of the vertex positions and then refit.  Returns the kernel's (face, bary, d2)."""
    face, bary, d2 = _closest(v, faces, p, w)
    for b in range(len(v)):
        wf, wb, wd = bo.closest_points(v[b], faces, p[b], None if w is None else w[b])
        bad = np.nonzero(face[b] != wf)[0]
        assert len(bad) == 0, (b, bad[:5], face[b][bad[:5]], wf[bad[:5]], d2[b][bad[:5]], wd[bad[:5]])
        assert np.array_equal(_bits(d2[b]), _bits(wd)), b
        assert np.array_equal(_bits(bary[b]), _bits(wb)), b
    if scramble:
        rng = np.random.default_rng(seed)
        perm = np.stack([rng.permutation(v.shape[1]) for _ in range(len(v))])
        tree, ff = ops.ScanTree(), _cuda(faces, torch.int32)
        _closest(np.take_along_axis(v, perm[:, :, None], 1), ff, p, w, tree=tree)
        key = tree.key
        refit = _closest(v, ff, p, w, tree=tree)
        assert tree.key == key                              # the second call refit the scrambled tree
        for x, y in zip((face, bary, d2), refit):
            assert np.array_equal(_bits(x), _bits(y))
    return face, bary, d2


def soup(B, P, seed, off=0.0, size=0.02, spread=1.0):
    """B bodies of P random triangles (different per body): vertices (B, 3P, 3) and faces (P, 3)."""
    rng = np.random.default_rng(seed)
    c = off + spread * rng.uniform(-0.5, 0.5, (B, P, 1, 3))
    v = (c + size * rng.normal(size=(B, P, 3, 3))).reshape(B, 3 * P, 3).astype(np.float32)
    return v, np.arange(3 * P, dtype=np.int32).reshape(P, 3)


def near_queries(v, n, seed, lo=-6, hi=-1, spread=1.0):
    """n queries per body around the body's vertices, at 10^lo to 10^hi times `spread` from them."""
    rng = np.random.default_rng(seed)
    out = []
    for vb in v:
        base = vb[rng.integers(len(vb), size=n)].astype(np.float64)
        d = rng.normal(size=(n, 3))
        d *= spread * 10 ** rng.uniform(lo, hi, (n, 1)) / np.linalg.norm(d, axis=1, keepdims=True)
        out.append(base + d)
    return np.stack(out).astype(np.float32)


# ------------------------------------------------------------------------------------------- closest points
@pytest.mark.parametrize('P', [1, 2, 3, 31, 32, 33, 1023, 1024, 1025, 32767, 32768])
def test_closest_points_at_tree_sizes(P):
    v, faces = soup(2, P, P, off=np.array([0.0, 3.0])[:, None, None, None], spread=max(0.1, (P / 1000) ** (1 / 3)))
    n = 128 if P > 2000 else 256
    p = near_queries(v, n, P + 1, spread=0.1)
    check_closest(v, faces, p, scramble=P > 1, seed=P)


def test_closest_points_identical_coplanar_collinear_and_outlier_scenes():
    rng = np.random.default_rng(11)
    P = 1000
    tri = np.float32([[0.1, 0.2, 0.3], [0.15, 0.2, 0.31], [0.1, 0.26, 0.29]])
    same = np.broadcast_to(tri, (P, 3, 3)).reshape(-1, 3)                   # one Morton code
    plane = rng.uniform(-1, 1, (P, 3, 3)) * [1, 1, 0] + rng.uniform(-1, 1, (P, 1, 3)) * [1, 1, 0]
    line = (rng.uniform(-1, 1, (P, 3, 1)) * 0.05 + rng.uniform(-1, 1, (P, 1, 1))) * [1.0, 0, 0] + [0, 2.0, -1.0]
    out, _ = soup(1, P, 12)
    out = out[0].reshape(P, 3, 3)
    out[7] += 1000.0                                                        # the rest share one Morton cell
    faces = np.arange(3 * P, dtype=np.int32).reshape(P, 3)
    v = np.stack([same, plane.reshape(-1, 3), line.reshape(-1, 3), out.reshape(-1, 3)]).astype(np.float32)
    p = near_queries(v, 256, 13, lo=-7, hi=0)
    p[:, :16] = rng.uniform(-2, 2, (4, 16, 3))
    p[1, 16:32, 2] = 0.0                                                    # queries in the plane
    face, _, _ = check_closest(v, faces, p, seed=14)
    assert (face[0] == 0).all()                                             # identical faces: the smallest index


@pytest.fixture(scope='module')
def body():
    from test_gpu_scan import _bodies, _model
    v = _bodies(2, 31).cpu().numpy() + np.float32([3.0, -3.0, 3.0])          # 3 m from the origin
    return v.astype(np.float32), _model().faces_tensor.cpu().numpy().astype(np.int32)


def _shared_queries(v, faces, n, seed):
    """Per body n queries 1 um to 1 cm from vertices and edge midpoints of the mesh (where faces meet)."""
    rng = np.random.default_rng(seed)
    out = []
    for vb in v.astype(np.float64):
        f = faces[rng.integers(len(faces), size=n)]
        k = rng.integers(3, size=n)
        a, b = vb[f[np.arange(n), k]], vb[f[np.arange(n), (k + 1) % 3]]
        t = np.where(rng.random(n) < 0.5, 0.0, rng.uniform(0, 1, n))[:, None]
        d = rng.normal(size=(n, 3))
        d *= 10 ** rng.uniform(-6, -2, (n, 1)) / np.linalg.norm(d, axis=1, keepdims=True)
        out.append(a + t * (b - a) + d)
    return np.stack(out).astype(np.float32)


def test_closest_points_on_the_offset_body_and_its_duplicated_faces(body):
    v, faces = body
    p = _shared_queries(v, faces, 512, 32)
    p[:, :32] += np.float32([100.0, 0, 0])                                 # far queries
    w = np.ones(p.shape[:2], np.float32)
    w[:, 40::17], w[:, 41::17] = 0.0, np.nan
    p[:, 42::17] = np.nan                                                   # a NaN point of weight 1: no face wins
    face, bary, d2 = check_closest(v, faces, p, w, seed=33)
    assert (face[:, 40::17] == -1).all() and (face[:, 41::17] == -1).all() and (face[:, 42::17] == -1).all()
    # every face listed twice (the first 16000 faces, so that 2F stays within the 32768 supported)
    F = 16000
    part = check_closest(v, faces[:F], p, w, scramble=False)
    dup = check_closest(v, np.concatenate([faces[:F], faces[:F]]), p, w, seed=34)
    assert (dup[0] < F).all()
    for x, y in zip(part, dup):
        assert np.array_equal(_bits(x), _bits(y))


def test_closest_points_on_the_flat_projected_mesh(body):
    v, faces = body
    # a pinhole camera 3 m in front of the body, in pixels of a 1000 x 1000 image, z = 0
    c = v - v.mean(1, keepdims=True)
    z = c[..., 2:] + 3.0
    uv = 1500.0 * c[..., :2] / z + 500.0
    flat = np.concatenate([uv, np.zeros_like(z)], -1).astype(np.float32)
    flat[1] = flat[1][:, [1, 0, 2]]                                         # a different scene on body 1
    p = near_queries(flat, 512, 41, lo=-4, hi=1.5)
    p[..., 2] = 0.0
    p[:, :64, :2] = np.round(p[:, :64, :2])                                 # pixel centres
    check_closest(flat, faces, p, seed=42)


# ------------------------------------------------------------------------------------------- nearest points
def _nearest(q, p, w=None):
    out = ops.nearest_points(_cuda(q), _cuda(p), None if w is None else _cuda(w))
    return [t.cpu().numpy() for t in out]


@pytest.mark.parametrize('N', [1, 2, 33, 1024, 32767, 32768])
def test_nearest_points_bits(N):
    rng = np.random.default_rng(N)
    B = 3
    pts = (rng.uniform(-0.5, 0.5, (B, N, 3)) + [[[0.0, 0, 0]], [[3.0, 3.0, 3.0]], [[0, 0, 0]]]).astype(np.float32)
    pts[0, N // 2:] = pts[0, :N - N // 2]                                   # clusters of duplicate points
    pts[2, :, 2] = 0.0                                                      # coplanar
    w = np.ones((B, N), np.float32)
    w[1, ::3] = 0.0
    w[1, 1::7] = np.nan
    q = np.concatenate([near_queries(pts, 200, N + 1, lo=-7, hi=-1), rng.uniform(-100, 100, (B, 56, 3))], 1)
    q = q.astype(np.float32)
    idx, d2 = _nearest(q, pts, w)
    for b in range(B):
        wi, wd = bo.nearest_points(q[b], pts[b], w[b])
        assert np.array_equal(idx[b], wi), b
        assert np.array_equal(_bits(d2[b]), _bits(wd)), b
    # every point of a body dropped
    w[0] = 0.0
    idx, d2 = _nearest(q, pts, w)
    assert (idx[0] == -1).all() and (d2[0] == 0).all()


# ------------------------------------------------------------------------------------------------- backward
def test_backward_on_one_face_with_32768_points():
    """32768 points whose closest face is one face: the backward's longest run of equal keys, and point ids at the
    u16 maximum.  The points lie 0.5 to 1 m off a 2 m face near the origin (the kernel forms q - p in world
    coordinates, so the error of one term is about u |x| / |q - p| of it).  Each of the face's vertices sums 32768
    terms of random sign in float32, in index order: that rounding is about sqrt(N) u of the entry, above the 5e-7 of
    the body scenes, while one point missing from the run would move an entry by about 1 / sqrt(N)."""
    rng = np.random.default_rng(51)
    B, N, P = 2, 32768, 64
    v, faces = soup(B, P, 52, off=5.0, size=0.05)
    v = v.reshape(B, P, 3, 3)
    target = np.array([40, 3])
    big = np.float32([[[-1.0, -0.6, 0.1], [1.0, -0.5, -0.1], [0.0, 1.0, 0.0]], [[0.9, 0.8, 0.2], [-0.8, 0.9, 0.0],
                                                                               [0.1, -1.0, -0.2]]])
    v[np.arange(B), target] = big
    v = v.reshape(B, 3 * P, 3)
    p = []
    for b in range(B):
        t = big[b].astype(np.float64)
        n = np.cross(t[1] - t[0], t[2] - t[0])
        side = rng.choice([-1.0, 1.0], (N, 1))
        p.append(rng.dirichlet([8, 8, 8], N) @ t + side * rng.uniform(0.5, 1.0, (N, 1)) * n / np.linalg.norm(n))
    p = np.stack(p).astype(np.float32)
    face, bary, _ = _closest(v, faces, p)
    assert (face == target[:, None]).all()
    g = rng.normal(size=(B, N)).astype(np.float32)
    grad = ops.closest_points_backward(_cuda(v), _cuda(faces, torch.int32), _cuda(p), _cuda(face, torch.int32),
                                       _cuda(bary), _cuda(g)).cpu().numpy()
    for b in range(B):
        want = so.sq_dist_grad(v[b], faces, p[b], face[b], bary[b], g[b])
        err = np.abs(grad[b] - want).max() / np.abs(want).max()
        print(f'[bvh] backward over one face, 32768 points: error / max entry {err:.2e}')
        assert err <= 8 * np.sqrt(N) * 2.0 ** -24


# --------------------------------------------------------------------------------------------- self-collisions
def comb(teeth, seed):
    """Face 0 in z = 0 pierced by `teeth` thin upright faces, then five bystanders: vertices (3F, 3), faces.  Face 0's
    pairs are selected kSelfSel at a time, over ceil(teeth / 8) rounds."""
    rng = np.random.default_rng(seed)
    base = [[[-1, -1, 0], [1, -1, 0], [0, 1, 0]]]
    x = rng.uniform(-0.3, 0.3, teeth)
    tooth = np.stack([np.stack([x, np.full(teeth, -0.2), np.full(teeth, -0.5)], 1),
                      np.stack([x + 1e-3, np.full(teeth, -0.2), np.full(teeth, 0.5)], 1),
                      np.stack([x, np.full(teeth, 0.2), np.full(teeth, 0.5)], 1)], 1)
    far = rng.uniform(5, 6, (5, 3, 3))
    tris = np.concatenate([base, tooth, far]).astype(np.float32)          # the pierced face first: its pairs
    return tris.reshape(-1, 3), np.arange(3 * len(tris), dtype=np.int32).reshape(-1, 3)


def _pairs(v, faces, max_pairs, **kw):
    pairs, count = ops.self_collisions(_cuda(v), _cuda(faces, torch.int32), max_pairs, **kw)
    return pairs.cpu().numpy(), count.cpu().numpy()


@pytest.mark.parametrize('teeth', [1, 7, 8, 9, 17, 100])
def test_self_collisions_comb(teeth):
    (v0, faces), (v1, _) = comb(teeth, teeth), comb(teeth, teeth + 1000)
    v = np.stack([v0, v1])
    pairs, count = _pairs(v, faces, 4 * teeth + 8)
    for b in range(2):
        want = po.self_collisions(v[b], faces, max_hits=512)
        assert len(want) >= teeth
        assert count[b] == len(want)
        np.testing.assert_array_equal(pairs[b, :len(want)], want)
        assert (pairs[b, len(want):] == -1).all()
        # max_pairs cutting inside a kSelfSel round, and the part filter dropping every pair with the pierced face
        for m in (3, 9, max(1, len(want) - 1)):
            pm, cm = _pairs(v[b:b + 1], faces, m)
            assert cm[0] == len(want)
            np.testing.assert_array_equal(pm[0, :min(m, len(want))], want[:m])
        tri = v[b].reshape(-1, 3, 3)
        lab = np.where(np.abs(tri[:, :, 2]).max(1) == 0, 1, 2).astype(np.int64)
        lab[np.abs(tri[:, 0, 0]) > 4] = 0
        pf, cf = _pairs(v[b:b + 1], faces, 4 * teeth + 8, part_labels=lab, ignored_part_pairs=[(1, 2)])
        wf = po.self_collisions(v[b], faces, lab, [(1, 2)], max_hits=512)
        assert cf[0] == len(wf)
        np.testing.assert_array_equal(pf[0, :len(wf)], wf)


def test_self_collisions_at_32768_faces_and_after_a_scrambled_refit():
    v, faces = soup(2, 32768, 61, size=0.002, spread=np.array([0.6, 0.5])[:, None, None, None])
    pairs, count = _pairs(v, faces, 8192)
    for b in range(2):
        want = po.self_collisions(v[b], faces, max_hits=64)
        assert 50 < len(want) <= 8192
        assert count[b] == len(want)
        np.testing.assert_array_equal(pairs[b, :len(want)], want)
    rng = np.random.default_rng(62)
    perm = np.stack([rng.permutation(v.shape[1]) for _ in range(2)])
    tree = ops.ScanTree()
    ff = _cuda(faces, torch.int32)
    ops.self_collisions(_cuda(np.take_along_axis(v, perm[:, :, None], 1)), ff, 16, tree=tree)
    key = tree.key
    p2, c2 = ops.self_collisions(_cuda(v), ff, 8192, tree=tree)
    assert tree.key == key
    assert np.array_equal(p2.cpu().numpy(), pairs) and np.array_equal(c2.cpu().numpy(), count)


# ------------------------------------------------------------------------------------------ mesh_to_mesh_forward
def _sets(faces, bcs, Q, M):
    out = []
    for q in range(Q):
        f, b = faces[q * M:(q + 1) * M], bcs[q * M:(q + 1) * M]
        k = f >= 0
        o = np.argsort(f[k], kind='stable')
        out.append((f[k][o], b[k][o]))
    return out


@pytest.mark.parametrize('dtype', [np.float32, np.float64])
def test_mmi_query_covering_a_32768_face_scene(dtype):
    """One query triangle whose box covers the whole scene and that cuts through a few hundred of its 32768 targets:
    every node is visited, the narrow phase drains the leaf queue over many 32-leaf rounds, and the hits overflow M
    (the node stack of this balanced tree peaks near 280 entries; test_mmi_single_pop_regime drives it past
    kStackCap - 128).  M below the hit count keeps M hits of the oracle's set; M above it keeps all of them."""
    B, F = 2, 32768
    rng = np.random.default_rng(71)
    c = rng.uniform(-1, 1, (B, F, 1, 3)) * [1.0, 1.0, 0.5]
    t = (c + rng.normal(size=(B, F, 3, 3)) * 0.01).astype(dtype)
    q = np.array([[[-3, -3, -1], [3, -3, 1], [0, 3, 0.1]]], dtype)
    q = np.stack([q, q[:, [1, 2, 0]] * np.array([1, -1, 1], dtype)])
    ref = measure_oracle.mesh_to_mesh_forward if dtype == np.float32 else mmi_oracle_f64.mesh_to_mesh_forward
    big = 4096
    rf, rb = ref(q, t, big)
    nhit = [(rf[b] >= 0).sum() for b in range(B)]
    assert min(nhit) > 96 and max(nhit) < big
    tdt = torch.float32 if dtype == np.float32 else torch.float64
    for M in (64, max(nhit) + 8):
        f, bc = ops.mesh_to_mesh_forward(_cuda(q, tdt), _cuda(t, tdt), M)
        f, bc = f.cpu().numpy(), bc.cpu().numpy()
        for b in range(B):
            (f1, b1), = _sets(f[b], bc[b], 1, M)
            (f2, b2), = _sets(rf[b], rb[b], 1, big)
            if M >= nhit[b]:
                np.testing.assert_array_equal(f1, f2)
                assert np.abs(b1 - b2).max() <= (1e-6 if dtype == np.float32 else 1e-12)
            else:
                assert len(f1) == M and np.isin(f1, f2).all()


def _spine_query(tris, faces):
    """A triangle 20 times the size of the one through the centroids of `faces`, in its plane: it cuts those faces,
    and its box covers the scene."""
    g = tris[faces].mean(1)
    return (g.mean(0) + 20 * (g - g.mean(0)))[None]


@pytest.mark.parametrize('dtype', [np.float32, np.float64])
def test_mmi_single_pop_regime(dtype):
    """bvh_query_kernel pops one node at a time once its stack holds more than kStackCap - 128 entries, which keeps
    the 1024-entry shared-memory stack from overflowing.  On bvh_f32_oracle.deep_spine_scene the restated build and
    warp traversal show the stack passing that mark (asserted here); the kernel's hits must still equal the oracle's,
    with M both below and above the hit count."""
    scenes = [bo.deep_spine_scene(1e-3, 72)[0], bo.deep_spine_scene(2e-3, 73)[0]]
    t = np.stack(scenes).astype(dtype)
    q = np.stack([_spine_query(t[0], [5, 2000, 4000]), _spine_query(t[1], [100, 2500, 4000])]).astype(dtype)
    for b in range(2):
        assert (q[b].min((0, 1)) < t[b].min((0, 1))).all() and (q[b].max((0, 1)) > t[b].max((0, 1))).all()
        peak_sp, peak_qn, single = bo.warp_traversal(*bo.karras_topology(bo.morton_codes(t[b])))
        assert single > 0 and peak_sp < bo.KSTACK_CAP and peak_qn <= bo.KQUEUE_CAP, (peak_sp, peak_qn, single)
    ref = measure_oracle.mesh_to_mesh_forward if dtype == np.float32 else mmi_oracle_f64.mesh_to_mesh_forward
    big = 4096
    rf, rb = ref(q, t, big)
    nhit = [(rf[b] >= 0).sum() for b in range(2)]
    assert min(nhit) >= 3
    tdt = torch.float32 if dtype == np.float32 else torch.float64
    for M in (2, max(nhit) + 8):
        f, bc = ops.mesh_to_mesh_forward(_cuda(q, tdt), _cuda(t, tdt), M)
        f, bc = f.cpu().numpy(), bc.cpu().numpy()
        for b in range(2):
            (f1, b1), = _sets(f[b], bc[b], 1, M)
            (f2, b2), = _sets(rf[b], rb[b], 1, big)
            if M >= nhit[b]:
                np.testing.assert_array_equal(f1, f2)
                assert np.abs(b1 - b2).max() <= (1e-6 if dtype == np.float32 else 1e-12)
            else:
                assert len(f1) == M and np.isin(f1, f2).all()
