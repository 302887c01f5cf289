"""The float64 mesh_to_mesh_forward on the CPU: the double build of the scalar-generic C oracle
(oracle/mmi_oracle_scalar.c via oracle/mmi_oracle_f64.py) against the reference operator's own float64 results
(tests/golden/ref_mmi_{plane,soup,quirk}_f64.npz, written by `python tools/make_golden.py mmi`), and the dtype
refusals of ops.mesh_to_mesh_forward, which come before any launch.

The input builders here are shared with tests/test_gpu_mmi_f64.py and tools/make_golden.py.

The reference's double instantiation rounds to float in two places (see oracle/mmi_oracle_scalar.c): the SAT
tolerance CMP and the projected intervals of the separating-axis test.  `quirk_inputs_f64` builds pairs where exactly
that rounding decides the answer, so an exact double SAT disagrees with the reference on them."""
import os

import numpy as np
import pytest
import torch

from oracle import measure_oracle, mmi_oracle_f64
from shapy_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLT_EPS = float(np.finfo(np.float32).eps)


def plane_inputs_f64(golden_dir):
    """(query, target, max_collisions): the chest-plane quads of the 4 real bodies against their 20 908 triangles, in
    float64, with seeded noise of 1e-7 on every vertex so that no body coordinate is a float32 value."""
    g = np.load(os.path.join(golden_dir, 'img00_body.npz'))
    lm = synth.load_landmarks()
    bodies = np.concatenate([g['v_shaped'][None], g['extra_v_shaped']], 0).astype(np.float64)
    bodies = bodies + np.random.default_rng(64).normal(0, 1e-7, bodies.shape)
    tris = np.ascontiguousarray(bodies[:, g['faces']])                          # (4, F, 3, 3)
    queries = []
    for b in range(bodies.shape[0]):
        h = float((tris[b, lm['chest']['face_idx']] * np.float64(lm['chest']['bc'])[:, None]).sum(0)[1])
        quad = np.float64([[-1, h, -1], [1, h, -1], [1, h, 1], [-1, h, 1]])    # body_measurements.py:90-97
        queries.append(np.stack([quad[[0, 1, 2]], quad[[0, 2, 3]]]))
    return np.stack(queries), tris, 256


def soup_inputs_f64():
    """(query, target, max_collisions): two seeded float64 triangle soups."""
    rng = np.random.default_rng(12)
    B, Q, F = 2, 96, 400

    def soup(n, spread, size):
        c = rng.uniform(-spread, spread, (B, n, 1, 3))
        return c + rng.normal(0, size, (B, n, 3, 3))
    query = soup(Q, 1.0, 0.15)
    return query, soup(F, 1.0, 0.15), 64


def _plane_frame(rng):
    """A tilted unit normal (every component at least 0.3) and two in-plane unit directions."""
    while True:
        n = rng.normal(size=3)
        n /= np.linalg.norm(n)
        if np.abs(n).min() > 0.3:
            break
    u = np.cross(n, [1.0, 0.0, 0.0])
    u /= np.linalg.norm(u)
    return n, u, np.cross(n, u)


def _tri(c, u, w, shape, k):
    return np.stack([c + k * (a * u + b * w) for a, b in shape])


def _normal_axis(t):
    """The SAT's first axis of triangle t (SatCrossEdge(v0, v1, v1, v2) = cross(v1 - v0, v2 - v1)) and its length²."""
    ax = np.cross(t[1] - t[0], t[2] - t[1])
    return ax, float(ax @ ax)


# non-degenerate shapes without right angles, so no edge pair makes the SAT fall back to an in-plane axis
SHAPES = [((0.0, 0.0), (1.0, 0.1), (0.3, 0.9)), ((0.0, 0.0), (0.9, -0.3), (0.6, 0.8)),
          ((-0.4, 0.1), (0.8, 0.0), (0.1, 1.0))]


def quirk_inputs_f64():
    """(query, target, max_collisions, pairs): B = 1, query i against target i, pairs far apart from one another.

    pairs is a list of (query index, target index, kind) with kind
      'interval'          a triangle and its copy shifted 1e-9 along the normal of its tilted plane.  Exact in double,
                          the normal axis separates them; rounded to float, as the reference's fminf / fmaxf do, every
                          projected interval is the same float, so nothing separates and the pair collides.  The plane
                          is moved along its normal so the projections sit 0.3 of a float ulp above a float value.
      'interval_control'  the same with a 1e-3 shift: separated either way.
      'cmp'               a triangle 1e-5 from its parallel copy, scaled so that the squared length of every normal
                          axis is FLT_EPSILON·(1 + 3e-8): above the CMP threshold in double, equal to it once rounded
                          to float, where CMP calls the axis degenerate and it cannot separate.  The pair collides.
      'cmp_control'       the same with the squared axis length FLT_EPSILON·(1 + 1e-3): separated either way.
    """
    rng = np.random.default_rng(2024)
    queries, targets, pairs = [], [], []

    def add(q, t, kind):
        pairs.append((len(queries), len(targets), kind))
        queries.append(q)
        targets.append(t)

    for i in range(6):
        n, u, w = _plane_frame(rng)
        c = 3.0 * n                         # 3 from the origin: the 1e-9 shift is < 1 % of a float ulp of n·v
        shape = SHAPES[i % 3]
        for _ in range(3):                  # place n·v at 0.3 ulp above a float (n is fixed by the shape and size)
            t = _tri(c, u, w, shape, 0.1)
            ax, _ = _normal_axis(t)
            d = float(ax @ t[0])
            lo = float(np.float32(d))
            if lo > d:
                lo = float(np.nextafter(np.float32(d), np.float32(-np.inf)))
            ulp = float(np.nextafter(np.float32(lo), np.float32(np.inf))) - lo
            c = c + n * ((lo + 0.3 * ulp - d) / np.linalg.norm(ax))
        t = _tri(c, u, w, shape, 0.1)
        add(t, t + 1e-9 * n, 'interval')
        add(t + 0.4 * u, t + 0.4 * u + 1e-3 * n, 'interval_control')
    slot = 0
    for i in range(4):
        n, u, w = _plane_frame(rng)
        shape = SHAPES[i % 3]
        for kind, rel in (('cmp', 3e-8), ('cmp_control', 1e-3)):
            c = np.array([6.0 + 1.5 * slot, -0.5, 0.2 + 0.1 * i])
            slot += 1
            _, l2 = _normal_axis(_tri(c, u, w, shape, 1.0))
            k = (FLT_EPS * (1 + rel) / l2) ** 0.25
            t = _tri(c, u, w, shape, k)
            add(t, t + 1e-5 * n, kind)
    return np.stack(queries)[None], np.stack(targets)[None], 8, pairs


def load_reference(name, query):
    """The stored float64 reference result for `query`: faces (B, Q * M) with -1 in empty slots, bcs (B, Q * M, 2, 3)."""
    d = np.load(os.path.join(ROOT, 'tests', 'golden', f'{name}.npz'))
    assert d['bcs'].dtype == np.float64 and d['query'].dtype == np.float64
    assert np.array_equal(d['query'], query), 'the inputs differ from those the reference was run on'
    shape = tuple(int(x) for x in d['shape'])
    faces = np.full(shape, -1, np.int64)
    bcs = np.zeros(shape + (2, 3), np.float64)
    idx = tuple(d['idx'].T)
    faces[idx] = d['faces']
    bcs[idx] = d['bcs']
    return faces, bcs


def as_dict(faces, bcs, M):
    """{(query, face): bcs (2,3)} of one body."""
    return {(int(s) // M, int(faces[s])): bcs[s] for s in np.nonzero(faces >= 0)[0]}


def compare(r, m, max_set_diff, what):
    """Collision sets equal up to max_set_diff borderline pairs (FMA contraction in the reference build); barycentrics
    of the common pairs equal to 1e-9 for all but 1 %.  Returns (common pairs, largest barycentric difference)."""
    diff = set(r) ^ set(m)
    assert len(diff) <= max_set_diff, (what, len(diff), sorted(diff)[:8])
    common = sorted(set(r) & set(m))
    errs = np.array([np.abs(r[k] - m[k]).max() for k in common]) if common else np.zeros(0)
    bad = int((errs > 1e-9).sum())
    assert bad <= len(common) // 100, (what, bad, len(common))
    return len(common), float(errs.max()) if len(errs) else 0.0


def check_quirk(faces, M, pairs, what):
    """Every quirk pair collides, no control pair does, and nothing else collides."""
    got = set(as_dict(faces, np.zeros(faces.shape + (2, 3)), M))
    want = {(q, t) for q, t, kind in pairs if not kind.endswith('control')}
    assert got == want, (what, sorted(got ^ want))


def test_quirk_inputs_are_what_they_claim():
    query, target, M, pairs = quirk_inputs_f64()
    assert len(pairs) == 20
    for q, t, kind in pairs:
        a, b = query[0, q], target[0, t]
        assert (a.min(0) <= b.max(0)).all() and (b.min(0) <= a.max(0)).all()              # AABBs overlap
        if kind.startswith('cmp'):
            for tri in (a, b):
                l2 = _normal_axis(tri)[1]
                assert l2 > FLT_EPS and (np.float32(l2) == np.float32(FLT_EPS)) == (kind == 'cmp')
        else:
            ax = _normal_axis(a)[0]
            pa, pb = a @ ax, b @ ax
            assert pa.max() < pb.min()                                                      # separated in double
            assert (len(set(np.float32(np.concatenate([pa, pb])))) == 1) == (kind == 'interval')


def test_plane_inputs_have_no_float32_coordinates(golden_dir):
    _, tris, _ = plane_inputs_f64(golden_dir)
    assert not (tris.astype(np.float32).astype(np.float64) == tris).any()


def _random_inputs(seed, Q, F, dtype):
    rng = np.random.RandomState(seed)
    B = 3

    def soup(n, size):
        return (rng.uniform(-1, 1, (B, n, 1, 3)) + rng.normal(0, size, (B, n, 3, 3))).astype(dtype)
    return soup(Q, 0.15), soup(F, 0.1)


def test_scalar_source_in_float_is_the_pinned_float_oracle(golden_dir):
    """The float build of oracle/mmi_oracle_scalar.c gives byte-identical outputs to oracle/mmi_oracle.c, which the
    reference's golden measurements pin; the double build differs from it only by its scalar type."""
    from test_gpu_zz_reference_op import plane_inputs, soup_inputs
    cases = [plane_inputs(golden_dir), soup_inputs()]
    cases += [_random_inputs(Q * 1000 + F, Q, F, np.float32) + (M,) for Q, F, M in ((64, 500, 32), (300, 3000, 8))]
    for query, target, M in cases:
        f1, b1 = measure_oracle.mesh_to_mesh_forward(query, target, M)
        f2, b2 = mmi_oracle_f64.mesh_to_mesh_forward(query, target, M, dtype=np.float32)
        assert (f1 >= 0).sum() > 50
        assert np.array_equal(f1, f2) and b1.dtype == b2.dtype and b1.tobytes() == b2.tobytes()


def test_double_oracle_vs_reference_plane(golden_dir):
    query, tris, M = plane_inputs_f64(golden_dir)
    ref_f, ref_b = load_reference('ref_mmi_plane_f64', query)
    f, b = mmi_oracle_f64.mesh_to_mesh_forward(query, tris, M)
    worst = 0.0
    for i in range(query.shape[0]):
        n, e = compare(as_dict(ref_f[i], ref_b[i], M), as_dict(f[i], b[i], M), 2, f'body {i}')
        assert n > 50
        worst = max(worst, e)
    print(f'plane: largest barycentric difference to the reference {worst:.2e}')


def test_double_oracle_vs_reference_soup():
    query, target, M = soup_inputs_f64()
    ref_f, ref_b = load_reference('ref_mmi_soup_f64', query)
    f, b = mmi_oracle_f64.mesh_to_mesh_forward(query, target, M)
    total, worst = 0, 0.0
    for i in range(query.shape[0]):
        r = as_dict(ref_f[i], ref_b[i], M)
        n, e = compare(r, as_dict(f[i], b[i], M), max(2, len(r) // 100), f'soup {i}')
        total, worst = total + n, max(worst, e)
    assert total > 100
    print(f'soup: largest barycentric difference to the reference {worst:.2e}')


def test_double_oracle_vs_reference_quirk():
    query, target, M, pairs = quirk_inputs_f64()
    ref_f, ref_b = load_reference('ref_mmi_quirk_f64', query)
    check_quirk(ref_f[0], M, pairs, 'reference')
    f, b = mmi_oracle_f64.mesh_to_mesh_forward(query, target, M)
    check_quirk(f[0], M, pairs, 'oracle')
    compare(as_dict(ref_f[0], ref_b[0], M), as_dict(f[0], b[0], M), 0, 'quirk')


class FakeCuda(torch.Tensor):
    """A CPU tensor that claims to live on the GPU, so the host checks in front of the launch can be reached without one"""
    @property
    def is_cuda(self):
        return True


@pytest.mark.parametrize('dq,dt', [(torch.float32, torch.float64), (torch.float64, torch.float32),
                                   (torch.float16, torch.float16), (torch.bfloat16, torch.bfloat16),
                                   (torch.float64, torch.float16)])
def test_dtype_refusals_before_any_launch(dq, dt):
    from shapy_b200 import ops
    q = torch.zeros(1, 2, 3, 3, dtype=dq).as_subclass(FakeCuda)
    t = torch.zeros(1, 4, 3, 3, dtype=dt).as_subclass(FakeCuda)
    with pytest.raises(RuntimeError) as e:
        ops.mesh_to_mesh_forward(q, t, 8)
    assert str(dq) in str(e.value) and str(dt) in str(e.value)
