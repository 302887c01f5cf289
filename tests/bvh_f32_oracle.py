"""Float32 NumPy restatement of the scan queries' arithmetic in shapy_b200/csrc/bvh.cu, operation for operation.

bvh.cu is compiled with -fmad=false and without fast math, so each float operation of the kernel rounds once, as a
NumPy float32 operation does: the restatement gives the kernel's bits.  Sums of three products keep the kernel's
order, (x + y) + z (dot3); fmaxf / fminf are np.fmax / np.fmin (a NaN operand loses).

    point_triangle(p, a, b, c)          (d2, v, w): the kernel's squared distance and barycentrics (1 - v - w, v, w)
    tri_box / box_d2                    a leaf's box and the squared distance of a point to a box
    scale(p, lo, hi)                    M, the largest coordinate magnitude of the query and the body's scene box
    prune_bound(best, M)                the largest box distance the query still descends into
    closest_points / nearest_points     brute force, the contract's answer: the lexicographic minimum of (float32 d2,
                                        index) over every primitive, with the weight rules of shapy_b200/ops.py

All arrays broadcast; every function takes and returns float32.
"""
import os
import re

import numpy as np

f32 = np.float32
ZERO, ONE = f32(0), f32(1)

_BVH_CU = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'shapy_b200', 'csrc', 'bvh.cu')


def _kernel_constant(name):
    """A `constexpr float name = <hex float>f;` of bvh.cu, so that the restated bound is the compiled one; None when
    bvh.cu has no such constant."""
    with open(_BVH_CU) as fh:
        m = re.search(r'constexpr float ' + name + r' = ([0-9a-fA-Fx.p+-]+)f;', fh.read())
    return None if m is None else f32(float.fromhex(m.group(1)))


PRUNE_SLACK = _kernel_constant('kPruneSlack')     # k u of the prune bound, k = 64, u = 2^-24


def _f(x):
    return np.asarray(x, f32)


def dot3(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _tri_d2(ab, ac, ap, v, w):
    d = ap - (ab * v[..., None] + ac * w[..., None])
    return dot3(d, d)


def _seg_t(ap, ab):
    l2 = dot3(ab, ab)
    pos = l2 > 0
    t = dot3(ap, ab) / np.where(pos, l2, ONE)
    return np.where(pos, np.fmin(np.fmax(t, ZERO), ONE), ZERO)


def _tri_region(ab, ac, ap, bp, cp):
    """(ok, v, w) of the Voronoi-region test; ok False where the kernel falls back to the edges."""
    d1, d2 = dot3(ab, ap), dot3(ac, ap)
    d3, d4 = dot3(ab, bp), dot3(ac, bp)
    d5, d6 = dot3(ab, cp), dot3(ac, cp)
    vc = d1 * d4 - d3 * d2
    vb = d5 * d2 - d1 * d6
    va = d3 * d6 - d5 * d4
    e1, e2 = d4 - d3, d5 - d6
    den = (va + vb) + vc

    def div(n, d):
        return n / np.where(d > 0, d, ONE)
    # the branches in the kernel's order, the first that holds wins
    conds = [
        (d1 <= 0) & (d2 <= 0),                                   # vertex a
        (d3 >= 0) & (d4 <= d3),                                  # vertex b
        (d6 >= 0) & (d5 <= d6),                                  # vertex c
        (vc <= 0) & (d1 >= 0) & (d3 <= 0),                       # edge ab
        (vb <= 0) & (d2 >= 0) & (d6 <= 0),                       # edge ac
        (va <= 0) & (e1 >= 0) & (e2 >= 0),                       # edge bc
    ]
    w_bc = np.where(e1 + e2 > 0, div(e1, e1 + e2), ZERO)
    vals = [
        (ZERO, ZERO), (ONE, ZERO), (ZERO, ONE),
        (np.where(d1 - d3 > 0, div(d1, d1 - d3), ZERO), ZERO),
        (ZERO, np.where(d2 - d6 > 0, div(d2, d2 - d6), ZERO)),
        (ONE - w_bc, w_bc),
    ]
    interior_ok = (den > 0) & (va >= 0) & (vb >= 0) & (vc >= 0)
    v = div(vb, den)
    w = div(vc, den)
    ok = interior_ok.copy()
    for c, (cv, cw) in zip(reversed(conds), reversed(vals)):
        v = np.where(c, cv, v)
        w = np.where(c, cw, w)
        ok = ok | c
    return ok, v.astype(f32), w.astype(f32)


def point_triangle(p, a, b, c):
    """The kernel's point_triangle: (d2, v, w), broadcasting over the leading axes of p (..., 3) and a, b, c."""
    p, a, b, c = _f(p), _f(a), _f(b), _f(c)
    with np.errstate(all='ignore'):
        ab, ac, ap = b - a, c - a, p - a
        bp, cp = p - b, p - c
        n = np.stack([ab[..., 1] * ac[..., 2] - ab[..., 2] * ac[..., 1],
                      ab[..., 2] * ac[..., 0] - ab[..., 0] * ac[..., 2],
                      ab[..., 0] * ac[..., 1] - ab[..., 1] * ac[..., 0]], -1)
        ok, v, w = _tri_region(ab, ac, ap, bp, cp)
        ok = ok & (dot3(n, n) > 0)
        d_in = _tri_d2(ab, ac, ap, v, w)
        # the fallback: the nearest of the edges ab, ac, bc, the first of them on a tie
        t0, t1, t2 = _seg_t(ap, ab), _seg_t(ap, ac), _seg_t(bp, c - b)
        zero = np.zeros_like(t0)
        best, bv, bw = _tri_d2(ab, ac, ap, t0, zero), t0, zero
        e1 = _tri_d2(ab, ac, ap, zero, t1)
        take = e1 < best
        best, bv, bw = np.where(take, e1, best), np.where(take, zero, bv), np.where(take, t1, bw)
        v2 = ONE - t2
        e2 = _tri_d2(ab, ac, ap, v2, t2)
        take = e2 < best
        best, bv, bw = np.where(take, e2, best), np.where(take, v2, bv), np.where(take, t2, bw)
        d2 = np.where(ok, d_in, best)
        return d2.astype(f32), np.where(ok, v, bv).astype(f32), np.where(ok, w, bw).astype(f32)


def tri_box(a, b, c):
    """A float triangle's exact box (lo, hi)."""
    a, b, c = _f(a), _f(b), _f(c)
    return np.minimum(np.minimum(a, b), c), np.maximum(np.maximum(a, b), c)


def box_d2(p, lo, hi):
    p, lo, hi = _f(p), _f(lo), _f(hi)
    with np.errstate(all='ignore'):
        d = np.fmax(np.fmax(lo - p, p - hi), ZERO)
        return dot3(d, d)


def scale(p, lo, hi):
    """M = max(|p|, |lo|, |hi|) over the coordinates, as the kernel takes it from the query and the root's box."""
    p, lo, hi = _f(p), _f(lo), _f(hi)
    m = np.fmax(np.fmax(np.abs(p), np.abs(lo)), np.abs(hi))
    return np.fmax(np.fmax(m[..., 0], m[..., 1]), m[..., 2])


def prune_bound(best, M):
    """(sqrt(best) + k u M)^2 in float32: a box farther than this holds no primitive as near as `best`.  (A bvh.cu
    without kPruneSlack prunes triangles by the relative bound.)"""
    if PRUNE_SLACK is None:
        return relative_prune_bound(best)
    with np.errstate(all='ignore'):
        r = np.sqrt(_f(best)) + _f(M) * PRUNE_SLACK
        return r * r


def relative_prune_bound(best):
    """The bound of the points query (and, before it covered its own rounding, of the triangle query too)."""
    best = _f(best)
    with np.errstate(all='ignore'):
        return best + best * f32(1e-5) + f32(1e-12)


def _lexmin(d2):
    """Row-wise first index of the smallest d2, NaN and inf never winning; -1 where nothing wins."""
    key = np.where(np.isfinite(d2), d2, np.inf)
    i = np.argmin(key, 1)
    r = np.arange(len(key))
    return np.where(np.isfinite(key[r, i]), i, -1)


def closest_points(vertices, faces, points, weights=None, chunk=16):
    """One body, as shapy_closest_points computes it: (face (N,) int32, bary (N, 3), d2 (N,)).  A point with weight
    <= 0 (or NaN) is not read, and a point no face gives a finite distance to gets face -1; both get zero barycentrics
    and distance."""
    tri = _f(vertices)[np.asarray(faces)]
    a, b, c = tri[None, :, 0], tri[None, :, 1], tri[None, :, 2]
    pts = _f(points)
    N = len(pts)
    face = np.full(N, -1, np.int32)
    bary, d2 = np.zeros((N, 3), f32), np.zeros(N, f32)
    keep = np.ones(N, bool) if weights is None else _f(weights) > 0
    rows_all = np.nonzero(keep)[0]
    for s in range(0, len(rows_all), chunk):
        rows = rows_all[s:s + chunk]
        e, v, w = point_triangle(pts[rows][:, None, :], a, b, c)
        f = _lexmin(e)
        hit = f >= 0
        r, fh = rows[hit], f[hit]
        k = np.arange(len(rows))[hit]
        vv, ww = v[k, fh], w[k, fh]
        face[r], d2[r] = fh, e[k, fh]
        bary[r] = np.stack([(ONE - vv) - ww, vv, ww], 1)
    return face, bary, d2


def nearest_points(queries, points, weights=None, chunk=64):
    """One body, as shapy_nearest_points computes it: (idx (Q,) int32, d2 (Q,)); a point with weight <= 0 (or NaN)
    is skipped, and a query without a point at a finite distance gets -1 and 0."""
    q, p = _f(queries), _f(points)
    keep = np.ones(len(p), bool) if weights is None else _f(weights) > 0
    idx, d2 = np.full(len(q), -1, np.int32), np.zeros(len(q), f32)
    for s in range(0, len(q), chunk):
        with np.errstate(all='ignore'):
            d = q[s:s + chunk, None, :] - p[None]
            e = dot3(d, d)
        e[:, ~keep] = np.nan
        i = _lexmin(e)
        hit = i >= 0
        idx[s:s + chunk] = i
        d2[s:s + chunk][hit] = e[np.arange(len(i))[hit], i[hit]]
    return idx, d2


# ------------------------------------------------------------------------------------- adversarial prune cases
OFFSETS = (0.0, 0.05, 1.0, 3.0, 10.0)          # metres from the origin
SHAPES = ('normal', 'thin', 'collinear', 'coincident')
REGIONS = ('vertex', 'edge', 'interior')


def adversarial_cases(rng, n):
    """n (p, a, b, c) float32 cases, (n, 3) each, built to stress point_triangle's rounding against box_d2: world
    scenes (triangles of 1 mm to 30 cm at OFFSETS from the origin) and flat pixel scenes (z = 0, coordinates up to
    1000, triangles of 1 to 300 px); normal, thin (height 1e-7 to 1e-2 of the edge), collinear and coincident-corner
    triangles; p off a vertex, an edge or the interior, at 1e-7 to 1e-1 of the triangle's size, along a random
    direction or the normal."""
    pix = rng.random(n) < 0.25
    off = np.where(pix[:, None], np.concatenate([rng.uniform(0, 1000, (n, 2)), np.zeros((n, 1))], 1),
                   np.asarray(OFFSETS)[rng.integers(len(OFFSETS), size=n)][:, None] * rng.choice([-1, 1], (n, 3)))
    size = np.where(pix, 10 ** rng.uniform(0, 2.5, n), 10 ** rng.uniform(-3, -0.5, n))
    flat = np.where(pix[:, None], np.array([1.0, 1.0, 0.0]), 1.0)

    def unit(x):
        x = x * flat
        return x / np.linalg.norm(x, axis=-1, keepdims=True)
    a = off + size[:, None] * rng.uniform(-1, 1, (n, 3)) * flat
    e1, e2 = unit(rng.normal(size=(n, 3))), unit(rng.normal(size=(n, 3)))
    b = a + size[:, None] * rng.uniform(0.2, 1, (n, 1)) * e1
    shape = rng.integers(len(SHAPES), size=n)
    c = a + size[:, None] * rng.uniform(0.2, 1, (n, 1)) * e2
    # thin: c near the line ab; collinear: c on it (rounded); coincident: c on a corner
    t = rng.uniform(-0.5, 1.5, (n, 1))
    on_line = a + t * (b - a)
    c = np.where((shape == 1)[:, None], on_line + size[:, None] * 10 ** rng.uniform(-7, -2, (n, 1)) * e2, c)
    c = np.where((shape == 2)[:, None], on_line, c)
    c = np.where((shape == 3)[:, None], np.where(rng.random((n, 1)) < 0.5, a, b), c)
    a, b, c = a.astype(f32), b.astype(f32), c.astype(f32)
    A, Bv, C = (x.astype(np.float64) for x in (a, b, c))
    region = rng.integers(len(REGIONS), size=n)
    bc = rng.dirichlet([1, 1, 1], n)
    k = rng.integers(3, size=n)
    edge = bc.copy()
    edge[np.arange(n), k] = 0
    edge /= edge.sum(1, keepdims=True)
    vert = np.eye(3)[k]
    w = np.where((region == 0)[:, None], vert, np.where((region == 1)[:, None], edge, bc))
    foot = w[:, :1] * A + w[:, 1:2] * Bv + w[:, 2:] * C
    nrm = np.cross(Bv - A, C - A)
    nn = np.linalg.norm(nrm, axis=1, keepdims=True)
    along_n = (rng.random(n) < 0.3) & (nn[:, 0] > 0) & ~pix
    dirn = np.where(along_n[:, None], nrm / np.where(nn > 0, nn, 1), unit(rng.normal(size=(n, 3))))
    dist = size * 10 ** rng.uniform(-7, -1, n)
    p = (foot + dist[:, None] * dirn).astype(f32)
    return p, a, b, c


def prune_margin(p, a, b, c):
    """(box_d2 of the leaf, point_triangle's d2, M, the k that the case needs: (sqrt(box) - sqrt(d2)) / (u M))."""
    d2, _, _ = point_triangle(p, a, b, c)
    lo, hi = tri_box(a, b, c)
    bx = box_d2(p, lo, hi)
    M = scale(p, lo, hi)
    need = (np.sqrt(bx.astype(np.float64)) - np.sqrt(d2.astype(np.float64))) / (2.0 ** -24 * np.maximum(M, 1e-30))
    return bx, d2, M, need


# ------------------------------------------------------------------------------------- the tree's shape
# bvh_prepare_kernel's Morton codes and sort, bvh_topology_kernel's Karras radix tree and bvh_query_kernel's warp
# stack, restated to show which branches of the warp traversal a scene reaches.
KSTACK_CAP, KQUEUE_CAP = 1024, 96        # bvh.cu's kStackCap and kQueueCap


def _expand_bits(v):
    v = (v * 0x00010001) & 0xFF0000FF
    v = (v * 0x00000101) & 0x0F00F00F
    v = (v * 0x00000011) & 0xC30C30C3
    v = (v * 0x00000005) & 0x49249249
    return v


def morton_codes(tris):
    """tris (F, 3, 3) float32 or float64 -> the 30-bit codes of bvh_prepare_kernel<T>: centroid and scene box in T,
    the normalised centroid rounded to float."""
    t = np.asarray(tris)
    T = t.dtype.type
    lo, hi = t.min((0, 1)), t.max((0, 1))
    with np.errstate(all='ignore'):
        cen = ((t[:, 0] + t[:, 1]) + t[:, 2]) / T(3)
        x = ((cen - lo) / (hi - lo)).astype(f32)
        x = np.fmin(np.fmax(x * f32(1024), f32(0)), f32(1023)).astype(np.int64)
    e = _expand_bits(x)
    return (e[:, 0] * 4 + e[:, 1] * 2 + e[:, 2]).astype(np.int64)


def _clz32(x):
    return 32 - int(x).bit_length()


def karras_topology(codes):
    """(left, right) child links of the F - 1 internal nodes over the (code, id)-sorted leaves, as bvh_topology_kernel
    builds them: >= 0 an internal node, < 0 the leaf ~j."""
    F = len(codes)
    ids = np.lexsort((np.arange(F), codes))
    c, d = [int(x) for x in codes[ids]], [int(x) for x in ids]

    def lcp(i, j):
        if j < 0 or j > F - 1:
            return -1
        return 32 + _clz32(d[i] ^ d[j]) if c[i] == c[j] else _clz32(c[i] ^ c[j])
    left, right = np.zeros(F - 1, np.int64), np.zeros(F - 1, np.int64)
    for i in range(F - 1):
        dr = 1 if lcp(i, i + 1) - lcp(i, i - 1) >= 0 else -1
        dmin = lcp(i, i - dr)
        lmax = 2
        while lcp(i, i + lmax * dr) > dmin:
            lmax *= 2
        ll, t = 0, lmax >> 1
        while t >= 1:
            if lcp(i, i + (ll + t) * dr) > dmin:
                ll += t
            t >>= 1
        j = i + ll * dr
        dnode = lcp(i, j)
        s, t = 0, ll
        while True:
            t = (t + 1) >> 1
            if lcp(i, i + (s + t) * dr) > dnode:
                s += t
            if t <= 1:
                break
        split = i + s * dr + min(dr, 0)
        left[i] = ~split if min(i, j) == split else split
        right[i] = ~(split + 1) if max(i, j) == split + 1 else split + 1
    return left, right


def warp_traversal(left, right):
    """bvh_query_kernel's stack and queue for a query whose box overlaps every node: (peak stack, peak queue, number
    of broad-phase steps that pop a single node because the stack holds more than kStackCap - 128)."""
    st, qn, peak_sp, peak_qn, single = [0], 0, 1, 0, 0
    while st or qn:
        if qn >= 32 or not st:
            qn -= min(qn, 32)
            continue
        take = 1 if len(st) > KSTACK_CAP - 128 else min(len(st), 32)
        single += take == 1 and len(st) > KSTACK_CAP - 128
        popped = st[len(st) - take:]
        del st[len(st) - take:]
        for links in (left, right):                 # the left children of all lanes, then the right ones
            for n in popped:
                if links[n] >= 0:
                    st.append(int(links[n]))
                else:
                    qn += 1
            peak_sp, peak_qn = max(peak_sp, len(st)), max(peak_qn, qn)
    return peak_sp, peak_qn, single


def deep_spine_scene(scale=1e-3, seed=72):
    """4096 small triangles whose tree drives bvh_query_kernel's stack past kStackCap - 128.  The scene spans a
    1024^3 Morton grid (scale metres per cell).  Each of the 32 cells of the top five code bits holds a right spine:
    25 groups of faces at codes (cell, 1^k 0...) for k < 25, whose group is the left child at depth k, then at code
    (cell, 1^25) six pairs of faces whose ids split at bits 11, 10, ..., 6 continue the spine by id.  A warp popping
    the 32 spine nodes of a level pushes 32 groups and 32 spine nodes, so the stack grows by 32 per level.  Returns
    triangles (F, 3, 3) float64 and their intended codes."""
    F, cells = 4096, 32
    id_spine = [0, 2048, 3072, 3584, 3840, 3968]          # 4096 - 2^(12 - k): ids split at bit 11 - k
    codes = np.full(F, -1, np.int64)
    for c in range(cells):
        for k, base in enumerate(id_spine):
            codes[base + 2 * c:base + 2 * c + 2] = (c << 25) | ((1 << 25) - 1)
    free = np.nonzero(codes < 0)[0]
    groups = [(c << 25) | (((1 << k) - 1) << (25 - k)) for c in range(cells) for k in range(25)]
    codes[free] = np.array(groups)[np.arange(len(free)) % len(groups)]
    # decode each code into its grid cell (x, y, z) and place a small triangle around the cell's centre
    xyz = np.zeros((F, 3), np.int64)
    for j in range(10):
        for a in range(3):
            xyz[:, a] |= ((codes >> (29 - 3 * j - a)) & 1) << (9 - j)
    rng = np.random.default_rng(seed)
    off = rng.uniform(-0.3, 0.3, (F, 3, 3))
    off -= off.mean(1, keepdims=True)
    tris = (xyz[:, None, :] + 0.5 + off) * scale
    # two faces stretch the scene box to the whole grid, so that each centre normalises into its own cell
    tris[0, 0] = 0.0
    tris[codes.argmax(), 0] = 1024 * scale
    return tris, codes
