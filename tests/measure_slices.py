"""Constructed meshes whose slices reach the edge cases of the measurement kernels (csrc/measure.cu).

Not a test module: tests/test_measure_slices_cpu.py proves on the float C oracle that each construction reaches the
case it is named for, and tests/test_gpu_measure_hull.py runs them through every measurement entry.

Every mesh has three slicing planes, chest / waist / hips at y = 0, 2 and 4, far enough apart that no face of one
plane's slice reaches another plane.  Faces 0..5 are markers outside the query quad's ±1 in x, so the kernels'
xz filter drops them: face 0 (the kernels skip face 0, as body_measurements.py:161 does), the three plane markers
(landmark bc (1, 0, 0) puts the plane exactly at their first vertex's y) and the head-top / left-heel pair of the
height.  What a slice holds is built from two pieces:
  - `prism`: a closed polygonal prism around the plane;
  - `needle`: one thin vertical triangle in a plane z = const crossing the slicing plane.  Away from the quad's
    diagonal it passes the SAT against one query triangle only, so it adds exactly one point, at its vertical edge.
"""
import functools
import math

import numpy as np

from oracle import measure_oracle

PLANES = ('chest', 'waist', 'hips')
HEIGHTS = (0.0, 2.0, 4.0)
CAP_POINTS = 1024          # points per plane, every entry
CAP_CAND = 8192            # (face, plane, query triangle) candidates per body, every entry
CHAIN_CAP = 640            # u16 candidate list per hull chain of measure_smem_kernel
GLOBAL_VERTS_V = 20000     # vertex count beyond what the kernel stages in shared memory: gathered from global memory


class Builder:
    def __init__(self):
        self.v, self.f = [], []
        self.lm = {}
        self.tri((5.0, 9.0, 0.0), (5.1, 9.0, 0.0), (5.0, 9.1, 0.1))             # face 0
        for p, h in zip(PLANES, HEIGHTS):
            self.lm[p] = dict(face_idx=self.tri((5.0, h, 0.0), (5.1, h, 0.0), (5.0, h, 0.1)), bc=[1.0, 0.0, 0.0])
        self.lm['head_top'] = dict(face_idx=self.tri((5.0, 6.1, 0.0), (5.1, 6.3, 0.0), (5.0, 6.7, 0.1)),
                                   bc=[0.2, 0.3, 0.5])
        self.lm['left_heel'] = dict(face_idx=self.tri((5.0, -1.3, 0.0), (5.2, -1.1, 0.0), (5.0, -1.2, 0.1)),
                                    bc=[0.6, 0.25, 0.15])

    def vert(self, p):
        self.v.append(p)
        return len(self.v) - 1

    def tri(self, a, b, c):
        self.f.append((self.vert(a), self.vert(b), self.vert(c)))
        return len(self.f) - 1

    def needle(self, x, z, h, s=0.6, eps=1e-3):
        """Vertical triangle in the plane z = const whose vertical edge at (x, z) crosses y = h at fraction s."""
        y0 = h - s
        return self.tri((x, y0, z), (x, y0 + 1.0, z), (x + eps, y0 + 0.5, z))

    def prism(self, poly, h, lo=0.5, hi=0.5, rings=None):
        """Closed prism over the xz polygon `poly` (counter-clockwise), from h - lo to h + hi; `rings` adds
        intermediate vertex rings at those heights."""
        ys = [h - lo] + list(rings or []) + [h + hi]
        n = len(poly)
        ids = [[self.vert((float(x), float(y), float(z))) for x, z in poly] for y in ys]
        for r in range(len(ys) - 1):
            a, b = ids[r], ids[r + 1]
            for i in range(n):
                j = (i + 1) % n
                self.f.append((a[i], b[j], a[j]))
                self.f.append((a[i], b[i], b[j]))
        for i in range(1, n - 1):
            self.f.append((ids[0][0], ids[0][i], ids[0][i + 1]))
            self.f.append((ids[-1][0], ids[-1][i + 1], ids[-1][i]))

    def mesh(self, **meta):
        return Mesh(np.asarray(self.v, np.float32), np.asarray(self.f, np.int32), dict(self.lm), meta)


class Mesh:
    def __init__(self, verts, faces, lm, meta):
        self.verts, self.faces, self.lm, self.meta = verts, faces, lm, meta

    @property
    def tris(self):
        return np.ascontiguousarray(self.verts[self.faces])

    def heights(self):
        """The three plane heights as the kernels compute them (fp32, v0*bc0 + v1*bc1 + v2*bc2, no FMA)."""
        t = self.tris
        out = []
        for p in PLANES:
            bc = np.asarray(self.lm[p]['bc'], np.float32)
            y = t[self.lm[p]['face_idx'], :, 1]
            out.append(np.float32(np.float32(y[0] * bc[0] + y[1] * bc[1]) + y[2] * bc[2]))
        return out

    def padded(self, nverts=GLOBAL_VERTS_V):
        """Same mesh with unused vertices appended up to `nverts` (the vertices entry then gathers them from global
        memory instead of staging them in shared memory)."""
        extra = np.full((nverts - len(self.verts), 3), 9.0, np.float32)
        return Mesh(np.concatenate([self.verts, extra]), self.faces, self.lm, dict(self.meta, padded=nverts))

    def permuted(self, seed):
        """Faces 1.. shuffled (face 0 stays: the kernels skip it), landmarks remapped."""
        rng = np.random.default_rng(seed)
        perm = np.concatenate([[0], 1 + rng.permutation(len(self.faces) - 1)])
        inv = np.empty_like(perm)
        inv[perm] = np.arange(len(perm))
        lm = {k: dict(face_idx=int(inv[v['face_idx']]), bc=v['bc']) for k, v in self.lm.items()}
        return Mesh(self.verts, np.ascontiguousarray(self.faces[perm]), lm, dict(self.meta, permuted=seed))

    def translated(self, d):
        return Mesh(self.verts + np.asarray(d, np.float32), self.faces, self.lm, dict(self.meta, translated=d))


# ------------------------------------------------------------------------------------------- oracle side
def oracle_points(mesh, p, max_collisions=4096):
    """The points the kernels must produce on plane p: the float C oracle's first intersection point of every
    (face > 0, query triangle) collision, evaluated as the kernels do ((v0 b0 + v1 b1) + v2 b2 in fp32)."""
    h = mesh.heights()[p]
    tris = mesh.tris
    faces, bcs = measure_oracle.mesh_to_mesh_forward(measure_oracle.plane_quad(h)[None], tris[None], max_collisions)
    faces, bcs = faces[0], bcs[0]
    for q in range(2):
        assert faces[q * max_collisions + max_collisions - 1] < 0, 'oracle collision buffer too small'
    keep = faces > 0
    t = tris[faces[keep]]
    b = bcs[keep][:, 0]
    assert np.array_equal(bcs[keep][:, 0], bcs[keep][:, 1])     # the second point is always a copy of the first
    return ((t[:, 0] * b[:, :1] + t[:, 1] * b[:, 1:2]) + t[:, 2] * b[:, 2:3]).astype(np.float32)


def candidate_count(mesh):
    """(face > 0, plane, query triangle) triples passing the kernels' AABB filter (inclusive, fp32)."""
    t = mesh.tris[1:]
    lo, hi = t.min(1), t.max(1)
    xz = (-1 <= hi[:, 0]) & (1 >= lo[:, 0]) & (-1 <= hi[:, 2]) & (1 >= lo[:, 2])
    return int(sum(2 * int(((h <= hi[:, 1]) & (h >= lo[:, 1]) & xz).sum()) for h in mesh.heights()))


def _key(x, z, k):
    dx, dz = (1, 1, 0, -1, -1, -1, 0, 1)[k], (0, 1, 1, 1, 0, -1, -1, -1)[k]
    return dx * float(x) + dz * float(z), -dz * float(x) + dx * float(z)


def extremes(pts):
    """Indices of the 8 extreme points of measure_smem_kernel (directions k * 45 deg, exact fp64 keys; exact ties
    to the first point in (y, z, x) bit order)."""
    from oracle import hull_exact
    ordb = hull_exact._ord_bits
    out = []
    for k in range(8):
        best = None
        for i in range(len(pts)):
            key = (_key(pts[i, 0], pts[i, 2], k), tuple(-int(ordb(pts[i, c])) for c in (1, 2, 0)))
            if best is None or key > best[0]:
                best = (key, i)
        out.append(best[1])
    return out


def chain_sizes(pts):
    """Points on the outer side of (or on) each chord E_k -> E_k+1 of measure_smem_kernel (exact)."""
    from fractions import Fraction as Fr
    e = extremes(pts)
    sizes = []
    for k in range(8):
        a, b = pts[e[k]], pts[e[(k + 1) % 8]]
        if a[0] == b[0] and a[2] == b[2]:
            sizes.append(0)
            continue
        ux, uz = Fr(float(b[0])) - Fr(float(a[0])), Fr(float(b[2])) - Fr(float(a[2]))
        n = sum(1 for p in pts if ux * (Fr(float(p[2])) - Fr(float(a[2]))) - uz * (Fr(float(p[0])) - Fr(float(a[0]))) <= 0)
        sizes.append(n)
    return sizes


# ------------------------------------------------------------------------------------------- families
def _poly(n, r, c=(0.0, 0.0), rot=0.1):
    return [(c[0] + r * math.cos(rot + 2 * math.pi * i / n), c[1] + r * math.sin(rot + 2 * math.pi * i / n))
            for i in range(n)]


def _off_diagonal(angles_deg):
    """Drops angles within 12 deg of the quad's diagonal (45 and 225 deg), where a needle hits both query triangles."""
    return [a for a in angles_deg if min(abs((a - 45) % 180), 180 - abs((a - 45) % 180)) > 12]


def ngon(n, center=(0.0, 0.0), r=0.5):
    b = Builder()
    for k, h in enumerate(HEIGHTS):
        b.prism(_poly(n, r, center, rot=0.1 + 0.37 * k), h)
    return b.mesh(family=f'ngon{n}' + ('_off' if center != (0.0, 0.0) else ''))


def clipped():
    """Prisms reaching past the query quad's ±1 in x and z: only the part inside the quad is sliced."""
    b = Builder()
    b.prism(_poly(40, 1.2), HEIGHTS[0])
    b.prism([(-0.5, -1.6), (1.6, -1.6), (1.6, 0.5), (-0.5, 0.5)], HEIGHTS[1])
    b.prism(_poly(24, 0.5, (0.8, -0.3)), HEIGHTS[2])
    return b.mesh(family='clipped')


def subdivided_square(m=16):
    """Square prism, each side subdivided into m segments: collinear points on every hull edge and exact ties in the
    45-degree keys (a whole side shares its x or z)."""
    b = Builder()
    for h, half in zip(HEIGHTS, (0.5, 0.25, 0.75)):
        s = [-half + 2 * half * i / m for i in range(m)]
        poly = ([(x, -half) for x in s] + [(half, z) for z in s] + [(-x, half) for x in s] + [(-half, -z) for z in s])
        b.prism(poly, h)
    return b.mesh(family='subdivided_square')


def arc_cluster(n_fill=980, n_arc=16):
    """One hull chain of measure_smem_kernel with more than 640 outer points (its candidate list overflows and it
    scans every point): n_arc hull vertices on an arc between the 0- and 45-degree extremes, n_fill needles just
    outside their chord but inside the hull, 4 anchors elsewhere (1 000 points on chest and hips).

    The arc is coarse enough that leaving out any one of its hull vertices shortens the perimeter by more than 2e-6
    (tests/test_measure_slices_cpu.py).  A scan that read only 640 of the 1 000 points would skip 360 of them; which
    ones depends on the slots that atomicAdd hands out, not on face order, but it would keep all 16 arc vertices with
    a chance of about 0.64^16 = 8e-4 per plane."""
    b = Builder()
    for k, h in enumerate(HEIGHTS):
        for x, z in ((-0.6, 0.5), (-0.7, -0.6), (0.2, -0.8), (-0.1, 0.8)):
            b.needle(x, z, h)
        arc = [(0.8 * math.cos(math.radians(a)), 0.8 * math.sin(math.radians(a))) for a in np.linspace(4, 40, n_arc)]
        (ax, az), (bx, bz) = arc[0], arc[-1]
        nx, nz = (bz - az), -(bx - ax)             # outward normal of the chord (the arc bulges to +x, +z)
        nn = math.hypot(nx, nz)
        nf = n_fill if k != 1 else 100
        for i in range(nf):
            t = 0.2 + 0.6 * i / max(nf - 1, 1)
            b.needle(ax + t * (bx - ax) + 0.004 * nx / nn, az + t * (bz - az) + 0.004 * nz / nn, h)
        for x, z in arc:
            b.needle(x, z, h)
    return b.mesh(family='arc_cluster')


def obtuse():
    """Three-point slices: a thin triangle whose obtuse vertex C is extreme in none of the 8 directions (chest), a
    plain triangle (waist), and the same thin triangle, mirrored (hips)."""
    b = Builder()
    A, B = np.array([-0.3, -0.5]), np.array([0.9, -0.1])
    d = (B - A) / np.linalg.norm(B - A)
    C = (A + B) / 2 + 0.015 * np.array([-d[1], d[0]])
    for x, z in (A, B, C):
        b.needle(float(x), float(z), HEIGHTS[0])
    for x, z in ((-0.5, 0.2), (0.4, -0.6), (0.6, 0.1)):
        b.needle(x, z, HEIGHTS[1])
    for x, z in (A, B, C):
        b.needle(float(-z), float(-x), HEIGHTS[2])
    return b.mesh(family='obtuse', obtuse=(A.tolist(), B.tolist(), C.tolist()))


def small_counts():
    """Exactly 3 points (chest), 2 points (waist), and a plane that misses the mesh (hips: 0 points)."""
    b = Builder()
    for x, z in ((-0.5, 0.3), (0.6, -0.4), (0.5, 0.2)):
        b.needle(x, z, HEIGHTS[0])
    for x, z in ((-0.5, 0.3), (0.6, -0.4)):
        b.needle(x, z, HEIGHTS[1])
    return b.mesh(family='small_counts')


def degenerate():
    """Points all collinear in xz (chest: needles on z = 0, so every z is exactly 0), all coincident (waist: three
    copies of one needle), and a plain ring (hips)."""
    b = Builder()
    for x in (0.1, 0.3, 0.5, 0.7, -0.4):
        b.needle(x, 0.0, HEIGHTS[0])
    for _ in range(3):
        b.needle(0.4, -0.3, HEIGHTS[1])
    b.prism(_poly(12, 0.4), HEIGHTS[2])
    return b.mesh(family='degenerate')


def through_vertices():
    """Planes through ring vertices: landmark bc (1, 0, 0) on a ring face.  Chest: the prism's bottom ring and cap lie
    in the plane; waist: the middle one of three vertex rings."""
    b = Builder()
    f0 = len(b.f)
    b.prism(_poly(16, 0.5), HEIGHTS[0] + 0.5)           # bottom ring at y = h, face f0 = (a0, b1, a1): a0 on it
    b.lm['chest'] = dict(face_idx=f0, bc=[1.0, 0.0, 0.0])
    f1 = len(b.f)
    b.prism(_poly(20, 0.45, rot=0.3), HEIGHTS[1] + 0.1, lo=0.5, hi=0.5, rings=[HEIGHTS[1]])
    b.lm['waist'] = dict(face_idx=f1 + 2 * 20, bc=[1.0, 0.0, 0.0])   # first face of the second band starts on the ring
    b.prism(_poly(9, 0.6), HEIGHTS[2])
    m = b.mesh(family='through_vertices')
    assert m.heights()[0] == HEIGHTS[0] and m.heights()[1] == HEIGHTS[1]
    return m


def face0_crossing():
    """Face 0 is a side face of the chest ring: the kernels, like body_measurements.py:161, drop its points."""
    b = Builder()
    b.prism(_poly(10, 0.5), HEIGHTS[0])
    k = len(b.f) - 2 * 10 - 2 * (10 - 2)         # first side face of that prism
    b.f[0], b.f[k] = b.f[k], b.f[0]
    for h in HEIGHTS[1:]:
        b.prism(_poly(10, 0.5), h)
    return b.mesh(family='face0_crossing')


@functools.lru_cache(maxsize=None)
def _tie_pair():
    """Two needle fractions s whose vertical edges at (0.5, 0) give points with exactly x = 0.5, z = 0 but different
    y (searched on the oracle: the y of a point is rounded differently per face)."""
    found = {}
    for s in np.linspace(0.55, 0.95, 81):
        b = Builder()
        b.needle(0.5, 0.0, HEIGHTS[0], s=float(s))
        p = oracle_points(b.mesh(), 0)
        if len(p) == 1 and p[0, 0] == np.float32(0.5) and p[0, 2] == 0:
            found.setdefault(float(p[0, 1]), float(s))
            if len(found) == 2:
                return tuple(found.values())
    raise AssertionError('no needle pair with identical (x, z) and different y')


def identical_xz():
    """A hull vertex shared by two points with identical (x, z) and different y (chest and hips), plus a ring."""
    b = Builder()
    s1, s2 = _tie_pair()
    for h in HEIGHTS:
        b.prism(_poly(14, 0.3), h)
    for h in (HEIGHTS[0], HEIGHTS[2]):
        b.needle(0.5, 0.0, h, s=s1)
        b.needle(0.5, 0.0, h, s=s2)
    return b.mesh(family='identical_xz')


def exact_count(n_chest, n_waist=CAP_POINTS, n_hips=300):
    """Needles on a circle of radius 0.8, away from the quad's diagonal: exactly one point each."""
    b = Builder()
    for n, h in zip((n_chest, n_waist, n_hips), HEIGHTS):
        ang = _off_diagonal(np.linspace(0, 360, 4 * n, endpoint=False))
        ang = [ang[int(i * len(ang) / n)] for i in range(n)]
        for a in ang:
            b.needle(0.8 * math.cos(math.radians(a)), 0.8 * math.sin(math.radians(a)), h)
    return b.mesh(family=f'count{n_chest}')


def overhang(n_faces, rings=True):
    """Faces whose AABB overlaps all three planes and the quad, but which cross the planes at x > 1: 6 candidates
    each and no point.  Plus a ring per plane."""
    b = Builder()
    if rings:
        for h in HEIGHTS:
            b.prism(_poly(30, 0.5), h)
    for i in range(n_faces):
        z = -0.9 + 1.8 * i / max(n_faces - 1, 1)
        # no edge perpendicular to a quad edge: the SAT's fallback axes would otherwise accept the pair (with no ray
        # hit, so a point at the origin)
        b.tri((0.9, 10.0, z), (1.5, -10.0, z + 0.13), (1.7, 10.0, z + 0.31))
    return b.mesh(family=f'overhang{n_faces}')


def value_families():
    """Every family whose slices are measured (values, point sets, entries against each other)."""
    return [ngon(3), ngon(4), ngon(7), ngon(64), ngon(333), ngon(500), ngon(150, center=(0.3, -0.2), r=0.45),
            clipped(), subdivided_square(), arc_cluster(), obtuse(), small_counts(), degenerate(), through_vertices(),
            face0_crossing(), identical_xz(), exact_count(CAP_POINTS), overhang(700)]
