// Virtual measurements (mass, height, chest / waist / hip circumference) in ONE launch, one CTA per body.
//
// Replaces, for the fixed query the reference issues (a 2-triangle horizontal quad per measurement):
//   BodyMeasurements.forward           mesh-mesh-intersection/body_measurements/body_measurements.py:217-246
//   3 x (LBVH build + traversal)       mesh-mesh-intersection/src/mesh_mesh_intersect_cuda_op.cu:969-1079
//   3 x scipy.spatial.ConvexHull (CPU) body_measurements.py:160-173
// A plane touches O(sqrt(F)) triangles, so one streaming pass over the faces (read v_shaped once,
// 125 KB / body) beats building a 3 MB BVH three times: every face is tested against the query quad of
// each plane with exactly the reference's predicates (inclusive AABB test, 11-axis SAT with its
// fallback axes, "first ray hit" point selection -- see mmi_device.cuh), hits are appended to a
// shared-memory point list, and the 2-D hull of each plane is gift-wrapped (exact fp64 orientation
// predicate on the fp32 points, as qhull sees them) with its 3-D edge lengths summed in fp32.
//
// One kernel, measure_smem_kernel<SRC>, 1 024 threads per body, for three sources of the triangles:
//   kStagedVerts  vertices + faces, the body's vertices staged ONCE in shared memory (125.7 KB of the SM's 227 KB):
//                 every face then gathers its 9 coordinates from shared memory instead of through L1 / L2 (gathers
//                 from global memory move 752 KB per body for 125.7 KB of data and are latency bound)
//   kGlobalVerts  vertices + faces whose vertices do not fit in shared memory (V > ~12 900): gathered from global
//   kTriangles    a (B, F, 3, 3) triangle array (BodyMeasurements.forward)
// The phases:
//   phase 0  (kStagedVerts only) coalesced copy of the body's vertices into shared memory (128-bit loads where the
//            row is aligned)
//   phase 1  one pass over the faces: signed volume + AABB filter against the three planes -> candidate queue
//   phase 2  exact SAT + "first ray hit" point, one candidate per thread
//   phase 3  per plane: the 8 extreme points in the directions k * 45 deg (exact: the keys x +- z are sums of two
//            floats in fp64) cut the hull into 8 chains; warp (plane, k) compacts the points on the outer side of the
//            chord E_k -> E_k+1 (exact fp64 orientation) and gift-wraps its chain from E_k to E_k+1.  The chain
//            lengths are summed in chain order, so the result does not depend on timing.
// Only phase 0 and the triangle accessor depend on the source, so every entry computes the same bits from the same
// triangles.  Every entry holds 1 024 points per plane and 8 192 candidates per body.  Capacity overflows are reported
// through `status` AND poison the affected outputs with NaN: a truncated point set must never pass for a measurement.
// Points that share (x, z) are told apart by value (pt_before), never by their slot, whose order depends on timing.
// A hull of zero area (fewer than 3 points, or all of them collinear or coincident in xz) is NaN: qhull raises on it.
// Compiled with -fmad=false (bit parity of the predicates with oracle/mmi_oracle.c).
//
// measure_smem_kernel<SRC, kGradient> is the backward of the five outputs (shapy_measure_backward*).  It reruns phases
// 0-3 from the same code, so it walks exactly the hull whose edge lengths the forward summed, with no state saved by
// the forward, and then writes the gradient (phase 4).  The reference's semantics (body_measurements.py:137-173,
// 182-215):
//   mass    985/6 sign(sum det) d det/d v per face: v1 x v2, v2 x v0, v0 x v1 for the rows v0, v1, v2
//   height  sign(y_head - y_heel) bc on the y components of the two landmark faces
//   chest / waist / hips  p = bc . T with bc held constant (the reference selects the points under no_grad); each hull
//           edge p_i -> p_j adds -u g to p_i and +u g to p_j, u the unit 3-D edge vector; points without a ray hit
//           have bc = 0 and get nothing.  There is no gradient through the plane height: the landmark only places the
//           query quad.
//   sign(0) = 0, as torch.abs gives.  A NaN circumference with a non-zero upstream gradient makes the body's whole
//   gradient NaN; with a zero upstream gradient it adds nothing.
// The gradient mode also keeps, per point slot, the (face, query half) code that produced it (phase 2) and, per hull
// vertex, the next vertex of the walk (phase 3b); points with equal bits are ordered by that code, so the hull and its
// gradient do not depend on timing either.  No float atomics touch the output: the dense mass term of a vertex (a
// face corner) is summed over its incident faces in a fixed order, then the hull and height terms are added in a
// fixed order, so a body's gradient is bit-identical from run to run and independent of the rest of the batch.
//
// measure_smem_kernel<SRC, kJacobian> (shapy_measure_jacobian_betas, vertex sources only) reruns the same phases 0-3,
// writes the forward's five outputs and then, in phase 4, jac (B,5,NB): row k is S^T times the gradient the backward
// gives for the cotangent e_k, S the model's shape rows -- the mass row densely over the vertices, the height row from
// the two landmark faces, each circumference row from its hull vertices only (see DESIGN.md section 4).
//
// kGradientExact / kJacobianExact (the _exact entries) are those two modes with the exact derivative of the
// circumferences.  Only the hull's combinatorics are held fixed: which points, in what order, from which face and which
// ray.  Phase 4 recovers each hull point's ray with mmi::isect_first_ray (the same ray tests in the same order as phase
// 2, nothing new stored), and hull_point_adjoint gives its corners' adjoints and the plane height's, the point moving
// with its triangle and with the plane.  Warp p sums the height adjoints of plane p in hull order (gh[p]), which reach
// the y components of the plane's landmark face with weights bc.  Everything else -- the measurements, the mass and
// height terms, the NaN rules, the summation orders -- is the mode's twin's.
#include "mmi_device.cuh"
#include "smplx.cuh"

namespace shapy {

constexpr int kThreads = 1024;
constexpr int kMaxPts = 1024;
constexpr int kMaxCand = 8192;     // (face, plane, query triangle) candidates that pass the AABB filter, per body; ints,
                                   // the buffer is reused for the per-chain candidate lists (u16) in phase 3
constexpr int kChainCap = 640;     // 24 chains x 640 x 2 B = 30 KB <= 32 KB
constexpr size_t kListBytes = 3 * kMaxPts * 12 + kMaxCand * 4;   // points + candidate queue, dynamic
// gradient and Jacobian modes only: per point slot its (face, query half) code (int) and the next hull vertex (u16)
constexpr size_t kGradBytes = 3 * kMaxPts * 4 + 3 * kMaxPts * 2;

enum TriSource { kStagedVerts, kGlobalVerts, kTriangles };
// kGradientExact / kJacobianExact: kGradient / kJacobian with the exact circumference derivative (see the top)
enum MeasureMode { kForward, kGradient, kJacobian, kGradientExact, kJacobianExact };
constexpr int kMaxJacBetas = 16;   // shape rows of the Jacobian mode

struct MeasureGrad {
  const float *gout;   // (B,5) upstream gradient
  const int *inc_ptr;  // (V+1) CSR: vertex -> incident (face, corner) entries 3 f + k, stably sorted (vertex sources)
  const int *inc;      // (3F)
  float *grad;         // (B,V,3) or (B,F,3,3)
  const float *S;      // Jacobian mode: the shape rows of the model's basis, [nb][ld]
  int ld, nb;
  float *jac;          // Jacobian mode: (B,5,nb)
};

struct MeasureArgs {
  const float *verts;  // (B,V,3) or null
  const int *faces;    // (F,3)
  const float *tris;   // (B,F,3,3) or null
  int B, V, F;
  shapy_measure_landmarks_t lm;
  float *out;          // (B,5)
  float *pts_out;      // (B,3,maxp,3) or null
  int *cnt_out;        // (B,3) or null
  int maxp;
  int *status;
  MeasureGrad g;       // gradient and Jacobian modes only
};

__device__ __forceinline__ bool better_next(double cx, double cz, float ax, float az, float bx, float bz) {
  // true when candidate b should replace a as the next hull vertex after c (counter-clockwise walk):
  // b is strictly to the right of c->a, or collinear and farther.
  double ux = (double)ax - cx, uz = (double)az - cz, wx = (double)bx - cx, wz = (double)bz - cz;
  double o = ux * wz - uz * wx;
  if (o < 0) return true;
  if (o > 0) return false;
  return (wx * wx + wz * wz) > (ux * ux + uz * uz);
}

// Total order on the float bit patterns (-0 before +0).
__device__ __forceinline__ int ord_bits(float f) {
  const int i = __float_as_int(f);
  return i >= 0 ? i : (i ^ 0x7fffffff);
}

// Order between two points (x, y, z) with the same (x, z) as floats: smaller y, then z, then x, as bits.  The hull
// takes the first of such points in this order, so its 3-D edge lengths do not depend on which point got which slot.
__device__ __forceinline__ bool pt_before(const float *a, const float *b) {
  const int ay = ord_bits(a[1]), by = ord_bits(b[1]);
  if (ay != by) return ay < by;
  const int az = ord_bits(a[2]), bz = ord_bits(b[2]);
  if (az != bz) return az < bz;
  return ord_bits(a[0]) < ord_bits(b[0]);
}

// pt_before, with full ties between two slots of plane p broken by their (face, query half) code when GRAD
template <bool GRAD>
__device__ __forceinline__ bool pt_order(const float *a, const float *b, const int *codes, int p, int i, int j) {
  if constexpr (GRAD) {
    if (pt_before(a, b)) return true;
    if (pt_before(b, a)) return false;
    return codes[p * kMaxPts + i] < codes[p * kMaxPts + j];
  } else {
    return pt_before(a, b);
  }
}

struct Extreme { float x, z; int idx; };

__device__ __forceinline__ void dir_key(float x, float z, int k, double &k1, double &k2) {
  // direction d_k = (dx, dz), k * 45 degrees (unnormalised, exact); tie-break direction = d_k rotated by +90 degrees
  const int dxs[8] = {1, 1, 0, -1, -1, -1, 0, 1}, dzs[8] = {0, 1, 1, 1, 0, -1, -1, -1};
  const double dx = dxs[k], dz = dzs[k];
  k1 = dx * (double)x + dz * (double)z;
  k2 = -dz * (double)x + dx * (double)z;
}

__device__ __forceinline__ float3 corner_cross(const mmi::Tri &T, int k) {
  // d det[v0; v1; v2] / d v_k
  const float3 a = k == 0 ? T.v1 : (k == 1 ? T.v2 : T.v0), c = k == 0 ? T.v2 : (k == 1 ? T.v0 : T.v1);
  return make_float3(a.y * c.z - a.z * c.y, a.z * c.x - a.x * c.z, a.x * c.y - a.y * c.x);
}

__device__ __forceinline__ float sign_of(float x) { return x > 0.f ? 1.f : (x < 0.f ? -1.f : (x == 0.f ? 0.f : x)); }

// Exact modes: the adjoint of one hull point of the plane at height h, produced on triangle T by ray `ray` of
// mmi::isect_first_ray against the query triangle Q, for the upstream vector g.  Writes the adjoint of T's corner k to
// dk and returns the plane height's.  The hull's combinatorics are held fixed (DESIGN.md section 4):
//   ray 3-5, edge point p = a + s (b - a), s = (h - a_y) / D, D = b_y - a_y (a, b the edge's corners; |D| >= 2.5e-5
//            by the ray test's |det| >= 1e-4):  d_a = (1 - s) g + e_y (g.(b - a)) (s - 1) / D,
//            d_b = s g - e_y (g.(b - a)) s / D, the third corner 0, d_h = g.(b - a) / D
//   ray 0-2, line point p = o + s w, o = (o_x, h, o_z) and w horizontal (the query edge), s = n.(v0 - o) / n.w,
//            n = (v1 - v0) x (v2 - v0), r = v0 - p, c = g.w / n.w:  d_v1 = c (v2 - v0) x r, d_v2 = c r x (v1 - v0),
//            d_v0 = c n - d_v1 - d_v2, d_h = g_y - c n_y
//   no ray   the point is a constant: all 0
__device__ __forceinline__ float hull_point_adjoint(const mmi::Tri &T, const mmi::Tri &Q, int ray, float h, float3 g,
                                                    int k, float3 &dk) {
  using mmi::cross3; using mmi::dot3; using mmi::sub3;
  auto corner = [](const mmi::Tri &X, int c) { return c == 0 ? X.v0 : (c == 1 ? X.v1 : X.v2); };
  dk = make_float3(0.f, 0.f, 0.f);
  if (ray >= 3) {
    const int i = ray - 3, j = i == 2 ? 0 : i + 1;
    const float3 a = corner(T, i), e = sub3(corner(T, j), a);
    const float D = e.y, s = (h - a.y) / D, q = dot3(g, e) / D;
    if (k == i) dk = make_float3((1.f - s) * g.x, (1.f - s) * g.y + q * (s - 1.f), (1.f - s) * g.z);
    if (k == j) dk = make_float3(s * g.x, s * g.y - q * s, s * g.z);
    return q;
  }
  if (ray < 0) return 0.f;
  const float3 o = corner(Q, ray), w = sub3(corner(Q, ray == 2 ? 0 : ray + 1), o);
  const float3 e1 = sub3(T.v1, T.v0), e2 = sub3(T.v2, T.v0), n = cross3(e1, e2);
  const float nw = dot3(n, w), s = dot3(n, sub3(T.v0, o)) / nw, c = dot3(g, w) / nw;
  const float3 r = make_float3(T.v0.x - (o.x + s * w.x), T.v0.y - (o.y + s * w.y), T.v0.z - (o.z + s * w.z));
  const float3 a = cross3(e2, r), b = cross3(r, e1);
  if (k == 0) dk = make_float3(c * (n.x - a.x - b.x), c * (n.y - a.y - b.y), c * (n.z - a.z - b.z));
  if (k == 1) dk = make_float3(c * a.x, c * a.y, c * a.z);
  if (k == 2) dk = make_float3(c * b.x, c * b.y, c * b.z);
  return g.y - c * n.y;
}

// MODE kForward: the forward; kGradient: the backward; kJacobian: the forward's outputs and their Jacobian with
// respect to betas; kGradientExact / kJacobianExact: the last two with the exact circumference derivative; see the top.
template <int SRC, int MODE = kForward>
__global__ void __launch_bounds__(kThreads, 1) measure_smem_kernel(MeasureArgs a) {
  constexpr bool GRAD = MODE != kForward;    // phases 0-3 keep the point codes and the hull walk
  constexpr bool BWD = MODE == kGradient || MODE == kGradientExact;      // writes a gradient
  constexpr bool EXACT = MODE == kGradientExact || MODE == kJacobianExact;
  extern __shared__ __align__(16) unsigned char smem[];
  const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int nvf = a.V * 3;
  float *vs = reinterpret_cast<float *>(smem);                                      // [V * 3] (+ pad to 16 B)
  const size_t vs_bytes = SRC == kStagedVerts ? ((size_t)nvf * 4 + 15) & ~(size_t)15 : 0;
  float *pts = reinterpret_cast<float *>(smem + vs_bytes);                          // [3][kMaxPts][3]
  int *cand = reinterpret_cast<int *>(smem + vs_bytes + 3 * kMaxPts * 12);          // [kMaxCand]
  unsigned short *clist = reinterpret_cast<unsigned short *>(cand);                // phase 3: [24][kChainCap]
  int *codes = reinterpret_cast<int *>(smem + vs_bytes + kListBytes);              // GRAD: [3][kMaxPts]
  unsigned short *nxt = reinterpret_cast<unsigned short *>(smem + vs_bytes + kListBytes + 3 * kMaxPts * 4);
  // query triangle q (0 or 1) of the horizontal quad [-1, 1]^2 at height h
  auto quad = [](float h, int q) {
    mmi::Tri Q;
    Q.v0 = make_float3(-1.f, h, -1.f);
    Q.v1 = q == 0 ? make_float3(1.f, h, -1.f) : make_float3(1.f, h, 1.f);
    Q.v2 = q == 0 ? make_float3(1.f, h, 1.f) : make_float3(-1.f, h, 1.f);
    return Q;
  };
  __shared__ int cnt[3];
  __shared__ int ncand;
  __shared__ float hs[3], lmy[2];
  __shared__ float red[kThreads / 32];
  __shared__ Extreme ext[3][8];
  __shared__ float chain_len[3][8];
  __shared__ int chain_edges[3][8];
  __shared__ int overflow;
  if (t < 3) cnt[t] = 0;
  if (t == 0) { ncand = 0; overflow = 0; }
  // ---- phase 0: vertices -> shared memory
  if constexpr (SRC == kStagedVerts) {
    const float *src = a.verts + (size_t)b * nvf;
    const int head = (int)((4 - (((size_t)b * nvf) & 3)) & 3);          // floats before the first 16-byte boundary
    const int nvec = nvf > head ? (nvf - head) / 4 : 0;
    for (int i = t; i < min(head, nvf); i += blockDim.x) vs[i] = src[i];
    const float4 *s4 = reinterpret_cast<const float4 *>(src + head);
    for (int i = t; i < nvec; i += blockDim.x) {
      const float4 q = __ldg(s4 + i);
      float *d = vs + head + 4 * i;
      d[0] = q.x; d[1] = q.y; d[2] = q.z; d[3] = q.w;
    }
    for (int i = head + 4 * nvec + t; i < nvf; i += blockDim.x) vs[i] = src[i];
    __syncthreads();
  }
  auto tri_of = [&](int f) {
    mmi::Tri T;
    if constexpr (SRC == kTriangles) {
      const float *p = a.tris + ((size_t)b * a.F + f) * 9;
      T.v0 = make_float3(__ldg(p), __ldg(p + 1), __ldg(p + 2));
      T.v1 = make_float3(__ldg(p + 3), __ldg(p + 4), __ldg(p + 5));
      T.v2 = make_float3(__ldg(p + 6), __ldg(p + 7), __ldg(p + 8));
    } else {
      const int *fi = a.faces + 3 * (size_t)f;
      const int i0 = __ldg(fi), i1 = __ldg(fi + 1), i2 = __ldg(fi + 2);
      if constexpr (SRC == kStagedVerts) {
        T.v0 = make_float3(vs[3 * i0], vs[3 * i0 + 1], vs[3 * i0 + 2]);
        T.v1 = make_float3(vs[3 * i1], vs[3 * i1 + 1], vs[3 * i1 + 2]);
        T.v2 = make_float3(vs[3 * i2], vs[3 * i2 + 1], vs[3 * i2 + 2]);
      } else {
        const float *vb = a.verts + (size_t)b * nvf;
        T.v0 = make_float3(__ldg(vb + 3 * i0), __ldg(vb + 3 * i0 + 1), __ldg(vb + 3 * i0 + 2));
        T.v1 = make_float3(__ldg(vb + 3 * i1), __ldg(vb + 3 * i1 + 1), __ldg(vb + 3 * i1 + 2));
        T.v2 = make_float3(__ldg(vb + 3 * i2), __ldg(vb + 3 * i2 + 1), __ldg(vb + 3 * i2 + 2));
      }
    }
    return T;
  };
  if (t < 5) {
    // (tri * bc.reshape(3,1)).sum(0): v0*bc0 + v1*bc1 + v2*bc2, y component
    mmi::Tri tr = tri_of(a.lm.face_idx[t]);
    float y = tr.v0.y * a.lm.bc[t][0] + tr.v1.y * a.lm.bc[t][1] + tr.v2.y * a.lm.bc[t][2];
    if (t < 2) lmy[t] = y; else hs[t - 2] = y;
  }
  __syncthreads();
  const float h0 = hs[0], h1 = hs[1], h2 = hs[2];
  // ---- phase 1: stream all faces once: signed volume + coarse (AABB) filter against the three planes.
  // Survivors go to a shared-memory queue so that the expensive exact predicates (phase 2) run with one
  // candidate per thread instead of one diverged lane per warp.
  float vol = 0.f;
  for (int f = t; f < a.F; f += blockDim.x) {
    mmi::Tri T = tri_of(f);
    // compute_mass, body_measurements.py:207-214
    vol += -T.v2.x * T.v1.y * T.v0.z + T.v1.x * T.v2.y * T.v0.z + T.v2.x * T.v0.y * T.v1.z -
           T.v0.x * T.v2.y * T.v1.z - T.v1.x * T.v0.y * T.v2.z + T.v0.x * T.v1.y * T.v2.z;
    const float ylo = fminf(T.v0.y, fminf(T.v1.y, T.v2.y)), yhi = fmaxf(T.v0.y, fmaxf(T.v1.y, T.v2.y));
    const bool c0 = (h0 <= yhi) && (h0 >= ylo), c1 = (h1 <= yhi) && (h1 >= ylo), c2 = (h2 <= yhi) && (h2 >= ylo);
    if (!(c0 || c1 || c2) || f == 0) continue;   // python keeps collision_faces > 0 only (body_measurements.py:161)
    mmi::Box tb = mmi::tri_box(T);
    if (!((-1.f <= tb.hi.x) && (1.f >= tb.lo.x) && (-1.f <= tb.hi.z) && (1.f >= tb.lo.z))) continue;
#pragma unroll
    for (int p = 0; p < 3; ++p) {
      if (!(p == 0 ? c0 : (p == 1 ? c1 : c2))) continue;
      const int slot = atomicAdd(&ncand, 2);
      if (slot + 1 < kMaxCand) { cand[slot] = (f << 3) | (p << 1); cand[slot + 1] = (f << 3) | (p << 1) | 1; }
    }
  }
  for (int o = 16; o; o >>= 1) vol += __shfl_xor_sync(0xffffffffu, vol, o);
  if (lane == 0) red[warp] = vol;
  __syncthreads();
  // ---- phase 2: exact SAT + "first ray hit" point selection, one (face, plane, query triangle) per thread
  {
    const int n = min(ncand, kMaxCand);
    if (ncand > kMaxCand && t == 0) overflow = 7;
    for (int i = t; i < n; i += blockDim.x) {
      const int c = cand[i], f = c >> 3, p = (c >> 1) & 3, q = c & 1;
      const float h = p == 0 ? h0 : (p == 1 ? h1 : h2);
      mmi::Tri T = tri_of(f);
      const mmi::Tri Q = quad(h, q);
      if (!mmi::sat11(Q, T)) continue;
      float3 b1 = make_float3(0, 0, 0), b2 = b1;
      mmi::isect_points(Q, T, b1, b2);  // no hit -> barycentrics stay 0 (first-body semantics)
      const int slot = atomicAdd(&cnt[p], 1);
      if (slot < kMaxPts) {
        float *o = pts + ((size_t)p * kMaxPts + slot) * 3;
        o[0] = T.v0.x * b1.x + T.v1.x * b1.y + T.v2.x * b1.z;
        o[1] = T.v0.y * b1.x + T.v1.y * b1.y + T.v2.y * b1.z;
        o[2] = T.v0.z * b1.x + T.v1.z * b1.y + T.v2.z * b1.z;
        if constexpr (GRAD) codes[p * kMaxPts + slot] = (f << 1) | q;
      }
    }
  }
  __syncthreads();     // the candidate queue is dead from here on: its storage becomes the chain lists
  if (!BWD && t == 0) {
    float v = 0.f;
    for (int i = 0; i < kThreads / 32; ++i) v += red[i];
    a.out[(size_t)b * 5 + 0] = fabsf(v) / 6.0f * 985.0f;
    a.out[(size_t)b * 5 + 1] = fabsf(lmy[0] - lmy[1]);
  }
  // ---- phase 3a: extreme points
  const int hp = warp / 8, hk = warp % 8;          // warps 0..23: (plane, chain)
  int n = 0;
  if (warp < 24) {
    n = cnt[hp];
    if (n > kMaxPts) { if (lane == 0) atomicOr(&overflow, 1 << hp); n = kMaxPts; }
    const float *P = pts + (size_t)hp * kMaxPts * 3;
    int best = -1;
    double b1 = 0, b2 = 0;
    for (int i = lane; i < n; i += 32) {
      double k1, k2;
      dir_key(P[3 * i], P[3 * i + 2], hk, k1, k2);
      if (best < 0 || k1 > b1 || (k1 == b1 && (k2 > b2 || (k2 == b2 && pt_order<GRAD>(P + 3 * i, P + 3 * best, codes, hp, i, best))))) {
        best = i; b1 = k1; b2 = k2;
      }
    }
    for (int o = 16; o; o >>= 1) {
      const int ob = __shfl_xor_sync(0xffffffffu, best, o);
      const double o1 = __shfl_xor_sync(0xffffffffu, b1, o), o2 = __shfl_xor_sync(0xffffffffu, b2, o);
      if (ob >= 0 && (best < 0 || o1 > b1 || (o1 == b1 && (o2 > b2 || (o2 == b2 && pt_order<GRAD>(P + 3 * ob, P + 3 * best, codes, hp, ob, best)))))) {
        best = ob; b1 = o1; b2 = o2;
      }
    }
    if (lane == 0) {
      Extreme e;
      e.idx = best;
      e.x = best >= 0 ? P[3 * best] : 0.f;
      e.z = best >= 0 ? P[3 * best + 2] : 0.f;
      ext[hp][hk] = e;
    }
  }
  __syncthreads();
  // ---- phase 3b: chain (plane hp, from E_hk to E_hk+1)
  if (warp < 24) {
    const float *P = pts + (size_t)hp * kMaxPts * 3;
    if (hk == 0) {
      if (a.cnt_out && lane == 0) a.cnt_out[(size_t)b * 3 + hp] = n;
      if (a.pts_out) {
        const int mcopy = min(n, a.maxp);
        for (int i = lane; i < mcopy * 3; i += 32) a.pts_out[(((size_t)b * 3 + hp) * a.maxp) * 3 + i] = P[i];
        if (n > a.maxp && lane == 0) atomicOr(&overflow, 8);
      }
    }
    float len = 0.f;
    int edges = 0;
    const Extreme e0 = ext[hp][hk], e1 = ext[hp][(hk + 1) & 7];
    if (n >= 3 && e0.idx >= 0 && !(e0.x == e1.x && e0.z == e1.z)) {
      // candidates of this chain: points on the outer side of (or on) the chord e0 -> e1
      unsigned short *L = clist + (size_t)warp * kChainCap;
      int nl = 0;
      bool listed = true;
      {
        const double ux = (double)e1.x - (double)e0.x, uz = (double)e1.z - (double)e0.z;
        for (int base = 0; base < n; base += 32) {
          const int i = base + lane;
          bool keep = false;
          if (i < n) {
            const double wx = (double)P[3 * i] - (double)e0.x, wz = (double)P[3 * i + 2] - (double)e0.z;
            keep = (ux * wz - uz * wx) <= 0.0;
          }
          const unsigned m = __ballot_sync(0xffffffffu, keep);
          const int pos = nl + __popc(m & ((1u << lane) - 1));
          if (keep && pos < kChainCap) L[pos] = (unsigned short)i;
          nl += __popc(m);
        }
        if (nl > kChainCap) listed = false;     // degenerate distribution: scan every point instead
        __syncwarp();
      }
      const int nscan = listed ? nl : n;
      int cur = e0.idx;
      float cx = e0.x, cz = e0.z;
      for (int it = 0; it < n + 1; ++it) {
        int nb = -1;
        float nx = 0.f, nz = 0.f;
        for (int q = lane; q < nscan; q += 32) {
          const int i = listed ? (int)L[q] : q;
          const float x = P[3 * i], z = P[3 * i + 2];
          if (x == cx && z == cz) continue;  // the point itself and its duplicates
          if (nb < 0 || better_next(cx, cz, nx, nz, x, z) || (x == nx && z == nz && pt_order<GRAD>(P + 3 * i, P + 3 * nb, codes, hp, i, nb))) {
            nb = i; nx = x; nz = z;
          }
        }
        for (int o = 16; o; o >>= 1) {
          const int ob = __shfl_xor_sync(0xffffffffu, nb, o);
          const float ox = __shfl_xor_sync(0xffffffffu, nx, o), oz = __shfl_xor_sync(0xffffffffu, nz, o);
          if (ob >= 0) {
            const bool take = nb < 0 || better_next(cx, cz, nx, nz, ox, oz) ||
                              (ox == nx && oz == nz && pt_order<GRAD>(P + 3 * ob, P + 3 * nb, codes, hp, ob, nb));
            if (take) { nb = ob; nx = ox; nz = oz; }
          }
        }
        nb = __shfl_sync(0xffffffffu, nb, 0);   // warp-uniform exits below: the shuffles above need every lane
        nx = __shfl_sync(0xffffffffu, nx, 0);
        nz = __shfl_sync(0xffffffffu, nz, 0);
        if (nb < 0) break;
        const float dx = P[3 * nb] - P[3 * cur], dy = P[3 * nb + 1] - P[3 * cur + 1], dz = P[3 * nb + 2] - P[3 * cur + 2];
        len += sqrtf(dx * dx + dy * dy + dz * dz);
        ++edges;
        if constexpr (GRAD) { if (lane == 0) nxt[hp * kMaxPts + cur] = (unsigned short)nb; }
        cur = nb; cx = nx; cz = nz;
        if (nx == e1.x && nz == e1.z) break;
      }
    }
    if (lane == 0) { chain_len[hp][hk] = len; chain_edges[hp][hk] = edges; }
  }
  __syncthreads();
  __shared__ float perim_s[3];
  if (t < 3) {
    const int p = t;
    float perim = 0.f;
    int edges = 0;
    for (int k = 0; k < 8; ++k) { perim += chain_len[p][k]; edges += chain_edges[p][k]; }
    // fewer than 3 hull edges: fewer than 3 points, or all of them collinear or coincident in xz.  The 8 extremes alone
    // cannot tell: a thin triangle's obtuse vertex is extreme in none of the 8 directions.  qhull raises on these.
    if (cnt[p] < 3 || edges < 3) perim = __int_as_float(0x7fc00000);
    if ((overflow & (1 << p))) perim = __int_as_float(0x7fc00000);   // truncated point set
    if constexpr (GRAD) perim_s[p] = perim;
    if constexpr (!BWD) a.out[(size_t)b * 5 + 2 + p] = perim;
  }
  if constexpr (!BWD) {
    if (t == 0 && overflow && a.status) atomicExch(a.status, 1);
  }
  if constexpr (MODE != kForward) {
    static_assert(BWD || SRC != kTriangles, "the Jacobian mode reads the model's faces and shape rows");
    // ---- phase 4: gradient or Jacobian.  The chain lists are dead: their storage holds the hull vertex list of each
    // plane (hull[p][j] = start slot of the j-th edge, chains in order) and, in gradient mode, then a bitmap of the
    // faces that carry a hull point.  The Jacobian mode builds what the gradient mode builds for an upstream gradient
    // of 1 on every output.
    unsigned short *hull = clist;                                                   // [3][kMaxPts]
    unsigned *fbits = reinterpret_cast<unsigned *>(clist + 3 * kMaxPts);
    const int nbits_words = (int)((kMaxCand * 4 - 3 * kMaxPts * 2) / 4);
    const bool all_flagged = a.F > nbits_words * 32;                                // bitmap too small: scan every face
    // mass scale, height scale, the 3 circumference gradients (NaN where the hull is unusable: a NaN circumference or
    // more than kMaxPts edges)
    __shared__ float gs[5];
    __shared__ int nedge[3], poison;
    const MeasureGrad &g = a.g;
    const float *go = BWD ? g.gout + (size_t)b * 5 : nullptr;
    if (t == 0) {
      auto up = [&](int k) { return BWD ? go[k] : 1.f; };                          // the upstream gradient
      float v = 0.f;
      for (int i = 0; i < kThreads / 32; ++i) v += red[i];                          // the forward's volume, same order
      gs[0] = up(0) * sign_of(v) * (985.0f / 6.0f);
      gs[1] = up(1) * sign_of(lmy[0] - lmy[1]);
      int bad = 0;
      for (int p = 0; p < 3; ++p) {
        int m = 0;
        for (int k = 0; k < 8; ++k) m += chain_edges[p][k];
        const bool usable = !isnan(perim_s[p]) && m <= kMaxPts, active = up(2 + p) != 0.f;
        gs[2 + p] = usable ? up(2 + p) : __int_as_float(0x7fc00000);
        nedge[p] = active && usable ? m : 0;
        bad |= active && !usable;
      }
      poison = BWD && bad;   // the Jacobian makes only the rows of unusable hulls NaN
    }
    if (warp < 24 && lane == 0) {
      int off = 0, m = 0;
      for (int k = 0; k < 8; ++k) { off += k < hk ? chain_edges[hp][k] : 0; m += chain_edges[hp][k]; }
      int cur = ext[hp][hk].idx;
      if (m <= kMaxPts)
        for (int s = 0; s < chain_edges[hp][hk]; ++s) { hull[hp * kMaxPts + off + s] = (unsigned short)cur; cur = nxt[hp * kMaxPts + cur]; }
    }
    if constexpr (BWD)
      for (int i = t; i < nbits_words; i += kThreads) fbits[i] = 0u;
    __syncthreads();
    // per hull vertex j of plane p: g (u_in - u_out), u the unit vectors of the edges into and out of it.  The walk is
    // one closed cycle (the end of each chain is the start of the next); a vertex where it is not poisons the body.
    float3 val[3];
    for (int it = 0; it < 3; ++it) {
      val[it] = make_float3(0.f, 0.f, 0.f);
      const int r = t + it * kThreads, p = r / kMaxPts, j = r % kMaxPts, m = nedge[p];
      if (j >= m) continue;
      const float *P = pts + (size_t)p * kMaxPts * 3;
      const unsigned short *H = hull + p * kMaxPts;
      const int cur = H[j], prev = H[(j + m - 1) % m], next = nxt[p * kMaxPts + cur];
      if (nxt[p * kMaxPts + prev] != cur || next != H[(j + 1) % m]) { poison = 1; continue; }
      const float ix = P[3 * cur] - P[3 * prev], iy = P[3 * cur + 1] - P[3 * prev + 1], iz = P[3 * cur + 2] - P[3 * prev + 2];
      const float ox = P[3 * next] - P[3 * cur], oy = P[3 * next + 1] - P[3 * cur + 1], oz = P[3 * next + 2] - P[3 * cur + 2];
      const float li = sqrtf(ix * ix + iy * iy + iz * iz), lo = sqrtf(ox * ox + oy * oy + oz * oz);
      const float gp = gs[2 + p];
      val[it] = make_float3(gp * (ix / li - ox / lo), gp * (iy / li - oy / lo), gp * (iz / li - oz / lo));
      if constexpr (BWD) {
        if (!all_flagged) {
          const int f = codes[p * kMaxPts + cur] >> 1;
          atomicOr(&fbits[f >> 5], 1u << (f & 31));
        }
      }
    }
    __syncthreads();                  // the points are dead: their storage takes the hull vertex vectors
    for (int it = 0; it < 3; ++it) {
      const int r = t + it * kThreads;
      if (r % kMaxPts < nedge[r / kMaxPts]) {
        pts[3 * r] = val[it].x; pts[3 * r + 1] = val[it].y; pts[3 * r + 2] = val[it].z;
      }
    }
    const float nan = __int_as_float(0x7fc00000);
    // sum of d det / d v over the (face, corner) entries e0..e1 of a vertex's incidence row, in that order
    auto incident_cross = [&](int e0, int e1) {
      float3 c = make_float3(0.f, 0.f, 0.f);
      for (int e = e0; e < e1; ++e) {
        const int fk = __ldg(g.inc + e);
        const float3 d = corner_cross(tri_of(fk / 3), fk % 3);
        c.x += d.x; c.y += d.y; c.z += d.z;
      }
      return c;
    };
    // the barycentrics phase 2 used for the point with (face, query half) code c of plane p, T the face's triangle
    auto hull_bc = [&](int p, int c, const mmi::Tri &T) {
      float3 b1 = make_float3(0, 0, 0), b2 = b1;
      mmi::isect_points(quad(hs[p], c & 1), T, b1, b2);
      return b1;
    };
    // exact modes: the ray that gave phase 2 that point, and the adjoint of its triangle's corner k for the hull vertex
    // vector at gv (returns the plane height's)
    auto hull_ray = [&](int p, int c, const mmi::Tri &T) { return mmi::isect_first_ray(quad(hs[p], c & 1), T); };
    auto hull_adj = [&](int p, int c, const mmi::Tri &T, int ray, const float *gv, int k, float3 &dk) {
      return hull_point_adjoint(T, quad(hs[p], c & 1), ray, hs[p], make_float3(gv[0], gv[1], gv[2]), k, dk);
    };
    // exact modes: gh[p], the adjoint of plane p's height, summed over its hull vertices in hull order by warp p
    float *gh = nullptr;
    if constexpr (EXACT) {
      __shared__ float gh_s[3];
      gh = gh_s;
      __syncthreads();
      if (warp < 3) {
        const int p = warp, m = nedge[p];
        float acc = 0.f;
        for (int base = 0; base < m; base += 32) {
          const int j = base + lane;
          float c = 0.f;
          if (j < m) {
            const int code = codes[p * kMaxPts + hull[p * kMaxPts + j]];
            const mmi::Tri T = tri_of(code >> 1);
            float3 dk;
            c = hull_adj(p, code, T, hull_ray(p, code, T), pts + 3 * (p * kMaxPts + j), 0, dk);
          }
          const int nj = min(32, m - base);
          for (int i = 0; i < nj; ++i) acc += __shfl_sync(0xffffffffu, c, i);
        }
        if (lane == 0) gh_s[p] = acc;
      }
    }
    if constexpr (BWD) {
      __syncthreads();
      const float sm = gs[0], sh = gs[1];
      const bool bad = poison != 0;
      // hull and height terms of corner k of face f (T = its triangle), in a fixed order: planes, hull order, (exact
      // modes) plane heights, height
      auto sparse = [&](int f, const mmi::Tri &T, int k, float3 &acc) {
        if (all_flagged || (fbits[f >> 5] >> (f & 31)) & 1u) {
          for (int p = 0; p < 3; ++p) {
            for (int j = 0; j < nedge[p]; ++j) {
              const int c = codes[p * kMaxPts + hull[p * kMaxPts + j]];
              if ((c >> 1) != f) continue;
              const float *gv = pts + 3 * (p * kMaxPts + j);
              if constexpr (EXACT) {
                float3 dk;
                hull_adj(p, c, T, hull_ray(p, c, T), gv, k, dk);
                acc.x += dk.x; acc.y += dk.y; acc.z += dk.z;
              } else {
                const float3 b1 = hull_bc(p, c, T);
                const float w = k == 0 ? b1.x : (k == 1 ? b1.y : b1.z);
                acc.x += w * gv[0]; acc.y += w * gv[1]; acc.z += w * gv[2];
              }
            }
          }
        }
        if constexpr (EXACT)
          for (int p = 0; p < 3; ++p)
            if (f == a.lm.face_idx[2 + p] && nedge[p] > 0) acc.y += gh[p] * a.lm.bc[2 + p][k];
        if (f == a.lm.face_idx[0]) acc.y += sh * a.lm.bc[0][k];
        if (f == a.lm.face_idx[1]) acc.y -= sh * a.lm.bc[1][k];
      };
      if constexpr (SRC == kTriangles) {
        for (int f = t; f < a.F; f += blockDim.x) {
          const mmi::Tri T = tri_of(f);
          float *o = g.grad + ((size_t)b * a.F + f) * 9;
          for (int k = 0; k < 3; ++k) {
            const float3 c = corner_cross(T, k);
            float3 acc = make_float3(sm * c.x, sm * c.y, sm * c.z);
            sparse(f, T, k, acc);
            o[3 * k] = bad ? nan : acc.x; o[3 * k + 1] = bad ? nan : acc.y; o[3 * k + 2] = bad ? nan : acc.z;
          }
        }
      } else {
        for (int v = t; v < a.V; v += blockDim.x) {
          const int e0 = __ldg(g.inc_ptr + v), e1 = __ldg(g.inc_ptr + v + 1);
          const float3 c = incident_cross(e0, e1);
          float3 acc = make_float3(sm * c.x, sm * c.y, sm * c.z);
          for (int e = e0; e < e1; ++e) {
            const int fk = __ldg(g.inc + e), f = fk / 3;
            bool want = all_flagged || f == a.lm.face_idx[0] || f == a.lm.face_idx[1] || ((fbits[f >> 5] >> (f & 31)) & 1u);
            if constexpr (EXACT) want = want || f == a.lm.face_idx[2] || f == a.lm.face_idx[3] || f == a.lm.face_idx[4];
            if (want) sparse(f, tri_of(f), fk % 3, acc);
          }
          float *o = g.grad + ((size_t)b * a.V + v) * 3;
          o[0] = bad ? nan : acc.x; o[1] = bad ? nan : acc.y; o[2] = bad ? nan : acc.z;
        }
      }
    } else {
      // Jacobian: row k of jac is S^T times the gradient for the cotangent e_k, S the nb shape rows of the basis.
      // Mass row: sum over the vertices of incident_cross . S[l][v], one thread per vertex at a time, then a fixed xor
      // tree per warp and the warps in order.
      __shared__ float jred[kThreads / 32][kMaxJacBetas];
      const int nb = g.nb;
      float part[kMaxJacBetas];
#pragma unroll
      for (int l = 0; l < kMaxJacBetas; ++l) part[l] = 0.f;
      for (int v = t; v < a.V; v += kThreads) {
        const float3 c = incident_cross(__ldg(g.inc_ptr + v), __ldg(g.inc_ptr + v + 1));
        const float *Sv = g.S + 3 * (size_t)v;
#pragma unroll
        for (int l = 0; l < kMaxJacBetas; ++l)
          if (l < nb) {
            const float *s = Sv + (size_t)l * g.ld;
            part[l] += c.x * __ldg(s) + c.y * __ldg(s + 1) + c.z * __ldg(s + 2);
          }
      }
#pragma unroll
      for (int l = 0; l < kMaxJacBetas; ++l) {
        if (l < nb) {
          float x = part[l];
          for (int o = 16; o; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
          if (lane == 0) jred[warp][l] = x;
        }
      }
      __syncthreads();
      const bool bad = poison != 0;
      float *J = g.jac + (size_t)b * 5 * nb;
      if (t < nb) {
        const int l = t;
        float s = 0.f;
        for (int w = 0; w < kThreads / 32; ++w) s += jred[w][l];
        J[l] = bad ? nan : gs[0] * s;
        // height row: the y components of the two landmark faces' corners
        const float *Sl = g.S + (size_t)l * g.ld + 1;
        float h = 0.f;
        for (int k = 0; k < 3; ++k) h += a.lm.bc[0][k] * __ldg(Sl + 3 * a.faces[3 * a.lm.face_idx[0] + k]);
        for (int k = 0; k < 3; ++k) h -= a.lm.bc[1][k] * __ldg(Sl + 3 * a.faces[3 * a.lm.face_idx[1] + k]);
        J[nb + l] = bad ? nan : gs[1] * h;
      }
      // circumference rows: warp (plane p, row l); lane i takes the hull vertices j = i mod 32, the bc-weighted sum
      // over its face's corners of (u_in - u_out) . S[l][corner], and the warp adds them in hull order
      for (int r = warp; r < 3 * nb; r += kThreads / 32) {
        const int p = r / nb, l = r % nb, m = nedge[p];
        const float *Sl = g.S + (size_t)l * g.ld;
        float acc = 0.f;
        for (int base = 0; base < m; base += 32) {
          const int j = base + lane;
          float c = 0.f;
          if (j < m) {
            const int code = codes[p * kMaxPts + hull[p * kMaxPts + j]], f = code >> 1;
            const float *gv = pts + 3 * (p * kMaxPts + j);
            if constexpr (EXACT) {
              // exact modes: the corner adjoints . S[l][corner]
              const mmi::Tri T = tri_of(f);
              const int ray = hull_ray(p, code, T);
              for (int k = 0; k < 3; ++k) {
                float3 dk;
                hull_adj(p, code, T, ray, gv, k, dk);
                const float *s = Sl + 3 * __ldg(a.faces + 3 * f + k);
                c += dk.x * __ldg(s) + dk.y * __ldg(s + 1) + dk.z * __ldg(s + 2);
              }
            } else {
              const float3 b1 = hull_bc(p, code, tri_of(f));
              for (int k = 0; k < 3; ++k) {
                const float w = k == 0 ? b1.x : (k == 1 ? b1.y : b1.z);
                const float *s = Sl + 3 * __ldg(a.faces + 3 * f + k);
                c += w * (gv[0] * __ldg(s) + gv[1] * __ldg(s + 1) + gv[2] * __ldg(s + 2));
              }
            }
          }
          const int nj = min(32, m - base);
          for (int i = 0; i < nj; ++i) acc += __shfl_sync(0xffffffffu, c, i);
        }
        if constexpr (EXACT) {
          // the plane height's adjoint gh[p] reaches the y components of the landmark face's corners
          if (lane == 0) {
            const int lf = a.lm.face_idx[2 + p];
            float hy = 0.f;
            for (int k = 0; k < 3; ++k) hy += a.lm.bc[2 + p][k] * __ldg(Sl + 3 * a.faces[3 * lf + k] + 1);
            acc += gh[p] * hy;
          }
        }
        if (lane == 0) J[(size_t)(2 + p) * nb + l] = (bad || isnan(gs[2 + p])) ? nan : acc;
      }
    }
  }
}

// Dynamic shared memory holds the staged vertices (when they fit under kMaxDynSmem), the point and candidate lists
// and, for the gradient and the Jacobian, the point codes and the hull walk: always more than the 48 KB default.
// kMaxDynSmem plus the largest static part (the Jacobian's 2 752 B) fits the SM's 227 KB.
constexpr size_t kMaxDynSmem = 220 * 1024;

template <int SRC, int MODE>
static int launch_source(const MeasureArgs &a, size_t smem, cudaStream_t stream) {
  static std::atomic<unsigned long long> attr_done{0};   // one per instantiation
  // set once per instantiation: the staged size varies with V, the others do not
  const int max_smem = (int)(SRC == kStagedVerts ? kMaxDynSmem : smem);
  SHAPY_CUDA_TRY(set_max_dynamic_smem(measure_smem_kernel<SRC, MODE>, max_smem, attr_done));
  measure_smem_kernel<SRC, MODE><<<a.B, kThreads, smem, stream>>>(a);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

// The work every entry shares: the landmark check, the status clear, and the source of the triangles with its
// shared memory.
template <int MODE>
static int launch_measure(const MeasureArgs &a, void *stream) {
  SHAPY_REQUIRE(a.B > 0 && a.F > 0, "shapy_measure: bad argument");
  for (int i = 0; i < 5; ++i)
    SHAPY_REQUIRE(a.lm.face_idx[i] >= 0 && a.lm.face_idx[i] < a.F, "landmark face %d out of range", a.lm.face_idx[i]);
  cudaStream_t s = (cudaStream_t)stream;
  if (a.status) SHAPY_CUDA_TRY(cudaMemsetAsync(a.status, 0, sizeof(int), s));
  const size_t list = kListBytes + (MODE == kForward ? 0 : kGradBytes);
  if constexpr (MODE != kJacobian && MODE != kJacobianExact)
    if (a.tris) return launch_source<kTriangles, MODE>(a, list, s);
  const size_t staged = (((size_t)a.V * 12 + 15) & ~(size_t)15) + list;
  if (a.V < 65536 && staged <= kMaxDynSmem) return launch_source<kStagedVerts, MODE>(a, staged, s);
  return launch_source<kGlobalVerts, MODE>(a, list, s);
}

}  // namespace shapy

using namespace shapy;

extern "C" int shapy_measure_forward(const float *v_shaped, const int32_t *faces, int batch, int num_verts,
                                     int num_faces, const shapy_measure_landmarks_t *lm, float *out,
                                     float *plane_points, int32_t *plane_counts, int max_points, int32_t *status,
                                     void *stream) {
  SHAPY_REQUIRE(v_shaped && faces && lm && out, "shapy_measure_forward: null argument");
  MeasureArgs a{v_shaped, faces, nullptr, batch, num_verts, num_faces, *lm, out, plane_points, plane_counts,
                max_points, status, MeasureGrad{}};
  return launch_measure<kForward>(a, stream);
}

extern "C" int shapy_measure_forward_tris(const float *triangles, int batch, int num_faces,
                                          const shapy_measure_landmarks_t *lm, float *out, float *plane_points,
                                          int32_t *plane_counts, int max_points, int32_t *status, void *stream) {
  SHAPY_REQUIRE(triangles && lm && out, "shapy_measure_forward_tris: null argument");
  MeasureArgs a{nullptr, nullptr, triangles, batch, 0, num_faces, *lm, out, plane_points, plane_counts, max_points,
                status, MeasureGrad{}};
  return launch_measure<kForward>(a, stream);
}

template <int MODE>
static int measure_backward(const char *name, const float *v_shaped, const int32_t *faces, const int32_t *inc_ptr,
                            const int32_t *inc, int batch, int num_verts, int num_faces,
                            const shapy_measure_landmarks_t *lm, const float *grad_out, float *grad_v, void *stream) {
  SHAPY_REQUIRE(v_shaped && faces && lm && grad_out && grad_v, "%s: null argument", name);
  SHAPY_REQUIRE(inc_ptr && inc && num_verts > 0, "%s: null incidence table", name);
  MeasureArgs a{v_shaped, faces, nullptr, batch, num_verts, num_faces, *lm, nullptr, nullptr, nullptr, 0, nullptr,
                MeasureGrad{grad_out, inc_ptr, inc, grad_v}};
  return launch_measure<MODE>(a, stream);
}

template <int MODE>
static int measure_backward_tris(const char *name, const float *triangles, int batch, int num_faces,
                                 const shapy_measure_landmarks_t *lm, const float *grad_out, float *grad_triangles,
                                 void *stream) {
  SHAPY_REQUIRE(triangles && lm && grad_out && grad_triangles, "%s: null argument", name);
  MeasureArgs a{nullptr, nullptr, triangles, batch, 0, num_faces, *lm, nullptr, nullptr, nullptr, 0, nullptr,
                MeasureGrad{grad_out, nullptr, nullptr, grad_triangles}};
  return launch_measure<MODE>(a, stream);
}

template <int MODE>
static int measure_jacobian_betas(const char *name, const shapy_smplx_t *m, const float *v_shaped,
                                  const int32_t *inc_ptr, const int32_t *inc, int batch,
                                  const shapy_measure_landmarks_t *lm, float *out, float *jac, int32_t *status,
                                  void *stream) {
  SHAPY_REQUIRE(m && v_shaped && inc_ptr && inc && lm && out && jac && batch > 0, "%s: bad argument", name);
  SHAPY_REQUIRE(((uintptr_t)v_shaped & 15) == 0, "%s: v_shaped must be 16-byte aligned", name);
  const SmplxDev &d = m->d;
  if (d.NB < 1 || d.NB > kMaxJacBetas) {
    set_error("%s: %d betas, at most %d are supported", name, d.NB, kMaxJacBetas);
    return SHAPY_ERR_UNSUPPORTED;
  }
  MeasureArgs a{v_shaped, d.faces, nullptr, batch, d.V, d.F, *lm, out, nullptr, nullptr, 0, status,
                MeasureGrad{nullptr, inc_ptr, inc, nullptr, d.basis, d.V3p, d.NB, jac}};
  return launch_measure<MODE>(a, stream);
}

extern "C" int shapy_measure_backward(const float *v_shaped, const int32_t *faces, const int32_t *inc_ptr,
                                      const int32_t *inc, int batch, int num_verts, int num_faces,
                                      const shapy_measure_landmarks_t *lm, const float *grad_out, float *grad_v,
                                      void *stream) {
  return measure_backward<kGradient>("shapy_measure_backward", v_shaped, faces, inc_ptr, inc, batch, num_verts,
                                     num_faces, lm, grad_out, grad_v, stream);
}

extern "C" int shapy_measure_backward_exact(const float *v_shaped, const int32_t *faces, const int32_t *inc_ptr,
                                            const int32_t *inc, int batch, int num_verts, int num_faces,
                                            const shapy_measure_landmarks_t *lm, const float *grad_out,
                                            float *grad_v, void *stream) {
  return measure_backward<kGradientExact>("shapy_measure_backward_exact", v_shaped, faces, inc_ptr, inc, batch,
                                          num_verts, num_faces, lm, grad_out, grad_v, stream);
}

extern "C" int shapy_measure_backward_tris(const float *triangles, int batch, int num_faces,
                                           const shapy_measure_landmarks_t *lm, const float *grad_out,
                                           float *grad_triangles, void *stream) {
  return measure_backward_tris<kGradient>("shapy_measure_backward_tris", triangles, batch, num_faces, lm, grad_out,
                                          grad_triangles, stream);
}

extern "C" int shapy_measure_backward_tris_exact(const float *triangles, int batch, int num_faces,
                                                 const shapy_measure_landmarks_t *lm, const float *grad_out,
                                                 float *grad_triangles, void *stream) {
  return measure_backward_tris<kGradientExact>("shapy_measure_backward_tris_exact", triangles, batch, num_faces, lm,
                                               grad_out, grad_triangles, stream);
}

extern "C" int shapy_measure_jacobian_betas(const shapy_smplx_t *m, const float *v_shaped, const int32_t *inc_ptr,
                                            const int32_t *inc, int batch, const shapy_measure_landmarks_t *lm,
                                            float *out, float *jac, int32_t *status, void *stream) {
  return measure_jacobian_betas<kJacobian>("shapy_measure_jacobian_betas", m, v_shaped, inc_ptr, inc, batch, lm, out,
                                           jac, status, stream);
}

extern "C" int shapy_measure_jacobian_betas_exact(const shapy_smplx_t *m, const float *v_shaped,
                                                  const int32_t *inc_ptr, const int32_t *inc, int batch,
                                                  const shapy_measure_landmarks_t *lm, float *out, float *jac,
                                                  int32_t *status, void *stream) {
  return measure_jacobian_betas<kJacobianExact>("shapy_measure_jacobian_betas_exact", m, v_shaped, inc_ptr, inc,
                                                batch, lm, out, jac, status, stream);
}
