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
#include "common.cuh"
#include "mmi_device.cuh"

namespace shapy {

constexpr int kThreads = 1024;
constexpr int kMaxPts = 1024;
constexpr int kMaxCand = 8192;     // (face, plane, query triangle) candidates that pass the AABB filter, per body; ints,
                                   // the buffer is reused for the per-chain candidate lists (u16) in phase 3
constexpr int kChainCap = 640;     // 24 chains x 640 x 2 B = 30 KB <= 32 KB
constexpr size_t kListBytes = 3 * kMaxPts * 12 + kMaxCand * 4;   // points + candidate queue, dynamic

enum TriSource { kStagedVerts, kGlobalVerts, kTriangles };

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

struct Extreme { float x, z; int idx; };

__device__ __forceinline__ void dir_key(float x, float z, int k, double &k1, double &k2) {
  // direction d_k = (dx, dz), k * 45 degrees (unnormalised, exact); tie-break direction = d_k rotated by +90 degrees
  const int dxs[8] = {1, 1, 0, -1, -1, -1, 0, 1}, dzs[8] = {0, 1, 1, 1, 0, -1, -1, -1};
  const double dx = dxs[k], dz = dzs[k];
  k1 = dx * (double)x + dz * (double)z;
  k2 = -dz * (double)x + dx * (double)z;
}

template <int SRC>
__global__ void __launch_bounds__(kThreads, 1) measure_smem_kernel(MeasureArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int nvf = a.V * 3;
  float *vs = reinterpret_cast<float *>(smem);                                      // [V * 3] (+ pad to 16 B)
  const size_t vs_bytes = SRC == kStagedVerts ? ((size_t)nvf * 4 + 15) & ~(size_t)15 : 0;
  float *pts = reinterpret_cast<float *>(smem + vs_bytes);                          // [3][kMaxPts][3]
  int *cand = reinterpret_cast<int *>(smem + vs_bytes + 3 * kMaxPts * 12);          // [kMaxCand]
  unsigned short *clist = reinterpret_cast<unsigned short *>(cand);                // phase 3: [24][kChainCap]
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
      mmi::Tri Q;
      Q.v0 = make_float3(-1.f, h, -1.f);
      Q.v1 = q == 0 ? make_float3(1.f, h, -1.f) : make_float3(1.f, h, 1.f);
      Q.v2 = q == 0 ? make_float3(1.f, h, 1.f) : make_float3(-1.f, h, 1.f);
      if (!mmi::sat11(Q, T)) continue;
      float3 b1 = make_float3(0, 0, 0), b2 = b1;
      mmi::isect_points(Q, T, b1, b2);  // no hit -> barycentrics stay 0 (first-body semantics)
      const int slot = atomicAdd(&cnt[p], 1);
      if (slot < kMaxPts) {
        float *o = pts + ((size_t)p * kMaxPts + slot) * 3;
        o[0] = T.v0.x * b1.x + T.v1.x * b1.y + T.v2.x * b1.z;
        o[1] = T.v0.y * b1.x + T.v1.y * b1.y + T.v2.y * b1.z;
        o[2] = T.v0.z * b1.x + T.v1.z * b1.y + T.v2.z * b1.z;
      }
    }
  }
  __syncthreads();     // the candidate queue is dead from here on: its storage becomes the chain lists
  if (t == 0) {
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
      if (best < 0 || k1 > b1 || (k1 == b1 && (k2 > b2 || (k2 == b2 && pt_before(P + 3 * i, P + 3 * best))))) {
        best = i; b1 = k1; b2 = k2;
      }
    }
    for (int o = 16; o; o >>= 1) {
      const int ob = __shfl_xor_sync(0xffffffffu, best, o);
      const double o1 = __shfl_xor_sync(0xffffffffu, b1, o), o2 = __shfl_xor_sync(0xffffffffu, b2, o);
      if (ob >= 0 && (best < 0 || o1 > b1 || (o1 == b1 && (o2 > b2 || (o2 == b2 && pt_before(P + 3 * ob, P + 3 * best)))))) {
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
          if (nb < 0 || better_next(cx, cz, nx, nz, x, z) || (x == nx && z == nz && pt_before(P + 3 * i, P + 3 * nb))) {
            nb = i; nx = x; nz = z;
          }
        }
        for (int o = 16; o; o >>= 1) {
          const int ob = __shfl_xor_sync(0xffffffffu, nb, o);
          const float ox = __shfl_xor_sync(0xffffffffu, nx, o), oz = __shfl_xor_sync(0xffffffffu, nz, o);
          if (ob >= 0) {
            const bool take = nb < 0 || better_next(cx, cz, nx, nz, ox, oz) ||
                              (ox == nx && oz == nz && pt_before(P + 3 * ob, P + 3 * nb));
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
        cur = nb; cx = nx; cz = nz;
        if (nx == e1.x && nz == e1.z) break;
      }
    }
    if (lane == 0) { chain_len[hp][hk] = len; chain_edges[hp][hk] = edges; }
  }
  __syncthreads();
  if (t < 3) {
    const int p = t;
    float perim = 0.f;
    int edges = 0;
    for (int k = 0; k < 8; ++k) { perim += chain_len[p][k]; edges += chain_edges[p][k]; }
    // fewer than 3 hull edges: fewer than 3 points, or all of them collinear or coincident in xz.  The 8 extremes alone
    // cannot tell: a thin triangle's obtuse vertex is extreme in none of the 8 directions.  qhull raises on these.
    if (cnt[p] < 3 || edges < 3) perim = __int_as_float(0x7fc00000);
    if ((overflow & (1 << p))) perim = __int_as_float(0x7fc00000);   // truncated point set
    a.out[(size_t)b * 5 + 2 + p] = perim;
  }
  if (t == 0 && overflow && a.status) atomicExch(a.status, 1);
}

size_t measure_smem_bytes(int V) { return (((size_t)V * 12 + 15) & ~(size_t)15) + kListBytes; }

template <int SRC>
static int launch_source(const MeasureArgs &a, size_t smem, int max_smem, cudaStream_t stream) {
  static std::atomic<unsigned long long> attr_done{0};   // one per instantiation
  SHAPY_CUDA_TRY(set_max_dynamic_smem(measure_smem_kernel<SRC>, max_smem, attr_done));
  measure_smem_kernel<SRC><<<a.B, kThreads, smem, stream>>>(a);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

}  // namespace shapy

using namespace shapy;

static int launch_measure(MeasureArgs a, void *stream) {
  SHAPY_REQUIRE(a.out && a.B > 0 && a.F > 0, "shapy_measure: bad argument");
  for (int i = 0; i < 5; ++i)
    SHAPY_REQUIRE(a.lm.face_idx[i] >= 0 && a.lm.face_idx[i] < a.F, "landmark face %d out of range", a.lm.face_idx[i]);
  cudaStream_t s = (cudaStream_t)stream;
  if (a.status) SHAPY_CUDA_TRY(cudaMemsetAsync(a.status, 0, sizeof(int), s));
  if (a.tris) return launch_source<kTriangles>(a, kListBytes, (int)kListBytes, s);          // 68 KB > 48 KB default
  if (a.V < 65536 && measure_smem_bytes(a.V) <= 220 * 1024)
    return launch_source<kStagedVerts>(a, measure_smem_bytes(a.V), 226 * 1024, s);        // + 656 B static <= 227 KB
  return launch_source<kGlobalVerts>(a, kListBytes, (int)kListBytes, s);
}

extern "C" int shapy_measure_forward(const float *v_shaped, const int32_t *faces, int batch, int num_verts,
                                     int num_faces, const shapy_measure_landmarks_t *lm, float *out,
                                     float *plane_points, int32_t *plane_counts, int max_points, int32_t *status,
                                     void *stream) {
  SHAPY_REQUIRE(v_shaped && faces && lm, "shapy_measure_forward: null argument");
  MeasureArgs a{v_shaped, faces, nullptr, batch, num_verts, num_faces, *lm, out, plane_points, plane_counts,
                max_points, status};
  return launch_measure(a, stream);
}

extern "C" int shapy_measure_forward_tris(const float *triangles, int batch, int num_faces,
                                          const shapy_measure_landmarks_t *lm, float *out, float *plane_points,
                                          int32_t *plane_counts, int max_points, int32_t *status, void *stream) {
  SHAPY_REQUIRE(triangles && lm, "shapy_measure_forward_tris: null argument");
  MeasureArgs a{nullptr, nullptr, triangles, batch, 0, num_faces, *lm, out, plane_points, plane_counts, max_points,
                status};
  return launch_measure(a, stream);
}
