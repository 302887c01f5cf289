// The conical distance-field self-penetration loss of SMPLify-X (reference mesh-mesh-intersection/
// mesh_mesh_intersection/loss.py, DistanceFieldPenetrationLoss with vectorized=True), forward and backward, at the
// face pairs of shapy_self_collisions.
//
//   penetration_forward_kernel    ONE CTA PER BODY: each thread sums its pairs (stride blockDim), then a fixed-order
//                                 tree reduction
//   penetration_backward_kernel   ONE CTA PER BODY: each pair writes the gradient of its six vertices to the workspace,
//                                 the (vertex, entry) keys are bitonic-sorted in shared memory, and the first entry of
//                                 each vertex's run sums the run in entry order
// No float atomics, so both are bit-identical run to run, and a body's result does not depend on the rest of the batch.
//
// A triangle (x0, x1, x2) is a cone: e0 = x1 - x0, e1 = x2 - x0, N = e0 x e1, unit axis n = N / |N|; with alpha = x0 - x2,
// beta = x1 - x2 the circumradius r = |alpha - beta| / (2 |N|) |alpha| |beta| and the circumcenter
// c = x2 + ((|alpha|^2 beta - |beta|^2 alpha) x (alpha x beta)) / (2 |N|^2)  (loss.py calc_circumcircle).  A point p:
// x = (p - c).n, a = |p - c - x n| / (-r / sigma x + r + 1e-6), psi = repulsion_intensity(x), u = (1 - a) psi,
// phi = ([a < 1] u^2)^2, and the point adds phi^2.  A pair adds its intruder's three vertices in the receiver's cone and
// its receiver's three vertices in the intruder's cone.  A zero-area face gives NaN, as in the reference.
#include "common.cuh"
#include "penetration.cuh"

namespace shapy {

constexpr int kPenMaxPairs = 4096;  // 6 entries per pair in the backward's 32768-key shared-memory sort

using PenCone = pen::Cone<float>;

__device__ __forceinline__ PenCone face_cone(const float *vb, const int v[3]) {
  return pen::make_cone(pen::ld<float>(vb + 3 * v[0]), pen::ld<float>(vb + 3 * v[1]), pen::ld<float>(vb + 3 * v[2]));
}

// The loss of one pair: intruder points in the receiver's cone, then receiver points in the intruder's cone.
__device__ __forceinline__ float pair_loss(const PenCone &rc, const PenCone &ic, const PenParams &pp) {
  float l = 0.f;
  for (int k = 0; k < 3; ++k) { const float f = pen::point_terms(ic.x[k], rc, pp).phi; l += f * f; }
  for (int k = 0; k < 3; ++k) { const float f = pen::point_terms(rc.x[k], ic, pp).phi; l += f * f; }
  return l;
}

// Gradient of g * phi^2 of the points `pts` in cone q: to the points in gp[3], to the cone's vertices in gq[3].
__device__ __forceinline__ void cone_points_backward(const PenCone &q, const pen::V3<float> pts[3], const PenParams &pp,
                                                     float g, pen::V3<float> gp[3], pen::V3<float> gq[3]) {
  pen::V3<float> gc{0.f, 0.f, 0.f}, gn = gc;
  float gr = 0.f;
  for (int k = 0; k < 3; ++k) {
    const pen::PointTerms<float> e = pen::point_terms(pts[k], q, pp);
    pen::point_backward(pts[k], q, e, pp, g * 2.f * e.phi, gp[k], gc, gn, gr);
  }
  pen::cone_backward(q, gc, gn, gr, gq);
}

__global__ void __launch_bounds__(256) penetration_forward_kernel(const float *__restrict__ vertices,
                                                                  const int *__restrict__ faces, int V, int F,
                                                                  const int *__restrict__ pairs, int C, PenParams pp,
                                                                  float *__restrict__ loss) {
  __shared__ float red[256];
  const int b = blockIdx.x, t = threadIdx.x;
  const float *vb = vertices + (size_t)b * V * 3;
  float l = 0.f;
  for (int p = t; p < C; p += blockDim.x) {
    int r[3], i[3];
    if (!pen::pair_faces(pairs + ((size_t)b * C + p) * 2, faces, F, r, i)) continue;
    l += pair_loss(face_cone(vb, r), face_cone(vb, i), pp);
  }
  red[t] = l;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (t < s) red[t] += red[t + s];
    __syncthreads();
  }
  if (t == 0) loss[b] = red[0];
}

// Dynamic smem: keys[npow2] (vertex, u32) + ids[npow2] (entry 6 pair + slot, u16).  contrib: [B][C][6][3].
__global__ void __launch_bounds__(512) penetration_backward_kernel(
    const float *__restrict__ vertices, const int *__restrict__ faces, int V, int F, const int *__restrict__ pairs,
    int C, PenParams pp, const float *__restrict__ grad_loss, int npow2, float *__restrict__ contrib,
    float *__restrict__ grad_v) {
  extern __shared__ __align__(16) unsigned char sm[];
  unsigned *keys = reinterpret_cast<unsigned *>(sm);
  unsigned short *ids = reinterpret_cast<unsigned short *>(sm + (size_t)npow2 * 4);
  const int b = blockIdx.x, t = threadIdx.x;
  const float *vb = vertices + (size_t)b * V * 3;
  float *cb = contrib + (size_t)b * C * 18;
  const float g = grad_loss[b];
  for (int p = t; p < C; p += blockDim.x) {
    int r[3], i[3];
    const bool ok = pen::pair_faces(pairs + ((size_t)b * C + p) * 2, faces, F, r, i);
    for (int k = 0; k < 6; ++k) keys[6 * p + k] = ok ? (unsigned)(k < 3 ? r[k] : i[k - 3]) : 0xFFFFFFFFu;
    if (!ok) continue;
    const PenCone rc = face_cone(vb, r), ic = face_cone(vb, i);
    pen::V3<float> gr3[3], gi3[3];
    for (int k = 0; k < 3; ++k) gr3[k] = gi3[k] = pen::V3<float>{0.f, 0.f, 0.f};
    cone_points_backward(rc, ic.x, pp, g, gi3, gr3);
    cone_points_backward(ic, rc.x, pp, g, gr3, gi3);
    float *o = cb + (size_t)p * 18;
    for (int k = 0; k < 3; ++k) {
      o[3 * k] = gr3[k].x; o[3 * k + 1] = gr3[k].y; o[3 * k + 2] = gr3[k].z;
      o[9 + 3 * k] = gi3[k].x; o[9 + 3 * k + 1] = gi3[k].y; o[9 + 3 * k + 2] = gi3[k].z;
    }
  }
  for (int e = 6 * C + t; e < npow2; e += blockDim.x) keys[e] = 0xFFFFFFFFu;
  for (int e = t; e < npow2; e += blockDim.x) ids[e] = (unsigned short)e;
  float *gb = grad_v + (size_t)b * V * 3;
  for (int e = t; e < V * 3; e += blockDim.x) gb[e] = 0.f;
  __syncthreads();
  for (int k = 2; k <= npow2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = t; i < npow2; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned ca = keys[i], cb2 = keys[ixj];
          const unsigned short ia = ids[i], ib = ids[ixj];
          const bool a_gt_b = ca > cb2 || (ca == cb2 && ia > ib);
          if (a_gt_b == ((i & k) == 0)) { keys[i] = cb2; keys[ixj] = ca; ids[i] = ib; ids[ixj] = ia; }
        }
      }
      __syncthreads();
    }
  }
  for (int i = t; i < npow2; i += blockDim.x) {
    const unsigned v = keys[i];
    if (v == 0xFFFFFFFFu || (i > 0 && keys[i - 1] == v)) continue;
    float s[3] = {0.f, 0.f, 0.f};
    for (int j = i; j < npow2 && keys[j] == v; ++j) {
      const float *c = cb + (size_t)ids[j] * 3;
      s[0] += c[0]; s[1] += c[1]; s[2] += c[2];
    }
    gb[3 * v] = s[0]; gb[3 * v + 1] = s[1]; gb[3 * v + 2] = s[2];
  }
}

static int pen_check(const char *name, int B, int V, int F, int C, float sigma, float linear_max) {
  SHAPY_REQUIRE(B >= 0 && V > 0 && F > 0 && C >= 0, "%s: bad sizes", name);
  SHAPY_REQUIRE(sigma > 0.f && !(linear_max != linear_max), "%s: sigma must be > 0 and linear_max not NaN", name);
  if (C > kPenMaxPairs) {
    set_error("%s: %d pairs per body exceed the %d supported (the backward sorts them in shared memory)", name, C,
              kPenMaxPairs);
    return SHAPY_ERR_UNSUPPORTED;
  }
  return SHAPY_OK;
}

}  // namespace shapy

using namespace shapy;

extern "C" int shapy_penetration_forward(const float *vertices, const int32_t *faces, int B, int V, int F,
                                         const int32_t *pairs, int C, float sigma, int penalize_outside,
                                         float linear_max, float *loss, void *stream) {
  const char *name = "shapy_penetration_forward";
  if (int rc = pen_check(name, B, V, F, C, sigma, linear_max)) return rc;
  if (B == 0) return SHAPY_OK;
  SHAPY_REQUIRE(vertices && faces && loss && (pairs || C == 0), "%s: null argument", name);
  const PenParams pp{sigma, linear_max, penalize_outside != 0};
  penetration_forward_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(vertices, faces, V, F, pairs, C, pp, loss);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

extern "C" size_t shapy_penetration_workspace_bytes(int B, int C) {
  if (B <= 0 || C <= 0) return 0;
  return (size_t)B * C * 18 * sizeof(float);
}

extern "C" int shapy_penetration_backward(const float *vertices, const int32_t *faces, int B, int V, int F,
                                          const int32_t *pairs, int C, float sigma, int penalize_outside,
                                          float linear_max, const float *grad_loss, float *grad_vertices,
                                          void *workspace, size_t workspace_bytes, void *stream) {
  const char *name = "shapy_penetration_backward";
  if (int rc = pen_check(name, B, V, F, C, sigma, linear_max)) return rc;
  if (B == 0) return SHAPY_OK;
  SHAPY_REQUIRE(vertices && faces && grad_loss && grad_vertices, "%s: null argument", name);
  cudaStream_t st = (cudaStream_t)stream;
  if (C == 0) {
    SHAPY_CUDA_TRY(cudaMemsetAsync(grad_vertices, 0, (size_t)B * V * 3 * sizeof(float), st));
    return SHAPY_OK;
  }
  SHAPY_REQUIRE(pairs && workspace && workspace_bytes >= shapy_penetration_workspace_bytes(B, C),
                "%s: null argument or workspace too small", name);
  int npow2 = 1;
  while (npow2 < 6 * C) npow2 <<= 1;
  const PenParams pp{sigma, linear_max, penalize_outside != 0};
  static std::atomic<unsigned long long> attr_done{0};
  SHAPY_CUDA_TRY(set_max_dynamic_smem(penetration_backward_kernel, 200 * 1024, attr_done));
  penetration_backward_kernel<<<B, 512, (size_t)npow2 * 6, st>>>(vertices, faces, V, F, pairs, C, pp, grad_loss,
                                                                  npow2, (float *)workspace, grad_vertices);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}
