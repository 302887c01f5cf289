// Evaluation metric on the GPU (SURVEY.md 8f rank 3): point-to-point error between two meshes of different topology
// through sparse point regressors, translation aligned.  Replaces regressor/human_shape/utils/metrics.py:368-456, which
// the reference runs in float64 on the CPU after a device->host copy of every predicted mesh (evaluation.py:227-265).
// HBM / latency bound: (V1 + V2) * 12 B read per body, P * 4 B written.  All reductions are deterministic (fixed order).
#include "common.cuh"
#include "metrics.cuh"

namespace shapy {

// d[b][p] = input point - target point
__global__ void __launch_bounds__(256) p2p_diff_kernel(const int *__restrict__ rp_in, const int *__restrict__ col_in,
                                                       const float *__restrict__ val_in, const int *__restrict__ rp_tg,
                                                       const int *__restrict__ col_tg, const float *__restrict__ val_tg,
                                                       const float *__restrict__ v_in, const float *__restrict__ v_tg, int B, int P,
                                                       int V1, int V2, float *__restrict__ d) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (p >= P || b >= B) return;
  float a[3], c[3];
  csr_row_point(rp_in, col_in, val_in, v_in + (size_t)b * V1 * 3, p, a);
  csr_row_point(rp_tg, col_tg, val_tg, v_tg + (size_t)b * V2 * 3, p, c);
  float *o = d + ((size_t)b * P + p) * 3;
  o[0] = a[0] - c[0]; o[1] = a[1] - c[1]; o[2] = a[2] - c[2];
}

// same-topology variant (PointError with TranslationAlignment / NoAlignment, metrics.py:232-277, 335-366): d = est - gt
__global__ void __launch_bounds__(256) v2v_diff_kernel(const float *__restrict__ v_in, const float *__restrict__ v_tg, size_t n,
                                                       float *__restrict__ d) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) d[i] = v_in[i] - v_tg[i];
}

// one block per body: t = -mean_p d  (= mean target - mean input), or 0 without alignment
__global__ void __launch_bounds__(256) p2p_translation_kernel(const float *__restrict__ d, int P, int align, float *__restrict__ t) {
  __shared__ float s[3][256];
  const int b = blockIdx.x;
  float x = 0.f, y = 0.f, z = 0.f;
  if (align)
    for (int p = threadIdx.x; p < P; p += 256) {
      const float *q = d + ((size_t)b * P + p) * 3;
      x += q[0]; y += q[1]; z += q[2];
    }
  s[0][threadIdx.x] = x; s[1][threadIdx.x] = y; s[2][threadIdx.x] = z;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if (threadIdx.x < w)
      for (int c = 0; c < 3; ++c) s[c][threadIdx.x] += s[c][threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x < 3) t[b * 3 + threadIdx.x] = -s[threadIdx.x][0] / (float)P;
}

// one block per body: error[b][p] = |d + t|, mean[b]
__global__ void __launch_bounds__(256) p2p_error_kernel(const float *__restrict__ d, const float *__restrict__ t, int P,
                                                        float *__restrict__ error, float *__restrict__ mean) {
  __shared__ float s[256];
  const int b = blockIdx.x;
  const float tb[3] = {t[b * 3], t[b * 3 + 1], t[b * 3 + 2]};
  float acc = 0.f;
  for (int p = threadIdx.x; p < P; p += 256) {
    const float e = aligned_error(d + ((size_t)b * P + p) * 3, tb);
    error[(size_t)b * P + p] = e;
    acc += e;
  }
  s[threadIdx.x] = acc;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if (threadIdx.x < w) s[threadIdx.x] += s[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) mean[b] = s[0] / (float)P;
}

// ---------------------------------------------------------------------------------------------------------------------
// PointError with ScaleAlignment / RootAlignment on same-topology point sets (metrics.py:173-229, 279-303, 335-366).
// Per body: statistics (8 floats: centre of est, centre of gt, scale, unused) into the workspace, then the error pass.
// Every reduction runs in a fixed order over a fixed block of 256 threads, so a body's result does not depend on the run
// or on the other bodies of the batch.
constexpr int kStats = 8;

struct RootList {
  int n;
  int idx[SHAPY_MAX_ROOTS];   // validated and made non-negative on the host
};

// in-place sum over the 256 threads of the block of N values each, fixed tree order; every thread gets the totals
template <int N>
__device__ __forceinline__ void block_sum256(float (&v)[N], float (*sh)[256]) {
  for (int c = 0; c < N; ++c) sh[c][threadIdx.x] = v[c];
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if (threadIdx.x < w)
      for (int c = 0; c < N; ++c) sh[c][threadIdx.x] += sh[c][threadIdx.x + w];
    __syncthreads();
  }
  for (int c = 0; c < N; ++c) v[c] = sh[c][0];
  __syncthreads();
}

// one block per body: mu1, mu2, then s = sqrt(var2 / var1) from the centred sums of squares in a second pass over the
// body (still in L2).  The means are taken about the body's first point, so the sums carry body-sized offsets rather than
// the metre-sized coordinates of a mesh far from the origin.  var1 == 0 is not guarded: s is what fp32 makes of it.
__global__ void __launch_bounds__(256) scale_stats_kernel(const float *__restrict__ est, const float *__restrict__ gt, int P,
                                                          float *__restrict__ stats) {
  __shared__ float sh[6][256];
  const int b = blockIdx.x;
  const float *a = est + (size_t)b * P * 3, *c = gt + (size_t)b * P * 3;
  float v[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int p = threadIdx.x; p < P; p += 256)
    for (int k = 0; k < 3; ++k) {
      v[k] += a[(size_t)p * 3 + k] - a[k];
      v[3 + k] += c[(size_t)p * 3 + k] - c[k];
    }
  block_sum256<6>(v, sh);
  float mu[6];
  for (int k = 0; k < 3; ++k) {
    mu[k] = a[k] + v[k] / (float)P;
    mu[3 + k] = c[k] + v[3 + k] / (float)P;
  }
  float q[2] = {0.f, 0.f};
  for (int p = threadIdx.x; p < P; p += 256)
    for (int k = 0; k < 3; ++k) {
      const float x = a[(size_t)p * 3 + k] - mu[k], y = c[(size_t)p * 3 + k] - mu[3 + k];
      q[0] += x * x;
      q[1] += y * y;
    }
  block_sum256<2>(q, sh);
  if (threadIdx.x == 0) {
    float *st = stats + (size_t)b * kStats;
    for (int k = 0; k < 6; ++k) st[k] = mu[k];
    st[6] = sqrtf(q[1] / q[0]);
    st[7] = 0.f;
  }
}

// one thread per (body, side, coordinate): the mean of the root points in list order; an empty list gives 0 / 0 = NaN,
// the mean numpy takes of an empty axis
__global__ void __launch_bounds__(128) root_stats_kernel(const float *__restrict__ est, const float *__restrict__ gt, int B, int P,
                                                         RootList roots, float *__restrict__ stats) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * 6) return;
  const int b = i / 6, side = (i % 6) / 3, k = i % 3;
  const float *x = (side ? gt : est) + (size_t)b * P * 3;
  float s = 0.f;
  for (int r = 0; r < roots.n; ++r) s += x[(size_t)roots.idx[r] * 3 + k];
  float *st = stats + (size_t)b * kStats;
  st[side * 3 + k] = s / (float)roots.n;
  if (side == 0 && k == 0) { st[6] = 1.f; st[7] = 0.f; }
}

// one block per body: error[b][p] with the body's statistics, mean[b]
__global__ void __launch_bounds__(256) aligned_point_error_kernel(const float *__restrict__ est, const float *__restrict__ gt,
                                                                  const float *__restrict__ stats, int P, int mode,
                                                                  float *__restrict__ error, float *__restrict__ mean) {
  __shared__ float sh[1][256];
  const int b = blockIdx.x;
  const float *a = est + (size_t)b * P * 3, *c = gt + (size_t)b * P * 3, *st = stats + (size_t)b * kStats;
  const float ca[3] = {st[0], st[1], st[2]}, cc[3] = {st[3], st[4], st[5]}, s = st[6];
  float acc[1] = {0.f};
  for (int p = threadIdx.x; p < P; p += 256) {
    const float e = mode == SHAPY_ALIGN_SCALE ? scaled_error(a + (size_t)p * 3, c + (size_t)p * 3, ca, cc, s)
                                              : root_error(a + (size_t)p * 3, c + (size_t)p * 3, ca, cc);
    error[(size_t)b * P + p] = e;
    acc[0] += e;
  }
  block_sum256<1>(acc, sh);
  if (threadIdx.x == 0) mean[b] = acc[0] / (float)P;
}

// points[b][p] = row p of the CSR regressor times the vertices of body b (the J14 einsum of evaluation.py:183-184)
__global__ void __launch_bounds__(256) regress_points_kernel(const int *__restrict__ row_ptr, const int *__restrict__ col,
                                                             const float *__restrict__ val, const float *__restrict__ verts, int B,
                                                             int P, int V, float *__restrict__ points) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)B * P) return;
  const int b = (int)(i / P), p = (int)(i % P);
  csr_row_point(row_ptr, col, val, verts + (size_t)b * V * 3, p, points + i * 3);
}

}  // namespace shapy

using namespace shapy;

extern "C" size_t shapy_p2p_workspace_bytes(int B, int P) { return (size_t)B * P * 3 * sizeof(float) + (size_t)B * 3 * sizeof(float) + 256; }

extern "C" int shapy_p2p_error(const int *in_row_ptr, const int *in_col, const float *in_val, const int *tg_row_ptr, const int *tg_col,
                               const float *tg_val, const float *input_vertices, const float *target_vertices, int B, int P, int V1,
                               int V2, int align, float *error, float *mean_error, void *workspace, size_t workspace_bytes,
                               void *stream) {
  SHAPY_REQUIRE(in_row_ptr && in_col && in_val && tg_row_ptr && tg_col && tg_val && input_vertices && target_vertices && error &&
                    mean_error && workspace,
                "shapy_p2p_error: null argument");
  SHAPY_REQUIRE(B > 0 && B <= 65535 && P > 0 && V1 > 0 && V2 > 0, "shapy_p2p_error: bad sizes");
  SHAPY_REQUIRE(workspace_bytes >= shapy_p2p_workspace_bytes(B, P), "shapy_p2p_error: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  float *d = (float *)workspace;
  float *t = d + (size_t)B * P * 3;
  p2p_diff_kernel<<<dim3(ceil_div(P, 256), B), 256, 0, st>>>(in_row_ptr, in_col, in_val, tg_row_ptr, tg_col, tg_val, input_vertices,
                                                             target_vertices, B, P, V1, V2, d);
  SHAPY_LAUNCH_CHECK();
  p2p_translation_kernel<<<B, 256, 0, st>>>(d, P, align, t);
  SHAPY_LAUNCH_CHECK();
  p2p_error_kernel<<<B, 256, 0, st>>>(d, t, P, error, mean_error);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

extern "C" int shapy_v2v_error(const float *input_vertices, const float *target_vertices, int B, int V, int align, float *error,
                               float *mean_error, void *workspace, size_t workspace_bytes, void *stream) {
  SHAPY_REQUIRE(input_vertices && target_vertices && error && mean_error && workspace, "shapy_v2v_error: null argument");
  SHAPY_REQUIRE(B > 0 && B <= 65535 && V > 0, "shapy_v2v_error: bad sizes");
  SHAPY_REQUIRE(workspace_bytes >= shapy_p2p_workspace_bytes(B, V), "shapy_v2v_error: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  float *d = (float *)workspace;
  float *t = d + (size_t)B * V * 3;
  const size_t n = (size_t)B * V * 3;
  v2v_diff_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(input_vertices, target_vertices, n, d);
  SHAPY_LAUNCH_CHECK();
  p2p_translation_kernel<<<B, 256, 0, st>>>(d, V, align, t);
  SHAPY_LAUNCH_CHECK();
  p2p_error_kernel<<<B, 256, 0, st>>>(d, t, V, error, mean_error);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

extern "C" size_t shapy_point_error_workspace_bytes(int B) { return (size_t)(B > 0 ? B : 0) * kStats * sizeof(float); }

extern "C" int shapy_point_error_aligned(const float *input_points, const float *target_points, int B, int P, int mode,
                                         const int *roots, int num_roots, float *error, float *mean_error, void *workspace,
                                         size_t workspace_bytes, void *stream) {
  SHAPY_REQUIRE(input_points && target_points && error && mean_error && workspace, "shapy_point_error_aligned: null argument");
  SHAPY_REQUIRE(B > 0 && B <= 65535 && P > 0, "shapy_point_error_aligned: bad sizes (batch %d, points %d)", B, P);
  SHAPY_REQUIRE(mode == SHAPY_ALIGN_SCALE || mode == SHAPY_ALIGN_ROOT, "shapy_point_error_aligned: unknown alignment mode %d", mode);
  SHAPY_REQUIRE(workspace_bytes >= shapy_point_error_workspace_bytes(B), "shapy_point_error_aligned: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  float *stats = (float *)workspace;
  if (mode == SHAPY_ALIGN_SCALE) {
    scale_stats_kernel<<<B, 256, 0, st>>>(input_points, target_points, P, stats);
  } else {
    SHAPY_REQUIRE(num_roots >= 0 && num_roots <= SHAPY_MAX_ROOTS, "shapy_point_error_aligned: %d root indices (at most %d)",
                  num_roots, SHAPY_MAX_ROOTS);
    SHAPY_REQUIRE(roots || num_roots == 0, "shapy_point_error_aligned: null root list");
    RootList rl{};
    rl.n = num_roots;
    for (int r = 0; r < num_roots; ++r) {      // numpy indexing: -P <= index < P, negative counts from the end
      SHAPY_REQUIRE(roots[r] >= -P && roots[r] < P, "shapy_point_error_aligned: root index %d out of range for %d points",
                    roots[r], P);
      rl.idx[r] = roots[r] < 0 ? roots[r] + P : roots[r];
    }
    root_stats_kernel<<<ceil_div(B * 6, 128), 128, 0, st>>>(input_points, target_points, B, P, rl, stats);
  }
  SHAPY_LAUNCH_CHECK();
  aligned_point_error_kernel<<<B, 256, 0, st>>>(input_points, target_points, stats, P, mode, error, mean_error);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

extern "C" int shapy_regress_points(const int *row_ptr, const int *col, const float *val, const float *vertices, int B, int P,
                                    int V, float *points, void *stream) {
  SHAPY_REQUIRE(row_ptr && col && val && vertices && points, "shapy_regress_points: null argument");
  SHAPY_REQUIRE(B > 0 && P > 0 && V > 0 && (long long)B * P <= (long long)INT32_MAX * 256, "shapy_regress_points: bad sizes");
  const long long n = (long long)B * P;
  regress_points_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(row_ptr, col, val, vertices, B, P, V,
                                                                                       points);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}
