// Silhouette term of the perspective 2D fit: the exact distance transform and contour of person masks, the model ->
// mask distance of the projected vertices and its backward, and a pixel-centre silhouette rasteriser.
//
//   sil_edt_columns_kernel   per column: the vertical distance g to the nearest person pixel (H + W when the column has
//                            none), in integers, written as int32 into `dist`
//   sil_edt_rows_kernel      ONE WARP PER ROW: lane 0 builds the lower envelope of the parabolas (x - i)^2 + g_i^2
//                            (Meijster's second phase, integer separators), then every lane reads its pixels' minimum
//                            from the envelope; dist = sqrtf((float)d^2), 0 everywhere for an empty mask
//   sil_contour_count_kernel per row: the contour pixels (person pixels with a 4-neighbour inside the image that is not
//                            a person pixel)
//   sil_contour_scan_kernel  ONE CTA PER BODY: exclusive scan of the row counts, the count, the padding rows
//   sil_contour_write_kernel per row: each contour pixel's raster rank j; every k-th (k = ceil(count / max_points)) is
//                            written at j / k as (x = c, y = r, 0) with weight 1
//   sil_forward_kernel       ONE CTA PER BODY: the projected mesh (u, v, 0) and the mean of D(clamp(u, v))^2, a
//                            fixed-order tree reduction
//   sil_backward_kernel      per vertex: the chain rule through the projection of the bilinear-D gradient and of the
//                            (u, v) cotangent of the mask -> model term
//   sil_render_kernel        ONE WARP PER TRIANGLE: the pixel centres of its box inside the projected triangle (all
//                            three Y_z > 0, inclusive float edge test) are set to 1
// No float atomics anywhere: every output is bit-identical run to run and a body's result does not depend on the batch.
// The file is compiled with -fmad=false, so the projection and the edge test round like their NumPy restatement
// (tests/silhouette_oracle.py).
#include "common.cuh"

namespace shapy {

constexpr int kSilMaxSide = 4096;      // H, W: the row pass keeps a row's g and envelope in 8 W bytes of smem
constexpr int kSilMaxPoints = 32768;   // the contour is the `points` input of shapy_closest_points
constexpr float kSilZNear = 1e-3f;     // the projection depth of the model -> mask term is max(Y_z, z_near)

__global__ void __launch_bounds__(128) sil_edt_columns_kernel(const uint8_t *__restrict__ masks, int H, int W,
                                                              int *__restrict__ g) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (x >= W) return;
  const uint8_t *m = masks + (size_t)b * H * W + x;
  int *gb = g + (size_t)b * H * W + x;
  const int inf = H + W;
  int d = inf;
  for (int y = 0; y < H; ++y) {
    d = m[(size_t)y * W] ? 0 : min(d + 1, inf);
    gb[(size_t)y * W] = d;
  }
  d = inf;
  for (int y = H - 1; y >= 0; --y) {
    const int cur = gb[(size_t)y * W];
    d = cur == 0 ? 0 : min(d + 1, inf);
    if (d < cur) gb[(size_t)y * W] = d;
  }
}

// In place: the row's g is read whole into shared memory before any of its distances is written.
__global__ void __launch_bounds__(32) sil_edt_rows_kernel(int H, int W, float *__restrict__ dist) {
  extern __shared__ int sil_sm[];
  int *gr = sil_sm;
  short *s = reinterpret_cast<short *>(sil_sm + W), *t = s + W;
  __shared__ int nseg;
  const int y = blockIdx.x, b = blockIdx.y, lane = threadIdx.x;
  float *row = dist + ((size_t)b * H + y) * W;
  const int *grow = reinterpret_cast<const int *>(row);
  for (int x = lane; x < W; x += 32) gr[x] = grow[x];
  __syncwarp();
  if (lane == 0) {
    // f_i(x) = (x - i)^2 + g_i^2; sep(i, u) = floor of the abscissa where f_u starts to win over f_i (i < u), which
    // is >= 0 whenever it is taken, so integer division truncates like floor
    auto f = [&](int x, int i) { return (x - i) * (x - i) + gr[i] * gr[i]; };
    int q = 0;
    s[0] = 0;
    t[0] = 0;
    for (int u = 1; u < W; ++u) {
      while (q >= 0 && f(t[q], s[q]) > f(t[q], u)) --q;
      if (q < 0) {
        q = 0;
        s[0] = (short)u;
      } else {
        const int i = s[q];
        const int w = 1 + (u * u - i * i + gr[u] * gr[u] - gr[i] * gr[i]) / (2 * (u - i));
        if (w < W) {
          ++q;
          s[q] = (short)u;
          t[q] = (short)w;
        }
      }
    }
    nseg = q + 1;
  }
  __syncwarp();
  const int inf2 = (H + W) * (H + W);
  for (int x = lane; x < W; x += 32) {
    int lo = 0, hi = nseg - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (t[mid] <= x) lo = mid; else hi = mid - 1;
    }
    const int i = s[lo];
    const int d2 = (x - i) * (x - i) + gr[i] * gr[i];
    row[x] = d2 >= inf2 ? 0.f : sqrtf((float)d2);
  }
}

__device__ __forceinline__ bool sil_contour(const uint8_t *m, int H, int W, int r, int c) {
  const uint8_t *p = m + (size_t)r * W + c;
  if (!p[0]) return false;
  return (c > 0 && !p[-1]) || (c + 1 < W && !p[1]) || (r > 0 && !p[-W]) || (r + 1 < H && !p[W]);
}

__global__ void __launch_bounds__(128) sil_contour_count_kernel(const uint8_t *__restrict__ masks, int H, int W,
                                                                int *__restrict__ rows) {
  const int r = blockIdx.x, b = blockIdx.y;
  const uint8_t *m = masks + (size_t)b * H * W;
  int n = 0;
  for (int x0 = 0; x0 < W; x0 += blockDim.x) {
    const int c = x0 + threadIdx.x;
    n += __syncthreads_count(c < W && sil_contour(m, H, W, r, c));
  }
  if (threadIdx.x == 0) rows[(size_t)b * H + r] = n;
}

// rows (B, H) counts -> exclusive offsets in place; count (B); the padding entries [kept, max_points) zeroed.
__global__ void __launch_bounds__(1024) sil_contour_scan_kernel(int H, int max_points, int *__restrict__ rows,
                                                                int32_t *__restrict__ count, float *__restrict__ contour,
                                                                float *__restrict__ contour_w) {
  __shared__ int wsum[32];
  __shared__ int carry;
  const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  int *rb = rows + (size_t)b * H;
  if (t == 0) carry = 0;
  __syncthreads();
  for (int r0 = 0; r0 < H; r0 += 1024) {
    const int v = r0 + t < H ? rb[r0 + t] : 0;
    int incl = v;
    for (int o = 1; o < 32; o <<= 1) {
      const int n = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += n;
    }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int w = wsum[lane], wi = w;
      for (int o = 1; o < 32; o <<= 1) {
        const int n = __shfl_up_sync(0xffffffffu, wi, o);
        if (lane >= o) wi += n;
      }
      wsum[lane] = wi - w;
    }
    __syncthreads();
    if (r0 + t < H) rb[r0 + t] = carry + wsum[warp] + incl - v;
    __syncthreads();
    if (t == 1023) carry += wsum[31] + incl;
    __syncthreads();
  }
  const int total = carry;
  if (t == 0) count[b] = total;
  const int k = total > max_points ? (total + max_points - 1) / max_points : 1;
  const int kept = (total + k - 1) / k;
  for (int i = kept + t; i < max_points; i += blockDim.x) {
    float *p = contour + ((size_t)b * max_points + i) * 3;
    p[0] = p[1] = p[2] = 0.f;
    contour_w[(size_t)b * max_points + i] = 0.f;
  }
}

__global__ void __launch_bounds__(128) sil_contour_write_kernel(const uint8_t *__restrict__ masks, int H, int W,
                                                                int max_points, const int *__restrict__ rows,
                                                                const int32_t *__restrict__ count,
                                                                float *__restrict__ contour,
                                                                float *__restrict__ contour_w) {
  __shared__ int wcnt[4];
  const int r = blockIdx.x, b = blockIdx.y, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const uint8_t *m = masks + (size_t)b * H * W;
  const int total = count[b];
  const int k = total > max_points ? (total + max_points - 1) / max_points : 1;
  int base = rows[(size_t)b * H + r];
  for (int x0 = 0; x0 < W; x0 += 128) {
    const int c = x0 + t;
    const bool on = c < W && sil_contour(m, H, W, r, c);
    const unsigned bal = __ballot_sync(0xffffffffu, on);
    if (lane == 0) wcnt[warp] = __popc(bal);
    __syncthreads();
    int before = base + __popc(bal & ((1u << lane) - 1u));
    for (int w = 0; w < warp; ++w) before += wcnt[w];
    if (on && before % k == 0) {
      const int i = before / k;
      float *p = contour + ((size_t)b * max_points + i) * 3;
      p[0] = (float)c;
      p[1] = (float)r;
      p[2] = 0.f;
      contour_w[(size_t)b * max_points + i] = 1.f;
    }
    base += wcnt[0] + wcnt[1] + wcnt[2] + wcnt[3];
    __syncthreads();
  }
}

struct SilProj {
  float u, v, zc;   // the projection at depth zc = max(Y_z, z_near)
};

__device__ __forceinline__ SilProj sil_project(const float *y, const float *intr) {
  const float zc = fmaxf(y[2], kSilZNear);
  return {intr[0] * (y[0] / zc) + intr[1], intr[0] * (y[1] / zc) + intr[2], zc};
}

// D at (u, v) clamped to the rectangle of pixel centres, bilinear in the cell [c0, c0 + 1] x [r0, r0 + 1] with
// c0 = min(floor(x), W - 2) (0 when W = 1); its partial derivatives in u and v (0 along a clamped axis).
struct SilSample {
  float d, du, dv;
};

__device__ __forceinline__ SilSample sil_sample(const float *db, int H, int W, float u, float v) {
  const float x = fminf(fmaxf(u, 0.f), (float)(W - 1)), y = fminf(fmaxf(v, 0.f), (float)(H - 1));
  const int c0 = max(min((int)floorf(x), W - 2), 0), r0 = max(min((int)floorf(y), H - 2), 0);
  const int c1 = min(c0 + 1, W - 1), r1 = min(r0 + 1, H - 1);
  const float fx = x - (float)c0, fy = y - (float)r0;
  const float d00 = db[(size_t)r0 * W + c0], d01 = db[(size_t)r0 * W + c1];
  const float d10 = db[(size_t)r1 * W + c0], d11 = db[(size_t)r1 * W + c1];
  const float top = (1.f - fx) * d00 + fx * d01, bot = (1.f - fx) * d10 + fx * d11;
  SilSample s;
  s.d = (1.f - fy) * top + fy * bot;
  s.du = (u >= 0.f && u <= (float)(W - 1)) ? (1.f - fy) * (d01 - d00) + fy * (d11 - d10) : 0.f;
  s.dv = (v >= 0.f && v <= (float)(H - 1)) ? bot - top : 0.f;
  return s;
}

__global__ void __launch_bounds__(512) sil_forward_kernel(const float *__restrict__ vertices,
                                                          const float *__restrict__ intrinsics,
                                                          const float *__restrict__ dist, int V, int H, int W,
                                                          float *__restrict__ projected,
                                                          float *__restrict__ model_to_mask) {
  __shared__ float red[512];
  const int b = blockIdx.x, t = threadIdx.x;
  const float *intr = intrinsics + 3 * b, *db = dist + (size_t)b * H * W;
  float acc = 0.f;
  for (int i = t; i < V; i += blockDim.x) {
    const SilProj p = sil_project(vertices + ((size_t)b * V + i) * 3, intr);
    float *o = projected + ((size_t)b * V + i) * 3;
    o[0] = p.u;
    o[1] = p.v;
    o[2] = 0.f;
    const float d = sil_sample(db, H, W, p.u, p.v).d;
    acc += d * d;
  }
  red[t] = acc;
  __syncthreads();
  for (int s = 256; s > 0; s >>= 1) {
    if (t < s) red[t] += red[t + s];
    __syncthreads();
  }
  if (t == 0) model_to_mask[b] = red[0] / (float)V;
}

__global__ void __launch_bounds__(256) sil_backward_kernel(const float *__restrict__ vertices,
                                                           const float *__restrict__ intrinsics,
                                                           const float *__restrict__ dist, int B, int V, int H, int W,
                                                           const float *__restrict__ grad_m2m,
                                                           const float *__restrict__ grad_proj,
                                                           float *__restrict__ grad_vertices) {
  const size_t n = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= (size_t)B * V) return;
  const int b = (int)(n / V);
  const float *y = vertices + n * 3, *intr = intrinsics + 3 * b;
  const SilProj p = sil_project(y, intr);
  const SilSample s = sil_sample(dist + (size_t)b * H * W, H, W, p.u, p.v);
  const float g = grad_m2m[b] * (2.f * s.d) / (float)V;
  float gu = g * s.du, gv = g * s.dv;
  if (grad_proj) {
    gu += grad_proj[n * 3];
    gv += grad_proj[n * 3 + 1];
  }
  const float f = intr[0];
  float *o = grad_vertices + n * 3;
  o[0] = gu * f / p.zc;
  o[1] = gv * f / p.zc;
  // u - px = f Y_x / zc: d/dY_z = -(u - px) / zc while Y_z > z_near, 0 where the depth is clamped
  o[2] = y[2] > kSilZNear ? -(gu * (f * (y[0] / p.zc)) + gv * (f * (y[1] / p.zc))) / p.zc : 0.f;
}

__global__ void __launch_bounds__(256) sil_render_kernel(const float *__restrict__ vertices,
                                                         const int32_t *__restrict__ faces,
                                                         const float *__restrict__ intrinsics, int V, int F, int H,
                                                         int W, uint8_t *__restrict__ mask) {
  const int tri = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), b = blockIdx.y, lane = threadIdx.x & 31;
  if (tri >= F) return;
  const int32_t *fc = faces + 3 * tri;
  const float *intr = intrinsics + 3 * b;
  float u[3], v[3];
  for (int k = 0; k < 3; ++k) {
    const int vi = fc[k];
    if (vi < 0 || vi >= V) return;
    const float *y = vertices + ((size_t)b * V + vi) * 3;
    if (!(y[2] > 0.f)) return;
    u[k] = intr[0] * (y[0] / y[2]) + intr[1];
    v[k] = intr[0] * (y[1] / y[2]) + intr[2];
  }
  const float xlo = fmaxf(ceilf(fminf(u[0], fminf(u[1], u[2]))), 0.f);
  const float xhi = fminf(floorf(fmaxf(u[0], fmaxf(u[1], u[2]))), (float)(W - 1));
  const float ylo = fmaxf(ceilf(fminf(v[0], fminf(v[1], v[2]))), 0.f);
  const float yhi = fminf(floorf(fmaxf(v[0], fmaxf(v[1], v[2]))), (float)(H - 1));
  if (!(xlo <= xhi && ylo <= yhi)) return;          // also every NaN
  const int x0 = (int)xlo, y0 = (int)ylo, bw = (int)xhi - x0 + 1, n = bw * ((int)yhi - y0 + 1);
  uint8_t *mb = mask + (size_t)b * H * W;
  for (int i = lane; i < n; i += 32) {
    const int x = x0 + i % bw, yy = y0 + i / bw;
    const float px = (float)x, py = (float)yy;
    const float e0 = (u[1] - u[0]) * (py - v[0]) - (v[1] - v[0]) * (px - u[0]);
    const float e1 = (u[2] - u[1]) * (py - v[1]) - (v[2] - v[1]) * (px - u[1]);
    const float e2 = (u[0] - u[2]) * (py - v[2]) - (v[0] - v[2]) * (px - u[2]);
    if ((e0 >= 0.f && e1 >= 0.f && e2 >= 0.f) || (e0 <= 0.f && e1 <= 0.f && e2 <= 0.f))
      mb[(size_t)yy * W + x] = 1;
  }
}

static int sil_check_image(const char *name, int B, int H, int W) {
  SHAPY_REQUIRE(B >= 0 && H > 0 && W > 0, "%s: bad sizes", name);
  if (H > kSilMaxSide || W > kSilMaxSide) {
    set_error("%s: %d x %d masks exceed the %d x %d supported", name, H, W, kSilMaxSide, kSilMaxSide);
    return SHAPY_ERR_UNSUPPORTED;
  }
  return SHAPY_OK;
}

}  // namespace shapy

using namespace shapy;

extern "C" size_t shapy_silhouette_workspace_bytes(int batch, int height) {
  if (batch <= 0 || height <= 0) return 0;
  return (size_t)batch * height * sizeof(int);
}

extern "C" int shapy_silhouette_prepare(const uint8_t *masks, int batch, int height, int width, int max_points,
                                        float *dist, float *contour, float *contour_w, int32_t *contour_count,
                                        void *workspace, size_t workspace_bytes, void *stream) {
  const char *name = "shapy_silhouette_prepare";
  if (int rc = sil_check_image(name, batch, height, width)) return rc;
  SHAPY_REQUIRE(max_points > 0, "%s: max_points must be > 0", name);
  if (max_points > kSilMaxPoints) {
    set_error("%s: max_points %d exceeds the %d supported", name, max_points, kSilMaxPoints);
    return SHAPY_ERR_UNSUPPORTED;
  }
  if (batch == 0) return SHAPY_OK;
  SHAPY_REQUIRE(masks && dist && contour && contour_w && contour_count && workspace &&
                    workspace_bytes >= shapy_silhouette_workspace_bytes(batch, height),
                "%s: null argument or workspace too small", name);
  cudaStream_t st = (cudaStream_t)stream;
  const int H = height, W = width;
  int *rows = (int *)workspace;
  sil_edt_columns_kernel<<<dim3(ceil_div(W, 128), batch), 128, 0, st>>>(masks, H, W, (int *)dist);
  SHAPY_LAUNCH_CHECK();
  sil_edt_rows_kernel<<<dim3(H, batch), 32, (size_t)W * 8, st>>>(H, W, dist);
  SHAPY_LAUNCH_CHECK();
  sil_contour_count_kernel<<<dim3(H, batch), 128, 0, st>>>(masks, H, W, rows);
  SHAPY_LAUNCH_CHECK();
  sil_contour_scan_kernel<<<batch, 1024, 0, st>>>(H, max_points, rows, contour_count, contour, contour_w);
  SHAPY_LAUNCH_CHECK();
  sil_contour_write_kernel<<<dim3(H, batch), 128, 0, st>>>(masks, H, W, max_points, rows, contour_count, contour,
                                                           contour_w);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

extern "C" int shapy_silhouette_forward(const float *vertices, const float *intrinsics, const float *dist, int batch,
                                        int num_verts, int height, int width, float *projected, float *model_to_mask,
                                        void *stream) {
  const char *name = "shapy_silhouette_forward";
  if (int rc = sil_check_image(name, batch, height, width)) return rc;
  SHAPY_REQUIRE(num_verts > 0, "%s: bad sizes", name);
  if (batch == 0) return SHAPY_OK;
  SHAPY_REQUIRE(vertices && intrinsics && dist && projected && model_to_mask, "%s: null argument", name);
  sil_forward_kernel<<<batch, 512, 0, (cudaStream_t)stream>>>(vertices, intrinsics, dist, num_verts, height, width,
                                                              projected, model_to_mask);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

extern "C" int shapy_silhouette_backward(const float *vertices, const float *intrinsics, const float *dist, int batch,
                                         int num_verts, int height, int width, const float *grad_model_to_mask,
                                         const float *grad_projected, float *grad_vertices, void *stream) {
  const char *name = "shapy_silhouette_backward";
  if (int rc = sil_check_image(name, batch, height, width)) return rc;
  SHAPY_REQUIRE(num_verts > 0, "%s: bad sizes", name);
  if (batch == 0) return SHAPY_OK;
  SHAPY_REQUIRE(vertices && intrinsics && dist && grad_model_to_mask && grad_vertices, "%s: null argument", name);
  const size_t n = (size_t)batch * num_verts;
  sil_backward_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      vertices, intrinsics, dist, batch, num_verts, height, width, grad_model_to_mask, grad_projected, grad_vertices);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

extern "C" int shapy_render_silhouette(const float *vertices, const int32_t *faces, const float *intrinsics, int batch,
                                       int num_verts, int num_faces, int height, int width, uint8_t *mask,
                                       void *stream) {
  const char *name = "shapy_render_silhouette";
  if (int rc = sil_check_image(name, batch, height, width)) return rc;
  SHAPY_REQUIRE(num_verts > 0 && num_faces >= 0, "%s: bad sizes", name);
  if (batch == 0) return SHAPY_OK;
  SHAPY_REQUIRE(vertices && intrinsics && mask && (faces || num_faces == 0), "%s: null argument", name);
  cudaStream_t st = (cudaStream_t)stream;
  SHAPY_CUDA_TRY(cudaMemsetAsync(mask, 0, (size_t)batch * height * width, st));
  if (num_faces == 0) return SHAPY_OK;
  sil_render_kernel<<<dim3(ceil_div(num_faces, 8), batch), 256, 0, st>>>(vertices, faces, intrinsics, num_verts,
                                                                         num_faces, height, width, mask);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}
