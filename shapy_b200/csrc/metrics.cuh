// P2P-20k / v2v-HD evaluation metric arithmetic (SURVEY.md 8f rank 3), shared by the CUDA kernels (metrics.cu) and the
// host-compiled copy the tests build from the same source (oracle/metrics_host.cpp).
//
// Reference: regressor/human_shape/utils/metrics.py:368-456 (v2vhdError): HD points = sparse (P x V) point regressor times
// the vertices of each mesh; t = mean_p(target points) - mean_p(input points) when align; error_p = |input_p + t - target_p|;
// returns (error.mean(1), error).  Also regressor/hbw_evaluation/evaluate_hbw.py:44-58,147-151 (same with numpy).
// Scale / root alignments of PointError (metrics.py:173-229, 279-303, 335-366): the per-point errors after the per-body
// statistics of shapy_point_error_aligned.
#pragma once
#include <stddef.h>
#include <math.h>

#ifndef SHAPY_HD
#define SHAPY_HD __host__ __device__ __forceinline__
#endif

namespace shapy {

// row p of a CSR matrix (row_ptr, col, val) times the (V, 3) vertex array: one regressed point
SHAPY_HD void csr_row_point(const int *row_ptr, const int *col, const float *val, const float *verts, int p, float *out) {
  float x = 0.f, y = 0.f, z = 0.f;
  for (int k = row_ptr[p]; k < row_ptr[p + 1]; ++k) {
    const float w = val[k];
    const float *v = verts + (size_t)col[k] * 3;
    x += w * v[0];
    y += w * v[1];
    z += w * v[2];
  }
  out[0] = x; out[1] = y; out[2] = z;
}

// |d + t| for the un-aligned difference d = input point - target point
SHAPY_HD float aligned_error(const float *d, const float *t) {
  const float x = d[0] + t[0], y = d[1] + t[1], z = d[2] + t[2];
  return sqrtf(x * x + y * y + z * z);
}

// ScaleAlignment + point_error (metrics.py:173-229, 31-52): est' = s est + t with t = mu2 - s mu1, error = |est' - gt|.
// Evaluated as |s (a - mu1) - (c - mu2)|, the same value regrouped so that the metre-sized coordinates of an evaluation
// mesh cancel before the product instead of after it.
SHAPY_HD float scaled_error(const float *a, const float *c, const float *mu1, const float *mu2, float s) {
  const float x = s * (a[0] - mu1[0]) - (c[0] - mu2[0]);
  const float y = s * (a[1] - mu1[1]) - (c[1] - mu2[1]);
  const float z = s * (a[2] - mu1[2]) - (c[2] - mu2[2]);
  return sqrtf(x * x + y * y + z * z);
}

// RootAlignment + point_error (metrics.py:279-303): |(est - r_est) - (gt - r_gt)|, in the reference's order
SHAPY_HD float root_error(const float *a, const float *c, const float *ra, const float *rc) {
  const float x = (a[0] - ra[0]) - (c[0] - rc[0]);
  const float y = (a[1] - ra[1]) - (c[1] - rc[1]);
  const float z = (a[2] - ra[2]) - (c[2] - rc[2]);
  return sqrtf(x * x + y * y + z * z);
}

}  // namespace shapy
