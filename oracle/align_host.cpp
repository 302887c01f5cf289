// TEST INFRASTRUCTURE ONLY.  The per-point functions of shapy_b200/csrc/metrics.cuh behind shapy_point_error_aligned and
// shapy_regress_points, compiled for the host from the same source and looped over a batch, for the CPU tests.  The
// per-body statistics are accumulated in double here.  Built by oracle/align_oracle.py:build_align_host.
#define SHAPY_HD inline
#include "../shapy_b200/csrc/metrics.cuh"

// mode 1 = scale, 2 = root (SHAPY_ALIGN_*); roots follow numpy indexing and must be in [-P, P)
extern "C" void align_host(const float *est, const float *gt, int B, int P, int mode, const int *roots, int num_roots,
                           float *error, float *mean) {
  for (int b = 0; b < B; ++b) {
    const float *a = est + (size_t)b * P * 3, *c = gt + (size_t)b * P * 3;
    float ca[3], cc[3], s = 1.f;
    if (mode == 1) {
      double m[6] = {0, 0, 0, 0, 0, 0}, q[2] = {0, 0};
      for (int p = 0; p < P; ++p)
        for (int k = 0; k < 3; ++k) { m[k] += a[p * 3 + k]; m[3 + k] += c[p * 3 + k]; }
      for (int k = 0; k < 6; ++k) m[k] /= P;
      for (int p = 0; p < P; ++p)
        for (int k = 0; k < 3; ++k) {
          const double x = a[p * 3 + k] - m[k], y = c[p * 3 + k] - m[3 + k];
          q[0] += x * x;
          q[1] += y * y;
        }
      for (int k = 0; k < 3; ++k) { ca[k] = (float)m[k]; cc[k] = (float)m[3 + k]; }
      s = (float)sqrt(q[1] / q[0]);
    } else {
      for (int k = 0; k < 3; ++k) {
        double sa = 0, sc = 0;
        for (int r = 0; r < num_roots; ++r) {
          const int i = roots[r] < 0 ? roots[r] + P : roots[r];
          sa += a[i * 3 + k];
          sc += c[i * 3 + k];
        }
        ca[k] = (float)(sa / num_roots);
        cc[k] = (float)(sc / num_roots);
      }
    }
    double m = 0;
    for (int p = 0; p < P; ++p) {
      const float e = mode == 1 ? shapy::scaled_error(a + p * 3, c + p * 3, ca, cc, s) : shapy::root_error(a + p * 3, c + p * 3, ca, cc);
      error[(size_t)b * P + p] = e;
      m += e;
    }
    mean[b] = (float)(m / P);
  }
}

extern "C" void regress_host(const int *row_ptr, const int *col, const float *val, const float *verts, int B, int P, int V,
                             float *points) {
  for (int b = 0; b < B; ++b)
    for (int p = 0; p < P; ++p)
      shapy::csr_row_point(row_ptr, col, val, verts + (size_t)b * V * 3, p, points + ((size_t)b * P + p) * 3);
}
