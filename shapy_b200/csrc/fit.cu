// One Levenberg-Marquardt step of the batched fit of betas to the five virtual measurements (shapy_fit_lm_step).
//
// Per body the residuals are r_k = m_k(beta) - t_k over the terms with weight w_k > 0 and the loss is
// L = sum_k w_k r_k^2 + rho |beta|^2.  The caller evaluates the trial point (shapy_smplx_forward_shape, then
// shapy_measure_jacobian_betas) and this kernel, one warp per body:
//   1. computes the trial loss;
//   2. accepts the trial when it is finite and lower than the state's loss (always on the first step), copying it into
//      the state, and divides lambda by lambda_down, or rejects it and multiplies lambda by lambda_up;
//   3. solves (J^T W J + (rho + lambda) I) delta = -(J^T W r + rho beta) at the state by Cholesky and writes the next
//      trial beta + delta.
// Everything but the final roundings is fp64, the file is compiled with -fmad=false and every sum has a fixed order, so
// oracle/lm_oracle.py restates the decisions exactly.  No host synchronisation, no atomics: a body's trajectory is
// bit-identical from run to run and independent of the rest of the batch.
#include "common.cuh"

namespace shapy {

constexpr int kLmMaxBetas = 16;
constexpr float kLambdaMin = 1e-9f, kLambdaMax = 1e9f;   // lambda is clamped to this range
constexpr double kLambdaInit = 1e-3;                     // first lambda = kLambdaInit * max diag(J^T W J) ...
constexpr double kDiagFloor = 1e-6;                      // ... with that diagonal floored here

struct LmArgs {
  int B, nb;
  const float *targets, *weights;
  float rho, up, down;
  int first;
  float *betas, *meas, *jac, *loss, *lambda;
  int *accepted;
  float *trial;
  const float *trial_meas, *trial_jac;
};

__global__ void __launch_bounds__(128) lm_step_kernel(LmArgs a) {
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
  if (b >= a.B) return;                                    // warp-uniform
  const int nb = a.nb;
  const float *tg = a.targets + (size_t)b * 5, *wt = a.weights + (size_t)b * 5;
  float *beta = a.betas + (size_t)b * nb, *trial = a.trial + (size_t)b * nb;
  float *meas = a.meas + (size_t)b * 5, *jac = a.jac + (size_t)b * 5 * nb;
  const float *tmeas = a.trial_meas + (size_t)b * 5, *tjac = a.trial_jac + (size_t)b * 5 * nb;
  // 1. trial loss: the data terms in k order, then rho times the squares in l order
  const float tb = lane < nb ? trial[lane] : 0.f;
  double data = 0.0, reg = 0.0;
  for (int k = 0; k < 5; ++k) {
    const double w = wt[k];
    if (w > 0.0) {
      const double r = (double)tg[k] - (double)tmeas[k];
      data += w * r * r;
    }
  }
  for (int l = 0; l < nb; ++l) {
    const double x = __shfl_sync(0xffffffffu, tb, l);
    reg += x * x;
  }
  const double lt = data + (double)a.rho * reg;
  // 2. accept or reject
  const float lcur = a.loss[b];
  const bool accept = a.first || (isfinite(lt) && lt < (double)lcur);
  float lam = a.first ? 0.f : a.lambda[b];
  const float *J = accept ? tjac : jac;
  const float *M = accept ? tmeas : meas;
  float bcur = lane < nb ? (accept ? tb : beta[lane]) : 0.f;
  float lnew = lcur;
  if (accept) {
    lnew = isfinite(lt) ? (float)lt : __int_as_float(0x7fc00000);   // a non-finite start reports NaN
    if (lane < nb) beta[lane] = tb;
    if (lane < 5) meas[lane] = tmeas[lane];
    for (int i = lane; i < 5 * nb; i += 32) jac[i] = tjac[i];
    if (lane == 0) a.loss[b] = lnew;
  }
  __syncwarp();
  // 3. normal equations at the state, lane i holding row i: A_ij = sum_k (w_k J_ki) J_kj, g_i = sum_k (w_k J_ki) r_k
  double A[kLmMaxBetas], g = 0.0;
#pragma unroll
  for (int j = 0; j < kLmMaxBetas; ++j) A[j] = 0.0;
  for (int k = 0; k < 5; ++k) {
    const double w = wt[k];
    if (!(w > 0.0)) continue;                            // a dropped term's row is never read: it may be NaN
    const double r = (double)M[k] - (double)tg[k];
    const double wi = lane < nb ? w * (double)J[k * nb + lane] : 0.0;
#pragma unroll
    for (int j = 0; j < kLmMaxBetas; ++j)
      if (j < nb) A[j] += wi * (double)J[k * nb + j];
    g += wi * r;
  }
  g += (double)a.rho * (double)bcur;
  if (a.first) {
    double dmax = kDiagFloor;
#pragma unroll
    for (int j = 0; j < kLmMaxBetas; ++j)
      if (j < nb) dmax = fmax(dmax, __shfl_sync(0xffffffffu, A[j], j));     // lane j's diagonal
    lam = (float)(kLambdaInit * dmax);
  } else if (accept) {
    lam = lam / a.down;
  } else {
    lam = lam * a.up;
  }
  lam = fminf(fmaxf(lam, kLambdaMin), kLambdaMax);
  if (lane == 0) {
    a.lambda[b] = lam;
    if (accept && !a.first) a.accepted[b] += 1;
  }
  const double damp = (double)a.rho + (double)lam;
#pragma unroll
  for (int j = 0; j < kLmMaxBetas; ++j)
    if (j == lane) A[j] += damp;
  // Cholesky A = L L^T, right-looking, lane i keeps row i of L in A[0..i]
  bool ok = isfinite(lnew);                              // a body without a finite loss does not move
#pragma unroll
  for (int j = 0; j < kLmMaxBetas; ++j) {
    if (j < nb) {
      const double d = __shfl_sync(0xffffffffu, A[j], j);
      ok = ok && d > 0.0 && isfinite(d);
      const double ljj = sqrt(d);
      if (lane > j) A[j] /= ljj;
      if (lane == j) A[j] = ljj;
#pragma unroll
      for (int k = j + 1; k < kLmMaxBetas; ++k) {
        if (k < nb) {
          const double lkj = __shfl_sync(0xffffffffu, A[j], k);
          if (lane >= k) A[k] -= A[j] * lkj;
        }
      }
    }
  }
  // L y = -g (column order), then L^T delta = y (column order, from the last)
  double y = -g;
#pragma unroll
  for (int j = 0; j < kLmMaxBetas; ++j) {
    if (j < nb) {
      const double ljj = __shfl_sync(0xffffffffu, A[j], j);
      const double yj = __shfl_sync(0xffffffffu, y, j) / ljj;
      if (lane == j) y = yj;
      if (lane > j) y -= A[j] * yj;
    }
  }
#pragma unroll
  for (int j = kLmMaxBetas - 1; j >= 0; --j) {
    if (j < nb) {
      const double ljj = __shfl_sync(0xffffffffu, A[j], j);
      const double dj = __shfl_sync(0xffffffffu, y, j) / ljj;
      if (lane == j) y = dj;
#pragma unroll
      for (int i = 0; i < kLmMaxBetas; ++i) {
        if (i < j) {
          const double lji = __shfl_sync(0xffffffffu, A[i], j);             // L_ji, row j of lane j
          if (lane == i) y -= lji * dj;
        }
      }
    }
  }
  // ok is warp-uniform (every lane saw the same pivots); a failed factorisation leaves the trial at the state
  if (lane < nb) trial[lane] = ok ? (float)((double)bcur + y) : bcur;
}

// ---------------------------------------------------------------------------------------------------------------
// One Levenberg-Marquardt step of the fit of pose and shape to 3D keypoints (shapy_fit_lm_keypoints_step), one CTA per
// body.  Parameters [delta_j (3 n_rot) | beta (NB) | t (3)], P = 3 n_rot + NB + 3, R_j(delta) = R_j Exp(delta_j); the
// caller evaluates the trial with shapy_smplx_keypoint_jacobian.  The policy is lm_step_kernel's without the betas
// regulariser: L = sum_{w_k > 0} w_k |kp_k - target_k|^2 (fp64, k order), accept a finite trial loss below the state's,
// lambda / down or * up, clamped; then (J^T W J + lambda I) delta = -J^T W (kp - target) by a right-looking Cholesky of
// the P x P normal matrix in fp64 shared memory, and the next trial R_j Exp(delta_j) (Rodrigues in fp64, re-orthonormalised
// by the 6D decoder's Gram-Schmidt of the first two columns), beta + delta_beta, t + delta_t, rounded to fp32.
//
// MEAS (shapy_fit_lm_keypoints_measurements_step) stacks the five virtual measurements and the betas regulariser under
// the keypoint rows: L = L_kp + sum_{w_k > 0} w_k (t_k - m_k)^2 (k order) + rho |beta|^2 (l order), left to right.  The
// measurement Jacobian (5, NB) only has betas columns, so its rows are accumulated after the keypoint rows into the
// betas block of A and g (k order), then rho beta into g; the first lambda comes from diag(A) without rho (as in
// lm_step_kernel) and the betas diagonal gets (double)rho + (double)lambda.  With every measurement weight <= 0 and
// rho = 0 each extra term is skipped or adds an exact 0, so the step equals the keypoint step bit for bit.
constexpr int kLmKpMaxP = 96;
constexpr int kLmKpThreads = 256;
constexpr int kLmKpPairs = (kLmKpMaxP * (kLmKpMaxP + 1) / 2 + kLmKpThreads - 1) / kLmKpThreads;
constexpr int kLmKpRows = 16;           // Jacobian rows staged in shared memory at a time

struct LmKpArgs {
  int K, n_rot, nb, P;
  const float *targets, *weights;
  float up, down;
  int first;
  float *rot, *betas, *transl, *kp, *jac, *loss, *lambda;
  int *accepted;
  float *trot, *tbetas, *ttransl;
  const float *tkp, *tjac;
};

struct LmMeasArgs {                     // the measurement block of the MEAS step (unused otherwise)
  const float *targets, *weights;       // (B, 5): mass, height, chest, waist, hips
  float rho;                            // betas_weight
  float *meas, *jac;                    // state (B, 5), (B, 5, NB)
  const float *tmeas, *tjac;            // the trial's
};

// Phase 4 of the keypoint steps, by the whole CTA: Cholesky A = L L^T of the P x P lower triangle in shared memory,
// right-looking (column j scaled, then the trailing lower triangle updated), then L y = -g and L^T delta = y in place
// in y; thread 0 clears ok_s on a pivot that is not positive and finite
__device__ __forceinline__ void lm_kp_solve(double *A, double *y, int P, int &ok_s) {
  const int t = threadIdx.x;
  for (int j = 0; j < P; ++j) {
    __syncthreads();
    const double d = A[j * P + j];
    const double ljj = sqrt(d);
    __syncthreads();
    if (t == 0) {
      ok_s = ok_s && d > 0.0 && isfinite(d);
      A[j * P + j] = ljj;
    }
    for (int i = j + 1 + t; i < P; i += blockDim.x) A[i * P + j] /= ljj;
    __syncthreads();
    const int n = P - j - 1;
    for (int q = t; q < n * n; q += blockDim.x) {
      const int i = j + 1 + q / n, k = j + 1 + q % n;
      if (k <= i) A[i * P + k] -= A[i * P + j] * A[k * P + j];
    }
  }
  // L y = -g, then L^T delta = y
  for (int j = 0; j < P; ++j) {
    __syncthreads();
    const double yj = y[j] / A[j * P + j];
    __syncthreads();
    if (t == 0) y[j] = yj;
    for (int i = j + 1 + t; i < P; i += blockDim.x) y[i] -= A[i * P + j] * yj;
  }
  for (int j = P - 1; j >= 0; --j) {
    __syncthreads();
    const double dj = y[j] / A[j * P + j];
    __syncthreads();
    if (t == 0) y[j] = dj;
    for (int i = t; i < j; i += blockDim.x) y[i] -= A[j * P + i] * dj;
  }
  __syncthreads();
}

// The next trial rotations of the 2D keypoint step: R_j Exp(delta_j) by Rodrigues in fp64, re-orthonormalised by the 6D
// decoder's Gram-Schmidt of the first two columns and rounded to fp32, or R_j itself when the step failed (!ok).  The
// same operations as phase 5 of lm_kp_step_kernel, which keeps its own copy: inlining this helper there reorders
// its machine code.
__device__ __forceinline__ void lm_kp_next_rot(const float *sr, float *trr, int n_rot, const double *y, bool ok) {
  for (int j = threadIdx.x; j < n_rot; j += blockDim.x) {
    const float *Rs = sr + 9 * j;
    float *Rt = trr + 9 * j;
    if (!ok) {
      for (int e = 0; e < 9; ++e) Rt[e] = Rs[e];
      continue;
    }
    const double d0 = y[3 * j], d1 = y[3 * j + 1], d2 = y[3 * j + 2];
    const double th2 = d0 * d0 + d1 * d1 + d2 * d2, th = sqrt(th2);
    double s, c;                          // Exp(d) = I + s [d]x + c [d]x^2
    if (th < 1e-8) {
      s = 1.0 - th2 / 6.0;
      c = 0.5 - th2 / 24.0;
    } else {
      s = sin(th) / th;
      c = (1.0 - cos(th)) / th2;
    }
    const double dv[3] = {d0, d1, d2};
    const double Kx[9] = {0.0, -d2, d1, d2, 0.0, -d0, -d1, d0, 0.0};
    double E[9], Mr[9];
    for (int r = 0; r < 3; ++r)
      for (int q = 0; q < 3; ++q) E[r * 3 + q] = (r == q ? 1.0 : 0.0) + s * Kx[r * 3 + q] + c * (dv[r] * dv[q] - (r == q ? th2 : 0.0));
    for (int r = 0; r < 3; ++r)
      for (int q = 0; q < 3; ++q)
        Mr[r * 3 + q] = (double)Rs[r * 3] * E[q] + (double)Rs[r * 3 + 1] * E[3 + q] + (double)Rs[r * 3 + 2] * E[6 + q];
    // the 6D decoder's Gram-Schmidt of the first two columns
    const double x0 = Mr[0], x1 = Mr[3], x2 = Mr[6], c0 = Mr[1], c1 = Mr[4], c2 = Mr[7];
    const double n1 = fmax(sqrt(x0 * x0 + x1 * x1 + x2 * x2), 1e-12);
    const double b10 = x0 / n1, b11 = x1 / n1, b12 = x2 / n1;
    const double dd = b10 * c0 + b11 * c1 + b12 * c2;
    const double u0 = c0 - dd * b10, u1 = c1 - dd * b11, u2 = c2 - dd * b12;
    const double n2 = fmax(sqrt(u0 * u0 + u1 * u1 + u2 * u2), 1e-12);
    const double b20 = u0 / n2, b21 = u1 / n2, b22 = u2 / n2;
    const double b30 = b11 * b22 - b12 * b21, b31 = b12 * b20 - b10 * b22, b32 = b10 * b21 - b11 * b20;
    Rt[0] = (float)b10; Rt[1] = (float)b20; Rt[2] = (float)b30;
    Rt[3] = (float)b11; Rt[4] = (float)b21; Rt[5] = (float)b31;
    Rt[6] = (float)b12; Rt[7] = (float)b22; Rt[8] = (float)b32;
  }
}


template <bool MEAS>
__global__ void __launch_bounds__(kLmKpThreads) lm_kp_step_kernel(LmKpArgs a, LmMeasArgs mb) {
  extern __shared__ double A[];         // [P][P]: the lower triangle of J^T W J + lambda I, then its Cholesky factor
  __shared__ double Js[kLmKpRows][kLmKpMaxP], WJs[kLmKpRows][kLmKpMaxP];   // staged rows J_r and w J_r
  __shared__ double rs[kLmKpRows], ws[kLmKpRows], y[kLmKpMaxP];
  __shared__ double lt_s;
  __shared__ int ok_s;
  const int b = blockIdx.x, t = threadIdx.x, P = a.P, K = a.K, R3 = 3 * a.K;
  const float *tg = a.targets + (size_t)b * R3, *wt = a.weights + (size_t)b * K;
  const float lcur = a.loss[b];
  // 1. trial loss
  if (t == 0) {
    const float *m = a.tkp + (size_t)b * R3;
    double L = 0.0;
    for (int k = 0; k < K; ++k) {
      const double w = wt[k];
      if (!(w > 0.0)) continue;
      const double r0 = (double)m[3 * k] - (double)tg[3 * k], r1 = (double)m[3 * k + 1] - (double)tg[3 * k + 1],
                   r2 = (double)m[3 * k + 2] - (double)tg[3 * k + 2];
      L += w * (r0 * r0 + r1 * r1 + r2 * r2);
    }
    if constexpr (MEAS) {
      const float *tm = mb.tmeas + (size_t)b * 5, *mt = mb.targets + (size_t)b * 5, *mw = mb.weights + (size_t)b * 5;
      double Lm = 0.0;
      for (int k = 0; k < 5; ++k) {
        const double w = mw[k];
        if (w > 0.0) {                     // a dropped term is never read: its measurement may be NaN
          const double r = (double)mt[k] - (double)tm[k];
          Lm += w * r * r;
        }
      }
      L += Lm;
      if (mb.rho > 0.f) {
        const float *tb = a.tbetas + (size_t)b * a.nb;
        double reg = 0.0;
        for (int l = 0; l < a.nb; ++l) reg += (double)tb[l] * (double)tb[l];
        L += (double)mb.rho * reg;
      }
    }
    lt_s = L;
  }
  __syncthreads();
  // 2. accept or reject; on accept the trial's parameters, keypoints, Jacobian and loss become the state
  const double lt = lt_s;
  const bool accept = a.first || (isfinite(lt) && lt < (double)lcur);
  const float lnew = accept ? (isfinite(lt) ? (float)lt : __int_as_float(0x7fc00000)) : lcur;
  const float *J = (accept ? a.tjac : a.jac) + (size_t)b * R3 * P;
  const float *M = (accept ? a.tkp : a.kp) + (size_t)b * R3;
  if (accept) {
    const size_t nr = (size_t)a.n_rot * 9;
    for (size_t i = t; i < nr; i += blockDim.x) a.rot[b * nr + i] = a.trot[b * nr + i];
    for (int i = t; i < a.nb; i += blockDim.x) a.betas[(size_t)b * a.nb + i] = a.tbetas[(size_t)b * a.nb + i];
    if (t < 3) a.transl[(size_t)b * 3 + t] = a.ttransl[(size_t)b * 3 + t];
    for (int i = t; i < R3; i += blockDim.x) a.kp[(size_t)b * R3 + i] = M[i];
    for (size_t i = t; i < (size_t)R3 * P; i += blockDim.x) a.jac[(size_t)b * R3 * P + i] = J[i];
    if constexpr (MEAS) {
      for (int i = t; i < 5; i += blockDim.x) mb.meas[(size_t)b * 5 + i] = mb.tmeas[(size_t)b * 5 + i];
      for (int i = t; i < 5 * a.nb; i += blockDim.x) mb.jac[(size_t)b * 5 * a.nb + i] = mb.tjac[(size_t)b * 5 * a.nb + i];
    }
    if (t == 0) a.loss[b] = lnew;
  }
  // 3. normal equations: A_ij = sum_rows (w J_ri) J_rj (i >= j), g_i = sum_rows (w J_ri) (kp_r - target_r), rows in
  // keypoint-major xyz order, the rows of a dropped keypoint never read; thread t owns the lower-triangle entries
  // t + kLmKpThreads i (row-major) and g_t
  const int npairs = P * (P + 1) / 2;
  int pr[kLmKpPairs], pc[kLmKpPairs];
  double acc[kLmKpPairs];
#pragma unroll
  for (int i = 0; i < kLmKpPairs; ++i) {
    const int p = t + kLmKpThreads * i;
    int r = (int)((sqrt(8.0 * p + 1.0) - 1.0) * 0.5);
    while ((r + 1) * (r + 2) / 2 <= p) ++r;
    while (r * (r + 1) / 2 > p) --r;
    pr[i] = p < npairs ? r : -1;
    pc[i] = p - r * (r + 1) / 2;
    acc[i] = 0.0;
  }
  double g = 0.0;
  for (int r0 = 0; r0 < R3; r0 += kLmKpRows) {
    const int nr = min(kLmKpRows, R3 - r0);
    __syncthreads();
    for (int i = t; i < nr; i += blockDim.x) {
      const double w = wt[(r0 + i) / 3];
      ws[i] = w;
      rs[i] = w > 0.0 ? (double)M[r0 + i] - (double)tg[r0 + i] : 0.0;
    }
    for (int i = t; i < nr * P; i += blockDim.x) {
      const int row = i / P;
      const double w = wt[(r0 + row) / 3];
      if (w > 0.0) {
        const double x = J[(size_t)(r0 + row) * P + i % P];
        Js[row][i % P] = x;
        WJs[row][i % P] = w * x;
      }
    }
    __syncthreads();
    for (int row = 0; row < nr; ++row) {
      const double w = ws[row];
      if (!(w > 0.0)) continue;
#pragma unroll
      for (int i = 0; i < kLmKpPairs; ++i)
        if (pr[i] >= 0) acc[i] += WJs[row][pr[i]] * Js[row][pc[i]];
      if (t < P) g += WJs[row][t] * rs[row];
    }
  }
  if constexpr (MEAS) {
    // the five measurement rows, staged like the keypoint rows, into the betas block [o, o + nb) of A and g
    const int o = 3 * a.n_rot, nb = a.nb;
    const float *mt = mb.targets + (size_t)b * 5, *mw = mb.weights + (size_t)b * 5;
    const float *Jm = (accept ? mb.tjac : mb.jac) + (size_t)b * 5 * nb;
    const float *Mm = (accept ? mb.tmeas : mb.meas) + (size_t)b * 5;
    __syncthreads();
    for (int i = t; i < 5; i += blockDim.x) {
      const double w = mw[i];
      ws[i] = w;
      rs[i] = w > 0.0 ? (double)Mm[i] - (double)mt[i] : 0.0;
    }
    for (int i = t; i < 5 * nb; i += blockDim.x) {
      const int row = i / nb;
      const double w = mw[row];
      if (w > 0.0) {                       // a dropped term's row is never read: it may be NaN
        const double x = Jm[i];
        Js[row][i % nb] = x;
        WJs[row][i % nb] = w * x;
      }
    }
    __syncthreads();
    for (int row = 0; row < 5; ++row) {
      if (!(ws[row] > 0.0)) continue;
#pragma unroll
      for (int i = 0; i < kLmKpPairs; ++i)
        if (pc[i] >= o && pr[i] >= 0 && pr[i] < o + nb) acc[i] += WJs[row][pr[i] - o] * Js[row][pc[i] - o];
      if (t >= o && t < o + nb) g += WJs[row][t - o] * rs[row];
    }
    if (mb.rho > 0.f && t >= o && t < o + nb)
      g += (double)mb.rho * (double)(accept ? a.tbetas : a.betas)[(size_t)b * nb + t - o];
  }
#pragma unroll
  for (int i = 0; i < kLmKpPairs; ++i)
    if (pr[i] >= 0) A[pr[i] * P + pc[i]] = acc[i];
  if (t < P) y[t] = -g;
  __syncthreads();
  if (t == 0) {
    float lam = a.first ? 0.f : a.lambda[b];
    if (a.first) {
      double dmax = kDiagFloor;
      for (int j = 0; j < P; ++j) dmax = fmax(dmax, A[j * P + j]);
      lam = (float)(kLambdaInit * dmax);
    } else if (accept) {
      lam = lam / a.down;
    } else {
      lam = lam * a.up;
    }
    lam = fminf(fmaxf(lam, kLambdaMin), kLambdaMax);
    a.lambda[b] = lam;
    if (accept && !a.first) a.accepted[b] += 1;
    if constexpr (MEAS) {
      const int o = 3 * a.n_rot;
      const double damp = (double)mb.rho + (double)lam;
      for (int j = 0; j < P; ++j) A[j * P + j] += j >= o && j < o + a.nb ? damp : (double)lam;
    } else {
      for (int j = 0; j < P; ++j) A[j * P + j] += (double)lam;
    }
    ok_s = isfinite(lnew);               // a body without a finite loss does not move
  }
  lm_kp_solve(A, y, P, ok_s);
  // 5. next trial (ok is uniform: every thread reads it after the last barrier); a failed step keeps the state
  const bool ok = ok_s;
  const float *sr = a.rot + (size_t)b * a.n_rot * 9;
  float *trr = a.trot + (size_t)b * a.n_rot * 9;
  for (int j = t; j < a.n_rot; j += blockDim.x) {
    const float *Rs = sr + 9 * j;
    float *Rt = trr + 9 * j;
    if (!ok) {
      for (int e = 0; e < 9; ++e) Rt[e] = Rs[e];
      continue;
    }
    const double d0 = y[3 * j], d1 = y[3 * j + 1], d2 = y[3 * j + 2];
    const double th2 = d0 * d0 + d1 * d1 + d2 * d2, th = sqrt(th2);
    double s, c;                          // Exp(d) = I + s [d]x + c [d]x^2
    if (th < 1e-8) {
      s = 1.0 - th2 / 6.0;
      c = 0.5 - th2 / 24.0;
    } else {
      s = sin(th) / th;
      c = (1.0 - cos(th)) / th2;
    }
    const double dv[3] = {d0, d1, d2};
    const double Kx[9] = {0.0, -d2, d1, d2, 0.0, -d0, -d1, d0, 0.0};
    double E[9], Mr[9];
    for (int r = 0; r < 3; ++r)
      for (int q = 0; q < 3; ++q) E[r * 3 + q] = (r == q ? 1.0 : 0.0) + s * Kx[r * 3 + q] + c * (dv[r] * dv[q] - (r == q ? th2 : 0.0));
    for (int r = 0; r < 3; ++r)
      for (int q = 0; q < 3; ++q)
        Mr[r * 3 + q] = (double)Rs[r * 3] * E[q] + (double)Rs[r * 3 + 1] * E[3 + q] + (double)Rs[r * 3 + 2] * E[6 + q];
    // the 6D decoder's Gram-Schmidt of the first two columns
    const double x0 = Mr[0], x1 = Mr[3], x2 = Mr[6], c0 = Mr[1], c1 = Mr[4], c2 = Mr[7];
    const double n1 = fmax(sqrt(x0 * x0 + x1 * x1 + x2 * x2), 1e-12);
    const double b10 = x0 / n1, b11 = x1 / n1, b12 = x2 / n1;
    const double dd = b10 * c0 + b11 * c1 + b12 * c2;
    const double u0 = c0 - dd * b10, u1 = c1 - dd * b11, u2 = c2 - dd * b12;
    const double n2 = fmax(sqrt(u0 * u0 + u1 * u1 + u2 * u2), 1e-12);
    const double b20 = u0 / n2, b21 = u1 / n2, b22 = u2 / n2;
    const double b30 = b11 * b22 - b12 * b21, b31 = b12 * b20 - b10 * b22, b32 = b10 * b21 - b11 * b20;
    Rt[0] = (float)b10; Rt[1] = (float)b20; Rt[2] = (float)b30;
    Rt[3] = (float)b11; Rt[4] = (float)b21; Rt[5] = (float)b31;
    Rt[6] = (float)b12; Rt[7] = (float)b22; Rt[8] = (float)b32;
  }
  const int o = 3 * a.n_rot;
  for (int l = t; l < a.nb; l += blockDim.x) {
    const float x = a.betas[(size_t)b * a.nb + l];
    a.tbetas[(size_t)b * a.nb + l] = ok ? (float)((double)x + y[o + l]) : x;
  }
  if (t < 3) {
    const float x = a.transl[(size_t)b * 3 + t];
    a.ttransl[(size_t)b * 3 + t] = ok ? (float)((double)x + y[o + a.nb + t]) : x;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// One Levenberg-Marquardt step of the fit of pose, shape and weak-perspective camera to 2D keypoints
// (shapy_fit_lm_keypoints_2d_step), one CTA per body, with lm_kp_step_kernel's policy, solve and rotation update.
// Parameters [delta_j (3 n_rot) | beta (NB) | c0, c1, c2], P = 3 n_rot + NB + 3: the camera takes the columns of transl
// (which a weak-perspective camera cannot see along z, and which duplicates c1, c2 in x and y).  With s = softplus(c0)
// (threshold 20, as the forward) the projection is p_k = s (kp_k,xy + (c1, c2)), and per body, in fp64, left to right:
//   L = sum_{w_k > 0} w_k rho(|p_k - x_k|^2)  (k order)
//     + 1/2 pose_w sum_{j >= 1} |R_j - R0_j|_F^2  (j order, row-major entries; when pose_w > 0)
//     + betas_w |beta|^2  (l order; when betas_w > 0)
// rho(e) = e at sigma = inf, else e q with q = sigma^2 / (sigma^2 + e) (Geman-McClure).  Rows of the normal equations,
// accumulated into A and g in this order:
//   keypoint rows 2k + c (c = 0 x, 1 y), weight w_k q_k^2 (the IRLS weight rho'(e_k), 1 at sigma = inf) at the state,
//     residual p_kc - x_kc, Jacobian staged from the 3D keypoint Jacobian (transl columns skipped): s J_{3k+c} on the
//     rotation and betas columns, ds/dc0 (kp_kc + c_{1+c}) on c0, s on c_{1+c};
//   pose-prior rows (R_j - R0_j)_e, weight pose_w / 2, Jacobian R_j [e_a]x in column 3 j + a (d(R Exp d) = R [d]x),
//     j = 1 .. n_rot - 1, e in row-major order: they only reach the 3 x 3 diagonal block of joint j;
//   then g += betas_w beta on the betas columns.
// The first lambda is 1e-3 max(diag A, 1e-6) of the keypoint rows alone; the diagonal then gets betas_w + lambda on the
// betas columns and lambda elsewhere.  The next trial is R_j Exp(delta_j), beta + delta_beta, c + delta_c.
struct LmKp2dArgs {
  int K, n_rot, nb, P;
  const float *targets, *weights, *anchor;    // (B, K, 2), (B, K), (B, n_rot, 3, 3)
  float sigma, pose_w, betas_w, up, down;
  int first;
  float *rot, *betas, *camera, *kp, *jac, *loss, *lambda;
  int *accepted;
  float *trot, *tbetas, *tcamera;
  const float *tkp, *tjac;
};

// softplus(c0) and its derivative, with F.softplus' threshold of 20 (smplx.cu's projection)
__device__ __forceinline__ void softplus_d(double c0, double &s, double &ds) {
  if (c0 > 20.0) {
    s = c0;
    ds = 1.0;
  } else {
    s = log1p(exp(c0));
    ds = 1.0 / (1.0 + exp(-c0));
  }
}

// (R [e_a]x)_e, e = 3 r + q: the columns of R [e_0]x are (0, R_2, -R_1), of R [e_1]x (-R_2, 0, R_0), of R [e_2]x
// (R_1, -R_0, 0)
__device__ __forceinline__ double rot_tangent(const float *R, int a, int e) {
  const int r = e / 3, q = e % 3;
  if (q == a) return 0.0;
  const int m = 3 - a - q;                     // the third index
  const double v = (double)R[r * 3 + m];
  return ((q - a + 3) % 3 == 1) ? v : -v;      // -eps_{a m q} R_rm
}

__global__ void __launch_bounds__(kLmKpThreads, 2) lm_kp2d_step_kernel(LmKp2dArgs a) {
  extern __shared__ double A[];         // [P][P]: the lower triangle of the normal matrix, then its Cholesky factor
  __shared__ double Js[kLmKpRows][kLmKpMaxP], WJs[kLmKpRows][kLmKpMaxP];   // staged rows J_r and w J_r
  __shared__ double rs[kLmKpRows], ws[kLmKpRows], y[kLmKpMaxP], dg[kLmKpMaxP];
  __shared__ double lt_s;
  __shared__ int ok_s;
  const int b = blockIdx.x, t = threadIdx.x, P = a.P, K = a.K, R3 = 3 * a.K, nb = a.nb, nr9 = 9 * a.n_rot;
  const int o = 3 * a.n_rot, oc = o + nb;     // first betas and first camera column
  const float *tg = a.targets + (size_t)b * 2 * K, *wt = a.weights + (size_t)b * K;
  const float *anc = a.anchor ? a.anchor + (size_t)b * nr9 : nullptr;
  const bool robust = isfinite(a.sigma);
  const double s2 = (double)a.sigma * (double)a.sigma;
  const float lcur = a.loss[b];
  // 1. trial loss
  if (t == 0) {
    const float *m = a.tkp + (size_t)b * R3, *cam = a.tcamera + (size_t)b * 3;
    double s, ds;
    softplus_d((double)cam[0], s, ds);
    const double cx = cam[1], cy = cam[2];
    double L = 0.0;
    for (int k = 0; k < K; ++k) {
      const double w = wt[k];
      if (!(w > 0.0)) continue;
      const double dx = s * ((double)m[3 * k] + cx) - (double)tg[2 * k];
      const double dy = s * ((double)m[3 * k + 1] + cy) - (double)tg[2 * k + 1];
      const double e = dx * dx + dy * dy;
      L += w * (robust ? e * (s2 / (s2 + e)) : e);
    }
    if (a.pose_w > 0.f) {
      const float *tr = a.trot + (size_t)b * nr9;
      double q = 0.0;
      for (int i = 9; i < nr9; ++i) {
        const double d = (double)tr[i] - (double)anc[i];
        q += d * d;
      }
      L += 0.5 * (double)a.pose_w * q;
    }
    if (a.betas_w > 0.f) {
      const float *tb = a.tbetas + (size_t)b * nb;
      double reg = 0.0;
      for (int l = 0; l < nb; ++l) reg += (double)tb[l] * (double)tb[l];
      L += (double)a.betas_w * reg;
    }
    lt_s = L;
  }
  __syncthreads();
  // 2. accept or reject; on accept the trial's parameters, keypoints, Jacobian and loss become the state
  const double lt = lt_s;
  const bool accept = a.first || (isfinite(lt) && lt < (double)lcur);
  const float lnew = accept ? (isfinite(lt) ? (float)lt : __int_as_float(0x7fc00000)) : lcur;
  const float *J = (accept ? a.tjac : a.jac) + (size_t)b * R3 * P;
  const float *M = (accept ? a.tkp : a.kp) + (size_t)b * R3;
  const float *Rst = (accept ? a.trot : a.rot) + (size_t)b * nr9;
  const float *Bst = (accept ? a.tbetas : a.betas) + (size_t)b * nb;
  const float *Cst = (accept ? a.tcamera : a.camera) + (size_t)b * 3;
  if (accept) {
    for (int i = t; i < nr9; i += blockDim.x) a.rot[(size_t)b * nr9 + i] = a.trot[(size_t)b * nr9 + i];
    for (int i = t; i < nb; i += blockDim.x) a.betas[(size_t)b * nb + i] = a.tbetas[(size_t)b * nb + i];
    if (t < 3) a.camera[(size_t)b * 3 + t] = a.tcamera[(size_t)b * 3 + t];
    for (int i = t; i < R3; i += blockDim.x) a.kp[(size_t)b * R3 + i] = M[i];
    for (size_t i = t; i < (size_t)R3 * P; i += blockDim.x) a.jac[(size_t)b * R3 * P + i] = J[i];
    if (t == 0) a.loss[b] = lnew;
  }
  double s, ds;
  softplus_d((double)Cst[0], s, ds);
  const double cxy[2] = {(double)Cst[1], (double)Cst[2]};
  // 3. normal equations, thread t owning the lower-triangle entries t + kLmKpThreads i (row-major) and g_t
  const int npairs = P * (P + 1) / 2;
  int pr[kLmKpPairs], pc[kLmKpPairs];
  double acc[kLmKpPairs];
#pragma unroll
  for (int i = 0; i < kLmKpPairs; ++i) {
    const int p = t + kLmKpThreads * i;
    int r = (int)((sqrt(8.0 * p + 1.0) - 1.0) * 0.5);
    while ((r + 1) * (r + 2) / 2 <= p) ++r;
    while (r * (r + 1) / 2 > p) --r;
    pr[i] = p < npairs ? r : -1;
    pc[i] = p - r * (r + 1) / 2;
    acc[i] = 0.0;
  }
  double g = 0.0;
  const int R2 = 2 * K;
  for (int r0 = 0; r0 < R2; r0 += kLmKpRows) {
    const int nr = min(kLmKpRows, R2 - r0);
    __syncthreads();
    for (int i = t; i < nr; i += blockDim.x) {   // row weight (IRLS at the state) and residual
      const int k = (r0 + i) >> 1, c = (r0 + i) & 1;
      const double w = wt[k];
      double wr = w, res = 0.0;
      if (w > 0.0) {
        const double dx = s * ((double)M[3 * k] + cxy[0]) - (double)tg[2 * k];
        const double dy = s * ((double)M[3 * k + 1] + cxy[1]) - (double)tg[2 * k + 1];
        if (robust) {
          const double q = s2 / (s2 + (dx * dx + dy * dy));
          wr = w * (q * q);
        }
        res = c ? dy : dx;
      }
      ws[i] = wr;
      rs[i] = res;
    }
    __syncthreads();
    for (int i = t; i < nr * P; i += blockDim.x) {
      const int row = i / P, col = i % P;
      const double wr = ws[row];
      if (wr > 0.0) {                    // a dropped keypoint's rows are never read: they may be NaN
        const int k = (r0 + row) >> 1, c = (r0 + row) & 1;
        double x;
        if (col < oc) x = s * (double)J[(size_t)(3 * k + c) * P + col];
        else if (col == oc) x = ds * ((double)M[3 * k + c] + cxy[c]);
        else x = col - oc - 1 == c ? s : 0.0;
        Js[row][col] = x;
        WJs[row][col] = wr * x;
      }
    }
    __syncthreads();
    for (int row = 0; row < nr; ++row) {
      const double w = ws[row];
      if (!(w > 0.0)) continue;
#pragma unroll
      for (int i = 0; i < kLmKpPairs; ++i)
        if (pr[i] >= 0) acc[i] += WJs[row][pr[i]] * Js[row][pc[i]];
      if (t < P) g += WJs[row][t] * rs[row];
    }
  }
#pragma unroll
  for (int i = 0; i < kLmKpPairs; ++i)
    if (pr[i] >= 0 && pr[i] == pc[i]) dg[pr[i]] = acc[i];     // the diagonal of the keypoint rows: the first lambda
  if (a.pose_w > 0.f) {
    // the pose-prior rows of joint j only reach its diagonal block: no staging
    const double hw = 0.5 * (double)a.pose_w;
#pragma unroll
    for (int i = 0; i < kLmKpPairs; ++i) {
      const int j = pr[i] / 3;
      if (pr[i] >= 3 && pr[i] < o && pc[i] / 3 == j) {
        const float *R = Rst + 9 * j;
        for (int e = 0; e < 9; ++e) acc[i] += (hw * rot_tangent(R, pr[i] % 3, e)) * rot_tangent(R, pc[i] % 3, e);
      }
    }
    if (t >= 3 && t < o) {
      const float *R = Rst + 9 * (t / 3), *R0 = anc + 9 * (t / 3);
      for (int e = 0; e < 9; ++e) g += (hw * rot_tangent(R, t % 3, e)) * ((double)R[e] - (double)R0[e]);
    }
  }
  if (a.betas_w > 0.f && t >= o && t < oc) g += (double)a.betas_w * (double)Bst[t - o];
#pragma unroll
  for (int i = 0; i < kLmKpPairs; ++i)
    if (pr[i] >= 0) A[pr[i] * P + pc[i]] = acc[i];
  if (t < P) y[t] = -g;
  __syncthreads();
  if (t == 0) {
    float lam = a.first ? 0.f : a.lambda[b];
    if (a.first) {
      double dmax = kDiagFloor;
      for (int j = 0; j < P; ++j) dmax = fmax(dmax, dg[j]);
      lam = (float)(kLambdaInit * dmax);
    } else if (accept) {
      lam = lam / a.down;
    } else {
      lam = lam * a.up;
    }
    lam = fminf(fmaxf(lam, kLambdaMin), kLambdaMax);
    a.lambda[b] = lam;
    if (accept && !a.first) a.accepted[b] += 1;
    const double damp = (double)a.betas_w + (double)lam;
    for (int j = 0; j < P; ++j) A[j * P + j] += j >= o && j < oc ? damp : (double)lam;
    ok_s = isfinite(lnew);               // a body without a finite loss does not move
  }
  // 4. Cholesky and the two triangular solves
  lm_kp_solve(A, y, P, ok_s);
  // 5. next trial (ok is uniform: every thread reads it after the last barrier); a failed step keeps the state
  const bool ok = ok_s;
  lm_kp_next_rot(a.rot + (size_t)b * nr9, a.trot + (size_t)b * nr9, a.n_rot, y, ok);
  for (int l = t; l < nb; l += blockDim.x) {
    const float x = a.betas[(size_t)b * nb + l];
    a.tbetas[(size_t)b * nb + l] = ok ? (float)((double)x + y[o + l]) : x;
  }
  if (t < 3) {
    const float x = a.camera[(size_t)b * 3 + t];
    a.tcamera[(size_t)b * 3 + t] = ok ? (float)((double)x + y[oc + t]) : x;
  }
}

// One CTA of kLmKpThreads per body with P x P doubles of dynamic shared memory; past 48 KB of static plus dynamic
// shared memory the launch has to opt in
template <typename... Args>
int launch_lm_kp(void (*kernel)(Args...), int batch, int P, void *stream, Args... args) {
  const size_t smem = (size_t)P * P * sizeof(double);
  cudaFuncAttributes attr;
  SHAPY_CUDA_TRY(cudaFuncGetAttributes(&attr, kernel));
  if (smem + attr.sharedSizeBytes > 48 * 1024)
    SHAPY_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kernel<<<batch, kLmKpThreads, smem, (cudaStream_t)stream>>>(args...);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

}  // namespace shapy

using namespace shapy;

extern "C" int shapy_fit_lm_step(int batch, int nb, const float *targets, const float *weights, float betas_weight,
                                 float lambda_up, float lambda_down, int first, float *betas, float *meas, float *jac,
                                 float *loss, float *lambda, int32_t *accepted, float *trial, const float *trial_meas,
                                 const float *trial_jac, void *stream) {
  SHAPY_REQUIRE(targets && weights && betas && meas && jac && loss && lambda && accepted && trial && trial_meas &&
                    trial_jac && batch > 0,
                "shapy_fit_lm_step: bad argument");
  SHAPY_REQUIRE(lambda_up >= 1.f && lambda_down >= 1.f && betas_weight >= 0.f,
                "shapy_fit_lm_step: lambda_up and lambda_down must be >= 1 and betas_weight >= 0");
  if (nb < 1 || nb > kLmMaxBetas) {
    set_error("shapy_fit_lm_step: %d betas, at most %d are supported", nb, kLmMaxBetas);
    return SHAPY_ERR_UNSUPPORTED;
  }
  LmArgs a{batch, nb, targets, weights, betas_weight, lambda_up, lambda_down, first ? 1 : 0, betas, meas, jac, loss,
           lambda, accepted, trial, trial_meas, trial_jac};
  lm_step_kernel<<<ceil_div(batch, 4), 128, 0, (cudaStream_t)stream>>>(a);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

extern "C" int shapy_fit_lm_keypoints_step(int batch, int num_keypoints, int n_rot, int nb, const float *targets,
                                           const float *weights, float lambda_up, float lambda_down, int first,
                                           float *rot, float *betas, float *transl, float *keypoints, float *jac,
                                           float *loss, float *lambda, int32_t *accepted, float *trial_rot,
                                           float *trial_betas, float *trial_transl, const float *trial_keypoints,
                                           const float *trial_jac, void *stream) {
  SHAPY_REQUIRE(targets && weights && rot && betas && transl && keypoints && jac && loss && lambda && accepted &&
                    trial_rot && trial_betas && trial_transl && trial_keypoints && trial_jac,
                "shapy_fit_lm_keypoints_step: null argument");
  SHAPY_REQUIRE(batch >= 0 && num_keypoints >= 1 && n_rot >= 1 && n_rot <= 64 && nb >= 1,
                "shapy_fit_lm_keypoints_step: bad size (batch %d, %d keypoints, n_rot %d, %d betas)", batch,
                num_keypoints, n_rot, nb);
  SHAPY_REQUIRE(lambda_up >= 1.f && lambda_down >= 1.f,
                "shapy_fit_lm_keypoints_step: lambda_up and lambda_down must be >= 1");
  const int P = 3 * n_rot + nb + 3;
  if (P > kLmKpMaxP) {
    set_error("shapy_fit_lm_keypoints_step: %d parameters, at most %d are supported", P, kLmKpMaxP);
    return SHAPY_ERR_UNSUPPORTED;
  }
  if (batch == 0) return SHAPY_OK;
  LmKpArgs a{num_keypoints, n_rot, nb, P, targets, weights, lambda_up, lambda_down, first ? 1 : 0, rot, betas, transl,
             keypoints, jac, loss, lambda, accepted, trial_rot, trial_betas, trial_transl, trial_keypoints, trial_jac};
  return launch_lm_kp(lm_kp_step_kernel<false>, batch, P, stream, a, LmMeasArgs{});
}

extern "C" int shapy_fit_lm_keypoints_measurements_step(
    int batch, int num_keypoints, int n_rot, int nb, const float *targets, const float *weights,
    const float *meas_targets, const float *meas_weights, float betas_weight, float lambda_up, float lambda_down,
    int first, float *rot, float *betas, float *transl, float *keypoints, float *jac, float *meas, float *meas_jac,
    float *loss, float *lambda, int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_transl,
    const float *trial_keypoints, const float *trial_jac, const float *trial_meas, const float *trial_meas_jac,
    void *stream) {
  SHAPY_REQUIRE(targets && weights && meas_targets && meas_weights && rot && betas && transl && keypoints && jac &&
                    meas && meas_jac && loss && lambda && accepted && trial_rot && trial_betas && trial_transl &&
                    trial_keypoints && trial_jac && trial_meas && trial_meas_jac,
                "shapy_fit_lm_keypoints_measurements_step: null argument");
  SHAPY_REQUIRE(batch >= 0 && num_keypoints >= 1 && n_rot >= 1 && n_rot <= 64 && nb >= 1,
                "shapy_fit_lm_keypoints_measurements_step: bad size (batch %d, %d keypoints, n_rot %d, %d betas)",
                batch, num_keypoints, n_rot, nb);
  SHAPY_REQUIRE(lambda_up >= 1.f && lambda_down >= 1.f && betas_weight >= 0.f,
                "shapy_fit_lm_keypoints_measurements_step: lambda_up and lambda_down must be >= 1 and betas_weight "
                ">= 0");
  const int P = 3 * n_rot + nb + 3;
  if (P > kLmKpMaxP) {
    set_error("shapy_fit_lm_keypoints_measurements_step: %d parameters, at most %d are supported", P, kLmKpMaxP);
    return SHAPY_ERR_UNSUPPORTED;
  }
  if (batch == 0) return SHAPY_OK;
  LmKpArgs a{num_keypoints, n_rot, nb, P, targets, weights, lambda_up, lambda_down, first ? 1 : 0, rot, betas, transl,
             keypoints, jac, loss, lambda, accepted, trial_rot, trial_betas, trial_transl, trial_keypoints, trial_jac};
  LmMeasArgs m{meas_targets, meas_weights, betas_weight, meas, meas_jac, trial_meas, trial_meas_jac};
  return launch_lm_kp(lm_kp_step_kernel<true>, batch, P, stream, a, m);
}

extern "C" int shapy_fit_lm_keypoints_2d_step(int batch, int num_keypoints, int n_rot, int nb, const float *targets,
                                              const float *weights, const float *pose_anchor, float robust_sigma,
                                              float pose_prior_weight, float betas_weight, float lambda_up,
                                              float lambda_down, int first, float *rot, float *betas, float *camera,
                                              float *keypoints, float *jac, float *loss, float *lambda,
                                              int32_t *accepted, float *trial_rot, float *trial_betas,
                                              float *trial_camera, const float *trial_keypoints, const float *trial_jac,
                                              void *stream) {
  SHAPY_REQUIRE(targets && weights && rot && betas && camera && keypoints && jac && loss && lambda && accepted &&
                    trial_rot && trial_betas && trial_camera && trial_keypoints && trial_jac &&
                    (pose_anchor || !(pose_prior_weight > 0.f)),
                "shapy_fit_lm_keypoints_2d_step: null argument");
  SHAPY_REQUIRE(batch >= 0 && num_keypoints >= 1 && n_rot >= 1 && n_rot <= 64 && nb >= 1,
                "shapy_fit_lm_keypoints_2d_step: bad size (batch %d, %d keypoints, n_rot %d, %d betas)", batch,
                num_keypoints, n_rot, nb);
  SHAPY_REQUIRE(robust_sigma > 0.f && pose_prior_weight >= 0.f && betas_weight >= 0.f && lambda_up >= 1.f &&
                    lambda_down >= 1.f,
                "shapy_fit_lm_keypoints_2d_step: robust_sigma must be > 0 (inf: least squares), the prior weights >= 0 "
                "and lambda_up and lambda_down >= 1");
  const int P = 3 * n_rot + nb + 3;
  if (P > kLmKpMaxP) {
    set_error("shapy_fit_lm_keypoints_2d_step: %d parameters, at most %d are supported", P, kLmKpMaxP);
    return SHAPY_ERR_UNSUPPORTED;
  }
  if (batch == 0) return SHAPY_OK;
  LmKp2dArgs a{num_keypoints, n_rot, nb, P, targets, weights, pose_anchor, robust_sigma, pose_prior_weight,
               betas_weight, lambda_up, lambda_down, first ? 1 : 0, rot, betas, camera, keypoints, jac, loss, lambda,
               accepted, trial_rot, trial_betas, trial_camera, trial_keypoints, trial_jac};
  return launch_lm_kp(lm_kp2d_step_kernel, batch, P, stream, a);
}
