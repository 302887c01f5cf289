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
#include <type_traits>

#include "common.cuh"
#include "penetration.cuh"

namespace shapy {

constexpr int kLmMaxBetas = 16;
constexpr float kLambdaMin = 1e-9f, kLambdaMax = 1e9f;   // lambda is clamped to this range
constexpr double kLambdaInit = 1e-3;                     // first lambda = kLambdaInit * max diag(J^T W J) ...
constexpr double kDiagFloor = 1e-6;                      // ... with that diagonal floored here

// The policy of every step kernel of this file.  The trial is accepted on the first step, and afterwards when its loss
// is finite and below the state's
__device__ __forceinline__ bool lm_accept(int first, double lt, float lcur) {
  const bool better = isfinite(lt) && lt < (double)lcur;   // evaluated either way: `first || (...)` in one expression
  return first || better;                                  // costs lm_step_kernel eight registers
}

// The state's loss after that decision; a non-finite start reports NaN
__device__ __forceinline__ float lm_loss(bool accept, double lt, float lcur) {
  return accept ? (isfinite(lt) ? (float)lt : __int_as_float(0x7fc00000)) : lcur;
}

// The damping: on the first step from dmax, the largest diagonal entry of the undamped normal matrix floored at
// kDiagFloor; afterwards the previous lambda over `down` after an accepted trial, times `up` after a rejected one
__device__ __forceinline__ float lm_lambda(int first, bool accept, float lam, double dmax, float up, float down) {
  if (first) {
    lam = (float)(kLambdaInit * dmax);
  } else if (accept) {
    lam = lam / down;
  } else {
    lam = lam * up;
  }
  return fminf(fmaxf(lam, kLambdaMin), kLambdaMax);
}

// |x|^2 of n fp32 values in fp64, in l order: the sum of every betas and expression regulariser
__device__ __forceinline__ double lm_sq_norm(const float *x, int n) {
  double s = 0.0;
  for (int l = 0; l < n; ++l) s += (double)x[l] * (double)x[l];
  return s;
}

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
  const bool accept = lm_accept(a.first, lt, lcur);
  const float lnew = lm_loss(accept, lt, lcur);
  float lam = a.first ? 0.f : a.lambda[b];
  const float *J = accept ? tjac : jac;
  const float *M = accept ? tmeas : meas;
  float bcur = lane < nb ? (accept ? tb : beta[lane]) : 0.f;
  if (accept) {
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
  double dmax = kDiagFloor;
  if (a.first) {
#pragma unroll
    for (int j = 0; j < kLmMaxBetas; ++j)
      if (j < nb) dmax = fmax(dmax, __shfl_sync(0xffffffffu, A[j], j));     // lane j's diagonal
  }
  lam = lm_lambda(a.first, accept, lam, dmax, a.up, a.down);
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
// The Levenberg-Marquardt steps of the keypoint fits: pose and shape with a translation against 3D keypoints
// (lm_kp_step_kernel, one CTA per body), or with a camera against 2D keypoints (the grouped, calibrated and sequence
// kernels below; the single-image 2D step keeps its normal matrix in shared memory instead, lm_kp2d_step_kernel).
// Parameters [delta_j (3 n_rot) | beta (NB) | the last 3: t or c], P =3 n_rot + NB + 3, R_j(delta) = R_j Exp(delta_j);
// the caller evaluates the trial with shapy_smplx_keypoint_jacobian.  The kernels differ in their loss and in the rows
// they stage; the phases below, each by the whole CTA on the shared-memory state, are the same code in all:
//   2. lm_kp_take_trial: an accepted trial becomes the state;
//   3. lm_kp_pairs, lm_kp_add_rows, lm_kp_damp: the P x P normal matrix J^T W J and g = J^T W r from staged rows, the
//      lower triangle spread over the threads' registers, then lambda by lm_step_kernel's policy on the diagonal;
//   4. lm_kp_solve: a right-looking Cholesky in fp64 shared memory and the two triangular solves;
//   5. lm_kp_next_trial: R_j Exp(delta_j), beta + delta_beta and the last three + their delta, rounded to fp32.
constexpr int kLmKpMaxP = 96;
constexpr int kLmKpThreads = 256;
constexpr int kLmKpPairs = (kLmKpMaxP * (kLmKpMaxP + 1) / 2 + kLmKpThreads - 1) / kLmKpThreads;
constexpr int kLmKpRows = 16;           // Jacobian rows staged in shared memory at a time

struct LmKpArgs {                       // what the keypoint steps share; `last` is transl (3D) or camera (2D)
  int K, n_rot, nb, P;
  const float *targets, *weights;
  float up, down;
  int first;
  float *rot, *betas, *last, *kp, *jac, *loss, *lambda;
  int *accepted;
  float *trot, *tbetas, *tlast;
  const float *tkp, *tjac;
};

// Phase 2 on accept: the trial's parameters, keypoints, Jacobian and loss become the state; without `body` only the
// image's own part (rotations, the last three, keypoints, Jacobian): the grouped step keeps betas and loss per group
__device__ __forceinline__ void lm_kp_take_trial(const LmKpArgs &a, int b, float lnew, bool body = true) {
  const int t = threadIdx.x, nb = a.nb, R3 = 3 * a.K;
  const size_t nr9 = (size_t)a.n_rot * 9;
  for (size_t i = t; i < nr9; i += blockDim.x) a.rot[b * nr9 + i] = a.trot[b * nr9 + i];
  if (body)
    for (int i = t; i < nb; i += blockDim.x) a.betas[(size_t)b * nb + i] = a.tbetas[(size_t)b * nb + i];
  if (t < 3) a.last[(size_t)b * 3 + t] = a.tlast[(size_t)b * 3 + t];
  for (int i = t; i < R3; i += blockDim.x) a.kp[(size_t)b * R3 + i] = a.tkp[(size_t)b * R3 + i];
  for (size_t i = t; i < (size_t)R3 * a.P; i += blockDim.x)
    a.jac[(size_t)b * R3 * a.P + i] = a.tjac[(size_t)b * R3 * a.P + i];
  if (body && t == 0) a.loss[b] = lnew;
}

// Phase 3, ownership: thread t accumulates the lower-triangle entries t + kLmKpThreads i (row-major) of the normal
// matrix in acc[i], entry (pr[i], pc[i]), pr[i] = -1 past the last one (and g_t, by the caller)
__device__ __forceinline__ void lm_kp_pairs(int P, int (&pr)[kLmKpPairs], int (&pc)[kLmKpPairs],
                                            double (&acc)[kLmKpPairs]) {
  const int npairs = P * (P + 1) / 2;
#pragma unroll
  for (int i = 0; i < kLmKpPairs; ++i) {
    const int p = threadIdx.x + kLmKpThreads * i;
    int r = (int)((sqrt(8.0 * p + 1.0) - 1.0) * 0.5);
    while ((r + 1) * (r + 2) / 2 <= p) ++r;
    while (r * (r + 1) / 2 > p) --r;
    pr[i] = p < npairs ? r : -1;
    pc[i] = p - r * (r + 1) / 2;
    acc[i] = 0.0;
  }
}

// Phase 3, accumulation: A_ij += (w J_ri) J_rj and g_t += (w J_rt) res_r over the nr staged rows in order (Js = J_r,
// WJs = w J_r, ws = w, rs = res); a row with w <= 0 was not staged and is never read
__device__ __forceinline__ void lm_kp_add_rows(int nr, int P, const double (*Js)[kLmKpMaxP],
                                               const double (*WJs)[kLmKpMaxP], const double *ws, const double *rs,
                                               const int (&pr)[kLmKpPairs], const int (&pc)[kLmKpPairs],
                                               double (&acc)[kLmKpPairs], double &g) {
  for (int row = 0; row < nr; ++row) {
    const double w = ws[row];
    if (!(w > 0.0)) continue;
#pragma unroll
    for (int i = 0; i < kLmKpPairs; ++i)
      if (pr[i] >= 0) acc[i] += WJs[row][pr[i]] * Js[row][pc[i]];
    if (threadIdx.x < P) g += WJs[row][threadIdx.x] * rs[row];
  }
}

// Phase 3, the end: A (the P x P lower triangle) and y = -g go to shared memory
__device__ __forceinline__ void lm_kp_store(int P, double *A, double *y, const int (&pr)[kLmKpPairs],
                                            const int (&pc)[kLmKpPairs], const double (&acc)[kLmKpPairs], double g) {
#pragma unroll
  for (int i = 0; i < kLmKpPairs; ++i)
    if (pr[i] >= 0) A[pr[i] * P + pc[i]] = acc[i];
  if (threadIdx.x < P) y[threadIdx.x] = -g;
  __syncthreads();
}

// Phase 3, the end: lm_kp_store, then thread 0 sets lambda (lm_lambda; the first from the P
// entries diag[0], diag[stride], ...: the caller says which rows' diagonal counts), counts an accepted trial and damps
// the diagonal, by (double)rho + (double)lambda on the columns [lo, hi) and lambda elsewhere.  ok_s starts as "the
// state's loss is finite": a body without a finite loss does not move
__device__ __forceinline__ void lm_kp_damp(const LmKpArgs &a, int b, bool accept, float lnew, double *A, double *y,
                                           const int (&pr)[kLmKpPairs], const int (&pc)[kLmKpPairs],
                                           const double (&acc)[kLmKpPairs], double g, const double *diag, int stride,
                                           int lo, int hi, float rho, int &ok_s) {
  const int P = a.P;
  lm_kp_store(P, A, y, pr, pc, acc, g);
  if (threadIdx.x == 0) {
    double dmax = kDiagFloor;
    if (a.first)
      for (int j = 0; j < P; ++j) dmax = fmax(dmax, diag[j * stride]);
    const float lam = lm_lambda(a.first, accept, a.first ? 0.f : a.lambda[b], dmax, a.up, a.down);
    a.lambda[b] = lam;
    if (accept && !a.first) a.accepted[b] += 1;
    const double damp = (double)rho + (double)lam;
    for (int j = 0; j < P; ++j) A[j * P + j] += j >= lo && j < hi ? damp : (double)lam;
    ok_s = isfinite(lnew);
  }
}

// Phase 4: Cholesky A = L L^T of the P x P lower triangle in shared memory, right-looking (column j scaled, then the
// trailing lower triangle updated), then L y = -g and L^T delta = y in place in y; thread 0 clears ok_s on a pivot that
// is not positive and finite.  With n < P only the leading n columns are eliminated: the trailing block is then the
// Schur complement C - B^T A11^-1 B, y's tail -(g2 - B^T A11^-1 g1), and y's head -A11^-1 g1
__device__ __forceinline__ void lm_kp_solve(double *A, double *y, int P, int n, int &ok_s) {
  const int t = threadIdx.x;
  for (int j = 0; j < n; ++j) {
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
  for (int j = 0; j < n; ++j) {
    __syncthreads();
    const double yj = y[j] / A[j * P + j];
    __syncthreads();
    if (t == 0) y[j] = yj;
    for (int i = j + 1 + t; i < P; i += blockDim.x) y[i] -= A[i * P + j] * yj;
  }
  for (int j = n - 1; j >= 0; --j) {
    __syncthreads();
    const double dj = y[j] / A[j * P + j];
    __syncthreads();
    if (t == 0) y[j] = dj;
    for (int i = t; i < j; i += blockDim.x) y[i] -= A[j * P + i] * dj;
  }
  __syncthreads();
}

// R Exp(d) by Rodrigues in fp64, re-orthonormalised by the 6D decoder's Gram-Schmidt of the first two columns, rounded
// to fp32: the rotation update of every keypoint step
__device__ __forceinline__ void lm_exp_gs(const float *Rs, double d0, double d1, double d2, float *Rt) {
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

// The next trial rotation Rt: Rs Exp(d) (lm_exp_gs) when the step succeeded (ok), else a copy of the state's Rs
__device__ __forceinline__ void lm_rot_next(const float *Rs, const double *d, bool ok, float *Rt) {
  if (ok) lm_exp_gs(Rs, d[0], d[1], d[2], Rt);
  else
    for (int e = 0; e < 9; ++e) Rt[e] = Rs[e];
}

// Phase 5, the next trial from the state and delta = y: the rotations by lm_rot_next, beta + delta_beta and the last
// three parameters + their delta, all rounded to fp32; the state itself when the step failed (!ok)
__device__ __forceinline__ void lm_kp_next_trial(const LmKpArgs &a, int b, const double *y, bool ok) {
  const int t = threadIdx.x, nb = a.nb, o = 3 * a.n_rot;
  const float *sr = a.rot + (size_t)b * a.n_rot * 9;
  float *trr = a.trot + (size_t)b * a.n_rot * 9;
  for (int j = t; j < a.n_rot; j += blockDim.x) lm_rot_next(sr + 9 * j, y + 3 * j, ok, trr + 9 * j);
  for (int l = t; l < nb; l += blockDim.x) {
    const float x = a.betas[(size_t)b * nb + l];
    a.tbetas[(size_t)b * nb + l] = ok ? (float)((double)x + y[o + l]) : x;
  }
  if (t < 3) {
    const float x = a.last[(size_t)b * 3 + t];
    a.tlast[(size_t)b * 3 + t] = ok ? (float)((double)x + y[o + nb + t]) : x;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// The step of the fit to 3D keypoints (shapy_fit_lm_keypoints_step), the last three parameters the translation t.  The
// policy is lm_step_kernel's without the betas regulariser: L = sum_{w_k > 0} w_k |kp_k - target_k|^2 (fp64, k order),
// the rows the keypoint Jacobian's in keypoint-major xyz order, (J^T W J + lambda I) delta = -J^T W (kp - target).
//
// MEAS (shapy_fit_lm_keypoints_measurements_step) stacks the five virtual measurements and the betas regulariser under
// the keypoint rows: L = L_kp + sum_{w_k > 0} w_k (t_k - m_k)^2 (k order) + rho |beta|^2 (l order), left to right.  The
// measurement Jacobian (5, NB) only has betas columns, so its rows are accumulated after the keypoint rows into the
// betas block of A and g (k order), then rho beta into g; the first lambda comes from diag(A) without rho (as in
// lm_step_kernel) and the betas diagonal gets (double)rho + (double)lambda.  With every measurement weight <= 0 and
// rho = 0 each extra term is skipped or adds an exact 0, so the step equals the keypoint step bit for bit.
struct LmMeasArgs {                     // the measurement block of the MEAS step (unused otherwise)
  const float *targets, *weights;       // (B, 5): mass, height, chest, waist, hips
  float rho;                            // betas_weight
  float *meas, *jac;                    // state (B, 5), (B, 5, NB)
  const float *tmeas, *tjac;            // the trial's
};

// The measurement block's three pieces, shared by the 3D and the 2D MEAS kernels.  Phase 1, by thread 0: the trial's
// sum_{w_k > 0} w_k (t_k - m_k)^2 in k order, summed on its own; a dropped term is never read: its measurement may be NaN
__device__ __forceinline__ double lm_meas_loss(const LmMeasArgs &mb, int b) {
  const float *tm = mb.tmeas + (size_t)b * 5, *mt = mb.targets + (size_t)b * 5, *mw = mb.weights + (size_t)b * 5;
  double Lm = 0.0;
  for (int k = 0; k < 5; ++k) {
    const double w = mw[k];
    if (w > 0.0) {
      const double r = (double)mt[k] - (double)tm[k];
      Lm += w * r * r;
    }
  }
  return Lm;
}

// Phase 2 on accept: the trial's measurements and their Jacobian become the state's
__device__ __forceinline__ void lm_meas_take_trial(const LmMeasArgs &mb, int b, int nb) {
  const int t = threadIdx.x;
  for (int i = t; i < 5; i += blockDim.x) mb.meas[(size_t)b * 5 + i] = mb.tmeas[(size_t)b * 5 + i];
  for (int i = t; i < 5 * nb; i += blockDim.x) mb.jac[(size_t)b * 5 * nb + i] = mb.tjac[(size_t)b * 5 * nb + i];
}

// Phase 3: the five measurement rows (values Mm (5), Jacobian Jm (5, nb), at the state), staged like the keypoint rows,
// into the betas block [o, o + nb) of A and g in k order, residual m_k - t_k; a dropped term's row is never read: it
// may be NaN
__device__ __forceinline__ void lm_meas_add_rows(const LmMeasArgs &mb, int b, int nb, int o, const float *Mm,
                                                 const float *Jm, double (*Js)[kLmKpMaxP], double (*WJs)[kLmKpMaxP],
                                                 double *ws, double *rs, const int (&pr)[kLmKpPairs],
                                                 const int (&pc)[kLmKpPairs], double (&acc)[kLmKpPairs], double &g) {
  const int t = threadIdx.x;
  const float *mt = mb.targets + (size_t)b * 5, *mw = mb.weights + (size_t)b * 5;
  __syncthreads();
  for (int i = t; i < 5; i += blockDim.x) {
    const double w = mw[i];
    ws[i] = w;
    rs[i] = w > 0.0 ? (double)Mm[i] - (double)mt[i] : 0.0;
  }
  for (int i = t; i < 5 * nb; i += blockDim.x) {
    const int row = i / nb;
    const double w = mw[row];
    if (w > 0.0) {
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
}

template <bool MEAS>
__global__ void __launch_bounds__(kLmKpThreads) lm_kp_step_kernel(LmKpArgs a, LmMeasArgs mb) {
  extern __shared__ double A[];         // [P][P]: the lower triangle of J^T W J + lambda I, then its Cholesky factor
  __shared__ double Js[kLmKpRows][kLmKpMaxP], WJs[kLmKpRows][kLmKpMaxP];   // staged rows J_r and w J_r
  __shared__ double rs[kLmKpRows], ws[kLmKpRows], y[kLmKpMaxP];
  __shared__ double lt_s;
  __shared__ int ok_s;
  const int b = blockIdx.x, t = threadIdx.x, P = a.P, K = a.K, R3 = 3 * a.K;
  const int o = 3 * a.n_rot;              // first betas column
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
      L += lm_meas_loss(mb, b);
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
  // 2. accept or reject
  const double lt = lt_s;
  const bool accept = lm_accept(a.first, lt, lcur);
  const float lnew = lm_loss(accept, lt, lcur);
  const float *J = (accept ? a.tjac : a.jac) + (size_t)b * R3 * P;
  const float *M = (accept ? a.tkp : a.kp) + (size_t)b * R3;
  const float *Jm = MEAS ? (accept ? mb.tjac : mb.jac) + (size_t)b * 5 * a.nb : nullptr;   // the measurement block's
  const float *Mm = MEAS ? (accept ? mb.tmeas : mb.meas) + (size_t)b * 5 : nullptr;
  if (accept) {
    lm_kp_take_trial(a, b, lnew);
    if constexpr (MEAS) lm_meas_take_trial(mb, b, a.nb);
  }
  // 3. normal equations: A_ij = sum_rows (w J_ri) J_rj (i >= j), g_i = sum_rows (w J_ri) (kp_r - target_r), rows in
  // keypoint-major xyz order, the rows of a dropped keypoint never read
  int pr[kLmKpPairs], pc[kLmKpPairs];
  double acc[kLmKpPairs], g = 0.0;
  lm_kp_pairs(P, pr, pc, acc);
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
    lm_kp_add_rows(nr, P, Js, WJs, ws, rs, pr, pc, acc, g);
  }
  if constexpr (MEAS) {
    // the five measurement rows into the betas block [o, o + nb) of A and g
    const int nb = a.nb;
    lm_meas_add_rows(mb, b, nb, o, Mm, Jm, Js, WJs, ws, rs, pr, pc, acc, g);
    if (mb.rho > 0.f && t >= o && t < o + nb)
      g += (double)mb.rho * (double)(accept ? a.tbetas : a.betas)[(size_t)b * nb + t - o];
  }
  // the first lambda from all of diag(A); only the MEAS step has a betas regulariser to damp with
  lm_kp_damp(a, b, accept, lnew, A, y, pr, pc, acc, g, A, P + 1, MEAS ? o : 0, MEAS ? o + a.nb : 0, mb.rho, ok_s);
  lm_kp_solve(A, y, P, P, ok_s);
  // 5. next trial (ok is uniform: every thread reads it after the last barrier); a failed step keeps the state
  lm_kp_next_trial(a, b, y, ok_s);
}

// ---------------------------------------------------------------------------------------------------------------
// The pieces of the 2D keypoint steps: the single-image step (lm_kp2d_step_kernel, which states the loss and the rows)
// and the grouped, shared-pose, calibrated and sequence steps build on them.
struct LmKp2dArgs {                     // what the 2D step takes beside LmKpArgs (targets (B, K, 2), last = camera)
  const float *anchor;                  // (B, n_rot, 3, 3), or null without a pose prior
  float sigma, pose_w, betas_w;
  LmMeasArgs mb;                        // the MEAS step's block (unused otherwise); its rho is not read: betas_w is the
};                                      // one betas regulariser

// The perspective step's arguments: the intrinsics ride after LmKp2dArgs, so that the grouped kernels, which take
// LmKp2dArgs before their own block, keep their parameter layout
struct LmKp2dPerspArgs : LmKp2dArgs {
  const float *intr;                    // (B, 3): f, px, py
};

// One body's pinhole camera at a point of the fit: focal length, principal point and translation t, in fp64
struct PerspCam {
  double f, pp[2], t[3];
};

__device__ __forceinline__ PerspCam persp_cam(const float *in, const float *t) {
  return PerspCam{(double)in[0], {(double)in[1], (double)in[2]}, {(double)t[0], (double)t[1], (double)t[2]}};
}

// Y_k = kp_k + t and the residual p_k - x_k of the perspective projection, in fp64
__device__ __forceinline__ void persp_residual(const float *m, const float *tg, const PerspCam &pc, int k, double (&Y)[3],
                                               double &dx, double &dy) {
  for (int c = 0; c < 3; ++c) Y[c] = (double)m[3 * k + c] + pc.t[c];
  dx = pc.f * (Y[0] / Y[2]) + pc.pp[0] - (double)tg[2 * k];
  dy = pc.f * (Y[1] / Y[2]) + pc.pp[1] - (double)tg[2 * k + 1];
}

// The factors of perspective row c at Y: f / Y_z and Y_c / Y_z into fz[0], fz[1]
__device__ __forceinline__ void persp_factors(const PerspCam &pc, const double (&Y)[3], int c, double *fz) {
  fz[0] = pc.f / Y[2];
  fz[1] = Y[c] / Y[2];
}

// One calibrated view of a body at a point of the fit: the view's intrinsics, the body's world translation t (in
// PerspCam) and the view's world-to-camera extrinsics R (row-major), T, in fp64
struct CalibCam : PerspCam {
  double R[9], T[3];
};

__device__ __forceinline__ CalibCam calib_cam(const float *in, const float *ex, const float *t) {
  CalibCam c;
  static_cast<PerspCam &>(c) = persp_cam(in, t);
  for (int i = 0; i < 9; ++i) c.R[i] = (double)ex[i];
  for (int i = 0; i < 3; ++i) c.T[i] = (double)ex[9 + i];
  return c;
}

// Y_k = R (kp_k + t) + T (each row left to right, then + T_c) and the residual p_k - x_k of its projection, in fp64
__device__ __forceinline__ void persp_residual(const float *m, const float *tg, const CalibCam &pc, int k, double (&Y)[3],
                                               double &dx, double &dy) {
  double X[3];
  for (int c = 0; c < 3; ++c) X[c] = (double)m[3 * k + c] + pc.t[c];
  for (int c = 0; c < 3; ++c) Y[c] = pc.R[3 * c] * X[0] + pc.R[3 * c + 1] * X[1] + pc.R[3 * c + 2] * X[2] + pc.T[c];
  dx = pc.f * (Y[0] / Y[2]) + pc.pp[0] - (double)tg[2 * k];
  dy = pc.f * (Y[1] / Y[2]) + pc.pp[1] - (double)tg[2 * k + 1];
}

// The factors of calibrated row c at Y: the projected rotation row u_d = (f / Y_z) (R_cd - (Y_c / Y_z) R_2d) into
// fz[0 .. 2], so that the row is u . J3_k (u_d itself on the t column d)
__device__ __forceinline__ void persp_factors(const CalibCam &pc, const double (&Y)[3], int c, double *fz) {
  const double a = pc.f / Y[2], b = Y[c] / Y[2];
  for (int d = 0; d < 3; ++d) fz[d] = a * (pc.R[3 * c + d] - b * pc.R[6 + d]);
}

// The perspective rows' factors f / Y_z and Y_c / Y_z per staged row: shared memory only the perspective kernels have
__device__ __forceinline__ double *lm_persp_factors() {
  __shared__ double fz[2 * kLmKpRows];
  return fz;
}

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

// Phase 1 of the 2D steps, by one thread: the pose prior 1/2 pose_w sum_{j >= 1} |R_j - R0_j|_F^2 of the rotations tr
// (row-major entries in j order) against the anchor anc
__device__ __forceinline__ double lm_kp2d_prior_loss(const LmKp2dArgs &x2, const float *tr, const float *anc, int nr9) {
  double q = 0.0;
  for (int i = 9; i < nr9; ++i) {
    const double d = (double)tr[i] - (double)anc[i];
    q += d * d;
  }
  return 0.5 * (double)x2.pose_w * q;
}

// Phase 1 of the 2D steps, by one thread: the trial's robust keypoint term (k order) and pose prior, left to right.
// PERSP: the projection of the trial's camera pc (Cam: PerspCam, or CalibCam for one calibrated view), +inf under the
// depth rule
template <bool PERSP = false, typename Cam = PerspCam>
__device__ __forceinline__ double lm_kp2d_trial_loss(const LmKpArgs &a, const LmKp2dArgs &x2, int b, const float *tg,
                                                     const float *wt, const float *anc, bool robust, double s2,
                                                     const Cam *pc = nullptr) {
  const int K = a.K, R3 = 3 * a.K, nr9 = 9 * a.n_rot;
  const float *m = a.tkp + (size_t)b * R3, *cam = a.tlast + (size_t)b * 3;
  double s, ds;
  softplus_d((double)cam[0], s, ds);
  const double cx = cam[1], cy = cam[2];
  if constexpr (PERSP)
    if (!(pc->f > 0.0) || !isfinite(pc->f)) return INFINITY;
  double L = 0.0;
  for (int k = 0; k < K; ++k) {
    const double w = wt[k];
    if (!(w > 0.0)) continue;
    double dx, dy;
    if constexpr (PERSP) {
      double Y[3];
      persp_residual(m, tg, *pc, k, Y, dx, dy);
      if (!(Y[2] > 0.0) || !isfinite(Y[2])) return INFINITY;
    } else {
      dx = s * ((double)m[3 * k] + cx) - (double)tg[2 * k];
      dy = s * ((double)m[3 * k + 1] + cy) - (double)tg[2 * k + 1];
    }
    const double e = dx * dx + dy * dy;
    L += w * (robust ? e * (s2 / (s2 + e)) : e);
  }
  if (x2.pose_w > 0.f) L += lm_kp2d_prior_loss(x2, a.trot + (size_t)b * nr9, anc, nr9);
  return L;
}

// Phase 3 of the 2D steps: row c of keypoint k at the state (keypoints M, scale s, offset cxy), its weight w_k q_k^2 (the
// IRLS weight, w_k at sigma = inf) and residual; a dropped keypoint (w_k <= 0) keeps w_k and a zero residual.  PERSP:
// the state's camera pc, and the row's factors into fz (persp_factors of its Cam)
template <bool PERSP = false, typename Cam = PerspCam>
__device__ __forceinline__ void lm_kp2d_row(const float *M, const float *tg, const float *wt, double s,
                                            const double (&cxy)[2], bool robust, double s2, int k, int c, double &wr,
                                            double &res, const Cam *pc = nullptr, double *fz = nullptr) {
  const double w = wt[k];
  wr = w;
  res = 0.0;
  if (w > 0.0) {
    double dx, dy;
    if constexpr (PERSP) {
      double Y[3];
      persp_residual(M, tg, *pc, k, Y, dx, dy);
      persp_factors(*pc, Y, c, fz);
    } else {
      dx = s * ((double)M[3 * k] + cxy[0]) - (double)tg[2 * k];
      dy = s * ((double)M[3 * k + 1] + cxy[1]) - (double)tg[2 * k + 1];
    }
    if (robust) {
      const double q = s2 / (s2 + (dx * dx + dy * dy));
      wr = w * (q * q);
    }
    res = c ? dy : dx;
  }
}

// Column col of that row, the camera columns at oc: s J_{3k+c} on the rotation and betas columns, ds (kp_kc + c_{1+c})
// on c0, s on c_{1+c}.  REORDER: columns [delta | c | beta] (the grouped step), else [delta | beta | c].  PERSP (columns
// [delta | beta | t]): fz[0] (J_{3k+c} - fz[1] J_{3k+2}) with the row's factors fz, J_t = I; with a CalibCam, fz[0]
// J_{3k} + fz[1] J_{3k+1} + fz[2] J_{3k+2} (fz[d] on t column d).  REORDER and PERSP: the perspective row in the
// columns [delta | t | beta] (the sequence step), t at oc .. oc + 2
template <bool REORDER, bool PERSP = false, typename Cam = PerspCam>
__device__ __forceinline__ double lm_kp2d_entry(const float *J, const float *M, int P, int oc, int k, int c, int col,
                                                double s, double ds, const double (&cxy)[2],
                                                const double *fz = nullptr) {
  if constexpr (PERSP && std::is_same_v<Cam, CalibCam>) {
    if (col >= oc) return fz[col - oc];
    const float *Jk = J + (size_t)(3 * k) * P + col;
    return fz[0] * (double)Jk[0] + fz[1] * (double)Jk[P] + fz[2] * (double)Jk[2 * P];
  } else if constexpr (PERSP && REORDER) {
    const bool tcol = col >= oc && col < oc + 3;
    const int jcol = col < oc ? col : col - 3;      // a betas column of the Jacobian sits 3 to the left
    const double jc = tcol ? (col - oc == c ? 1.0 : 0.0) : (double)J[(size_t)(3 * k + c) * P + jcol];
    const double jz = tcol ? (col - oc == 2 ? 1.0 : 0.0) : (double)J[(size_t)(3 * k + 2) * P + jcol];
    return fz[0] * (jc - fz[1] * jz);
  } else if constexpr (PERSP) {
    const double jc = col < oc ? (double)J[(size_t)(3 * k + c) * P + col] : (col - oc == c ? 1.0 : 0.0);
    const double jz = col < oc ? (double)J[(size_t)(3 * k + 2) * P + col] : (col - oc == 2 ? 1.0 : 0.0);
    return fz[0] * (jc - fz[1] * jz);
  }
  const bool betas = REORDER && col > oc + 2;
  if (col < oc || betas) return s * (double)J[(size_t)(3 * k + c) * P + (betas ? col - 3 : col)];
  if (col == oc) return ds * ((double)M[3 * k + c] + cxy[c]);
  return col - oc - 1 == c ? s : 0.0;
}

// Phase 3 of the 2D steps: the keypoint rows 2k + c, staged kLmKpRows at a time and accumulated in row order.  PERSP:
// the perspective rows of the state's camera cam
template <bool REORDER, bool PERSP = false>
__device__ __forceinline__ void lm_kp2d_keypoint_rows(int K, int P, const float *J, const float *M,
                                                      const float *tg, const float *wt, double s, double ds,
                                                      const double (&cxy)[2], bool robust, double s2, int oc,
                                                      double (*Js)[kLmKpMaxP], double (*WJs)[kLmKpMaxP], double *ws,
                                                      double *rs, const int (&pr)[kLmKpPairs],
                                                      const int (&pc)[kLmKpPairs], double (&acc)[kLmKpPairs],
                                                      double &g, const PerspCam *cam = nullptr) {
  const int t = threadIdx.x, R2 = 2 * K;
  double *fz = nullptr;
  if constexpr (PERSP) fz = lm_persp_factors();
  for (int r0 = 0; r0 < R2; r0 += kLmKpRows) {
    const int nr = min(kLmKpRows, R2 - r0);
    __syncthreads();
    for (int i = t; i < nr; i += blockDim.x) {   // row weight (IRLS at the state) and residual
      double wr, res;
      lm_kp2d_row<PERSP>(M, tg, wt, s, cxy, robust, s2, (r0 + i) >> 1, (r0 + i) & 1, wr, res, cam,
                         PERSP ? fz + 2 * i : nullptr);
      ws[i] = wr;
      rs[i] = res;
    }
    __syncthreads();
    for (int i = t; i < nr * P; i += blockDim.x) {
      const int row = i / P, col = i % P;
      const double wr = ws[row];
      if (wr > 0.0) {                    // a dropped keypoint's rows are never read: they may be NaN
        const double x = lm_kp2d_entry<REORDER, PERSP>(J, M, P, oc, (r0 + row) >> 1, (r0 + row) & 1, col, s, ds, cxy,
                                                       PERSP ? fz + 2 * row : nullptr);
        Js[row][col] = x;
        WJs[row][col] = wr * x;
      }
    }
    __syncthreads();
    lm_kp_add_rows(nr, P, Js, WJs, ws, rs, pr, pc, acc, g);
  }
}

// Phase 3 of the 2D steps: the pose-prior rows of joint j only reach its diagonal block (parameters 3 j .. 3 j + 2, the
// same in both column orders): no staging.  Column c of A holds parameter c + SHIFT: 0 in the image steps, 3 in the
// shared block [delta_1 .. | beta] of the shared-pose group step
template <int SHIFT = 0>
__device__ __forceinline__ void lm_kp2d_prior_rows(const LmKp2dArgs &x2, int o, const float *Rst, const float *anc,
                                                   const int (&pr)[kLmKpPairs], const int (&pc)[kLmKpPairs],
                                                   double (&acc)[kLmKpPairs], double &g) {
  const int t = threadIdx.x;
  if (x2.pose_w > 0.f) {
    const double hw = 0.5 * (double)x2.pose_w;
#pragma unroll
    for (int i = 0; i < kLmKpPairs; ++i) {
      const int j = (pr[i] + SHIFT) / 3;
      if (pr[i] + SHIFT >= 3 && pr[i] + SHIFT < o && (pc[i] + SHIFT) / 3 == j) {
        const float *R = Rst + 9 * j;
        for (int e = 0; e < 9; ++e)
          acc[i] += (hw * rot_tangent(R, (pr[i] + SHIFT) % 3, e)) * rot_tangent(R, (pc[i] + SHIFT) % 3, e);
      }
    }
    if (t + SHIFT >= 3 && t + SHIFT < o) {
      const float *R = Rst + 9 * ((t + SHIFT) / 3), *R0 = anc + 9 * ((t + SHIFT) / 3);
      for (int e = 0; e < 9; ++e) g += (hw * rot_tangent(R, (t + SHIFT) % 3, e)) * ((double)R[e] - (double)R0[e]);
    }
  }
}

// What the 3D, grouped, calibrated and sequence keypoint entry points share, `fn` naming the one called: the checks of
// the arguments in `a` (its P is set here), with `extra_ok` the entry point's own pointers and `factors_ok` / `factors`
// its own scalars and the sentence that states their and the lambda factors' ranges; then the launch, one CTA of
// kLmKpThreads per body with P x P doubles of dynamic shared memory
inline int check_lm_kp(const char *fn, int batch, LmKpArgs &a, bool extra_ok, bool factors_ok, const char *factors) {
  SHAPY_REQUIRE(a.targets && a.weights && a.rot && a.betas && a.last && a.kp && a.jac && a.loss && a.lambda &&
                    a.accepted && a.trot && a.tbetas && a.tlast && a.tkp && a.tjac && extra_ok,
                "%s: null argument", fn);
  SHAPY_REQUIRE(batch >= 0 && a.K >= 1 && a.n_rot >= 1 && a.n_rot <= 64 && a.nb >= 1,
                "%s: bad size (batch %d, %d keypoints, n_rot %d, %d betas)", fn, batch, a.K, a.n_rot, a.nb);
  SHAPY_REQUIRE(a.up >= 1.f && a.down >= 1.f && factors_ok, "%s: %s", fn, factors);
  a.P = 3 * a.n_rot + a.nb + 3;
  if (a.P > kLmKpMaxP) {
    set_error("%s: %d parameters, at most %d are supported", fn, a.P, kLmKpMaxP);
    return SHAPY_ERR_UNSUPPORTED;
  }
  return SHAPY_OK;
}

// Lets `kernel` launch with `smem` bytes of dynamic shared memory: past 48 KB of static plus dynamic shared memory a
// launch has to opt in
template <typename... Args>
cudaError_t allow_dynamic_smem(void (*kernel)(Args...), size_t smem) {
  cudaFuncAttributes attr;
  cudaError_t e = cudaFuncGetAttributes(&attr, kernel);
  if (e == cudaSuccess && smem + attr.sharedSizeBytes > 48 * 1024)
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  return e;
}

// One launch of `kernel` on `grid` CTAs of `block` threads with `smem` bytes of dynamic shared memory, opted in when
// there are any, and its launch check
template <typename... Params, typename... Args>
int lm_launch(void (*kernel)(Params...), int grid, int block, size_t smem, void *stream, const Args &...args) {
  if (smem > 0) SHAPY_CUDA_TRY(allow_dynamic_smem(kernel, smem));
  kernel<<<grid, block, smem, (cudaStream_t)stream>>>(args...);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

// The dynamic shared memory of a CTA that holds one P x P fp64 normal matrix
inline size_t lm_kp_smem(int P) { return (size_t)P * P * sizeof(double); }

template <typename Extra>
int run_lm_kp(const char *fn, void (*kernel)(LmKpArgs, Extra), int batch, LmKpArgs a, Extra x, bool extra_ok,
              bool factors_ok, const char *factors, void *stream) {
  const int rc = check_lm_kp(fn, batch, a, extra_ok, factors_ok, factors);
  if (rc != SHAPY_OK) return rc;
  if (batch == 0) return SHAPY_OK;
  return lm_launch(kernel, batch, kLmKpThreads, lm_kp_smem(a.P), stream, a, x);
}

// The measurement block's six pointers of a _measurements_ entry
inline bool lm_meas_ptrs(const LmMeasArgs &m) {
  return m.targets && m.weights && m.meas && m.jac && m.tmeas && m.tjac;
}

// The scalars of the 2D steps, and the sentence that states their and the lambda factors' ranges
inline bool lm_kp2d_factors_ok(const LmKp2dArgs &x) { return x.sigma > 0.f && x.pose_w >= 0.f && x.betas_w >= 0.f; }
constexpr const char *kLmKp2dFactors =
    "robust_sigma must be > 0 (inf: least squares), the prior weights >= 0 and lambda_up and lambda_down >= 1";

// The pointers of a grouped, calibrated or sequence 2D entry beside check_lm_kp's: the anchor when there is a pose
// prior, and the measurement block's with `meas`
inline bool lm_kp2d_ptrs(const LmKp2dArgs &x, bool meas) {
  return (x.anchor || !(x.pose_w > 0.f)) && (!meas || lm_meas_ptrs(x.mb));
}

// ---------------------------------------------------------------------------------------------------------------
// The grouped 2D step (shapy_fit_lm_keypoints_2d_groups_step): the images [off[g], off[g + 1]) of group g share one
// beta_g, each keeps its rotations and camera.  Per group, in fp64, left to right:
//   L_g = sum_{i in g} (image order) [the 2D step's keypoint term + pose prior of image i]
//       + sum_{u_m > 0} u_m (t_gm - meas_gm)^2 (m order, summed on its own; the MEAS entry, on the T-pose of beta_g)
//       + betas_w |beta_g|^2 (l order; when betas_w > 0).
// The normal matrix of a group is block-arrow shaped: image i's block [delta_i | c_i] (n1 = 3 n_rot + 3 columns) only
// meets beta.  The exact LM step eliminates each image's block (a Schur complement), in three launches:
//   1. lm_kp2dg_loss_kernel, per image: the bracket of the trial's loss into its scratch; on the first step also the
//      diagonal of the trial's keypoint rows (the max of its n1 leading entries and its nb betas entries);
//   2. lm_kp2dg_image_kernel, per image: the decision of its group (lm_group_of; lm_group_decide from the siblings'
//      scratch), on accept the image's trial becomes its state; the 2D step's keypoint and pose-prior rows staged in the
//      column order [delta | c | beta], the leading n1 x n1 block damped by lambda and factored alone (lm_kp_solve with
//      n = n1), then X_i = A_i^-1 B_i (lm_kp_solve_rows); into scratch S_i = C_i - B_i^T X_i (the factor's trailing
//      block), s_i = g_beta,i - B_i^T A_i^-1 g_i, X_i, x_i = A_i^-1 g_i and the pivots' flag;
//   3. lm_kp2dg_group_kernel, per group: the same decision recorded in the group's state (lm_group_commit; on accept
//      also beta and the measurements), S = sum_i S_i and s = sum_i s_i (image order), then the measurement rows (m
//      order) and betas_w beta_g, (S + (betas_w + lambda) I) dbeta = -s by the same Cholesky, and per image delta_i =
//      -x_i - X_i dbeta (l order) and the next trial R Exp(delta) (lm_rot_next), c + delta_c, beta_g + dbeta (both
//      trial betas arrays).
// The first lambda is 1e-3 max(1e-6, the largest diagonal entry of the group's keypoint rows): per image on its pose
// and camera columns, summed over the images (image order) on the betas columns.  A group whose loss is not finite, or
// one of whose factorisations fails, keeps its state.  Every CTA of a group decides from the same scratch in the same
// order; no atomics, so a group's bits do not depend on the rest of the batch.  A group of one has the 2D step's loss,
// lambda and decision bit for bit; its trial differs by the order of elimination.
//
// SHARE, the shared-pose group step (shapy_fit_lm_keypoints_2d_shared_pose_step): the images of a group are views of
// one posed body at one moment, so they also share the body rotations R_g,j, j = 1 .. n_rot - 1 (each relative to its
// parent); only the global rotation R_0,i (which absorbs the camera's rotation) and the camera c_i are per image.  The
// group's pose prior is counted once, against a per-group anchor:
//   L_g = sum_{i in g} (image order) [the 2D step's keypoint term of image i]
//       + 1/2 pose_w sum_{j >= 1} |R_g,j - R0_g,j|_F^2 (j order, row-major entries; when pose_w > 0)
//       + the measurement and betas terms as above.
// The phases are the same with the image block [delta_0 | c] (n1 = 6) and the shared block [delta_1 .. delta_{n_rot-1}
// | beta] (ns = 3 (n_rot - 1) + nb): the keypoint rows staged in the order [delta_0 | c | delta_1 .. | beta] and no
// prior rows in launch 2; lm_group_decide adds the prior after the summed brackets, from the group's trial rotations
// (its first image's rows); launch 3 adds the pose-prior rows of joints 1 .. n_rot - 1 on the group's state rotations
// (again the first image's rows) before the measurement rows, which go to the betas block at 3 (n_rot - 1), damps the
// rotation diagonal by lambda and the betas diagonal by betas_w + lambda, and writes R_g,j Exp(dshared_j) identically
// into every image's trial rows.  The rows of joints 1 .. of every image of a group must hold the same rotations on the
// first step; the step keeps them so.  With n_rot = 1 nothing is shared but beta, and the step is the grouped step's.
struct LmGroupArgs {
  int G;
  const int *off;                       // (G + 1) offsets, the device copy in the workspace
  double *scr;                          // per image scratch, `stride` doubles each (lm_group_scratch)
  int stride;
  float *tbetas_img;                    // (B, nb): the trial betas per image, for the keypoint Jacobian
};

// The slots of an image's scratch: the bracket of its trial loss, the factorisation flag, the max of its first-step
// keypoint diagonal over the image block, then its ns shared-column diagonal entries, S_i (ns x ns, lower), s_i (ns),
// X_i (n1 x ns) and x_i (n1); ns = nb in the grouped step
constexpr int kScrLoss = 0, kScrOk = 1, kScrDmax = 2, kScrDiag = 3;
__host__ __device__ inline int lm_group_stride(int n1, int nb) { return kScrDiag + 2 * nb + nb * nb + n1 * nb + n1; }
inline size_t lm_group_offsets_bytes(int G) { return ((size_t)(G + 1) * sizeof(int) + 15) / 16 * 16; }

// The offsets `name` of a grouped entry, checked on the host: (G + 1) entries rising strictly from 0 to `rows` (the
// images, views or frames), so that no group, body or sequence is empty.  Then copied on the stream into the head of
// the workspace, where the kernels read them; nothing is copied for G = 0
inline int put_group_offsets(const char *fn, const char *name, int rows, int G, const int32_t *offsets,
                             void *workspace, void *stream) {
  SHAPY_REQUIRE(G >= 0 && offsets[0] == 0 && offsets[G] == rows, "%s: %s must run from 0 to %d over %d entries + 1",
                fn, name, rows, G);
  for (int g = 0; g < G; ++g)
    SHAPY_REQUIRE(offsets[g + 1] > offsets[g], "%s: %s must rise strictly (entries %d, %d: %d, %d)", fn, name, g,
                  g + 1, offsets[g], offsets[g + 1]);
  if (G > 0)
    SHAPY_CUDA_TRY(cudaMemcpyAsync(workspace, offsets, (size_t)(G + 1) * sizeof(int), cudaMemcpyHostToDevice,
                                   (cudaStream_t)stream));
  return SHAPY_OK;
}

struct LmGroupDecision {
  bool accept;
  float lnew, lam;
};

// The group's decision, by one thread, from the images' scratch of launch 1 and the group state: its trial loss L_g,
// accept (lm_accept), the state's loss after it (lm_loss) and lambda (lm_lambda, the first from the group diagonal).
// SHARE adds the group's pose prior after the keypoint brackets
template <bool SHARE>
__device__ LmGroupDecision lm_group_decide(const LmKpArgs &a, const LmKp2dArgs &x2, const LmGroupArgs &gr, int g) {
  const int i0 = gr.off[g], i1 = gr.off[g + 1], nb = a.nb;
  const int ns = SHARE ? a.P - 6 : nb;  // the shared columns
  const double *s0 = gr.scr + (size_t)i0 * gr.stride;
  double L = s0[kScrLoss];
  for (int i = i0 + 1; i < i1; ++i) L += gr.scr[(size_t)i * gr.stride + kScrLoss];
  if constexpr (SHARE) {
    const int nr9 = 9 * a.n_rot;
    if (x2.pose_w > 0.f) L += lm_kp2d_prior_loss(x2, a.trot + (size_t)i0 * nr9, x2.anchor + (size_t)g * nr9, nr9);
  }
  if (x2.mb.weights) L += lm_meas_loss(x2.mb, g);
  if (x2.betas_w > 0.f) L += (double)x2.betas_w * lm_sq_norm(a.tbetas + (size_t)g * nb, nb);
  const float lcur = a.loss[g];
  LmGroupDecision d;
  d.accept = lm_accept(a.first, L, lcur);
  d.lnew = lm_loss(d.accept, L, lcur);
  double dmax = kDiagFloor;
  if (a.first) {
    for (int i = i0; i < i1; ++i) dmax = fmax(dmax, gr.scr[(size_t)i * gr.stride + kScrDmax]);
    for (int l = 0; l < ns; ++l) {
      double d2 = s0[kScrDiag + l];
      for (int i = i0 + 1; i < i1; ++i) d2 += gr.scr[(size_t)i * gr.stride + kScrDiag + l];
      dmax = fmax(dmax, d2);
    }
  }
  d.lam = lm_lambda(a.first, d.accept, a.first ? 0.f : a.lambda[g], dmax, a.up, a.down);
  return d;
}

// lm_group_decide by the group's own CTA, which also records it in the group state: the loss on accept, lambda and
// the accept count
template <bool SHARE>
__device__ __forceinline__ LmGroupDecision lm_group_commit(const LmKpArgs &a, const LmKp2dArgs &x2,
                                                           const LmGroupArgs &gr, int g) {
  const LmGroupDecision d = lm_group_decide<SHARE>(a, x2, gr, g);
  if (d.accept) a.loss[g] = d.lnew;
  a.lambda[g] = d.lam;
  if (d.accept && !a.first) a.accepted[g] += 1;
  return d;
}

// The group g with off[g] <= b < off[g + 1] of image (view, frame) b, by one thread
__device__ __forceinline__ int lm_group_of(const LmGroupArgs &gr, int b) {
  int lo = 0, hi = gr.G - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (gr.off[mid] <= b) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// After lm_kp_solve(A, y, P, n, ..): X = A11^-1 B in place in the ns rows n.. of A, which held L21.  L11^T X = L21^T,
// column by column from the last, as the solve's L^T delta = y
__device__ __forceinline__ void lm_kp_solve_rows(double *A, int P, int n, int ns) {
  const int t = threadIdx.x;
  for (int j = n - 1; j >= 0; --j) {
    for (int l = t; l < ns; l += blockDim.x) A[(n + l) * P + j] /= A[j * P + j];
    __syncthreads();
    for (int q = t; q < ns * j; q += blockDim.x) {
      const int l = q / j, i = q % j;
      A[(n + l) * P + i] -= A[j * P + i] * A[(n + l) * P + j];
    }
    __syncthreads();
  }
}

template <bool SHARE>
__global__ void __launch_bounds__(128) lm_kp2dg_loss_kernel(LmKpArgs a, LmKp2dArgs x2, LmGroupArgs gr) {
  __shared__ double dg[kLmKpMaxP];
  const int b = blockIdx.x, t = threadIdx.x, P = a.P, K = a.K, o = 3 * a.n_rot;
  const int oc = SHARE ? 3 : o, ns = SHARE ? P - 6 : a.nb;   // the first camera column, the shared columns
  const float *tg = a.targets + (size_t)b * 2 * K, *wt = a.weights + (size_t)b * K;
  const float *anc = x2.anchor ? x2.anchor + (size_t)b * 9 * a.n_rot : nullptr;
  const bool robust = isfinite(x2.sigma);
  const double s2 = (double)x2.sigma * (double)x2.sigma;
  double *scr = gr.scr + (size_t)b * gr.stride;
  if (t == 0) {
    if constexpr (SHARE) {
      LmKp2dArgs xk = x2;                 // the keypoint term alone: the group counts its prior once
      xk.pose_w = 0.f;
      scr[kScrLoss] = lm_kp2d_trial_loss(a, xk, b, tg, wt, nullptr, robust, s2);
    } else {
      scr[kScrLoss] = lm_kp2d_trial_loss(a, x2, b, tg, wt, anc, robust, s2);
    }
  }
  if (!a.first) return;
  // the first step accepts: the diagonal of the trial's keypoint rows, column t of [delta | c | beta] (SHARE: [delta_0 |
  // c | delta_1 .. | beta]), in row order
  if (t < P) {
    const float *J = a.tjac + (size_t)b * 3 * K * P, *M = a.tkp + (size_t)b * 3 * K, *cam = a.tlast + (size_t)b * 3;
    double s, ds;
    softplus_d((double)cam[0], s, ds);
    const double cxy[2] = {(double)cam[1], (double)cam[2]};
    double d = 0.0;
    for (int r = 0; r < 2 * K; ++r) {
      double wr, res;
      lm_kp2d_row(M, tg, wt, s, cxy, robust, s2, r >> 1, r & 1, wr, res);
      if (!(wr > 0.0)) continue;
      const double x = lm_kp2d_entry<true>(J, M, P, oc, r >> 1, r & 1, t, s, ds, cxy);
      d += (wr * x) * x;
    }
    dg[t] = d;
  }
  __syncthreads();
  if (t == 0) {
    double m = kDiagFloor;
    for (int j = 0; j < oc + 3; ++j) m = fmax(m, dg[j]);
    scr[kScrDmax] = m;
  }
  if (t < ns) scr[kScrDiag + t] = dg[oc + 3 + t];
}

template <bool SHARE>
__global__ void __launch_bounds__(kLmKpThreads, 2) lm_kp2dg_image_kernel(LmKpArgs a, LmKp2dArgs x2, LmGroupArgs gr) {
  extern __shared__ double A[];         // [P][P]: the lower triangle of the image's normal matrix, then its factor
  __shared__ double Js[kLmKpRows][kLmKpMaxP], WJs[kLmKpRows][kLmKpMaxP];   // staged rows J_r and w J_r
  __shared__ double rs[kLmKpRows], ws[kLmKpRows], y[kLmKpMaxP];
  __shared__ float lam_s;
  __shared__ int accept_s, ok_s;
  const int b = blockIdx.x, t = threadIdx.x, P = a.P, K = a.K, R3 = 3 * a.K, nr9 = 9 * a.n_rot;
  const int o = 3 * a.n_rot, oc = SHARE ? 3 : o, n1 = oc + 3;  // first camera and first shared column
  const int ns = SHARE ? P - n1 : a.nb;                         // the shared columns
  const float *tg = a.targets + (size_t)b * 2 * K, *wt = a.weights + (size_t)b * K;
  const float *anc = x2.anchor ? x2.anchor + (size_t)b * nr9 : nullptr;
  const bool robust = isfinite(x2.sigma);
  const double s2 = (double)x2.sigma * (double)x2.sigma;
  // 2. the group's decision
  if (t == 0) {
    const LmGroupDecision d = lm_group_decide<SHARE>(a, x2, gr, lm_group_of(gr, b));
    accept_s = d.accept;
    lam_s = d.lam;
    ok_s = 1;
  }
  __syncthreads();
  const bool accept = accept_s;
  const float *J = (accept ? a.tjac : a.jac) + (size_t)b * R3 * P;
  const float *M = (accept ? a.tkp : a.kp) + (size_t)b * R3;
  const float *Rst = (accept ? a.trot : a.rot) + (size_t)b * nr9;
  const float *Cst = (accept ? a.tlast : a.last) + (size_t)b * 3;
  if (accept) lm_kp_take_trial(a, b, 0.f, false);
  double s, ds;
  softplus_d((double)Cst[0], s, ds);
  const double cxy[2] = {(double)Cst[1], (double)Cst[2]};
  // 3. the image's normal equations, columns [delta | c | beta] (SHARE: [delta_0 | c | delta_1 .. | beta], no prior)
  int pr[kLmKpPairs], pc[kLmKpPairs];
  double acc[kLmKpPairs], g = 0.0;
  lm_kp_pairs(P, pr, pc, acc);
  lm_kp2d_keypoint_rows<true>(K, P, J, M, tg, wt, s, ds, cxy, robust, s2, oc, Js, WJs, ws, rs, pr, pc, acc, g);
  if constexpr (!SHARE) lm_kp2d_prior_rows(x2, o, Rst, anc, pr, pc, acc, g);
  lm_kp_store(P, A, y, pr, pc, acc, g);
  if (t == 0)
    for (int j = 0; j < n1; ++j) A[j * P + j] += (double)lam_s;
  // 4. the leading block factored alone: S_i in the trailing block, -s_i in y's tail, -x_i in y's head
  lm_kp_solve(A, y, P, n1, ok_s);
  lm_kp_solve_rows(A, P, n1, ns);       // X_i = A_i^-1 B_i
  double *scr = gr.scr + (size_t)b * gr.stride;
  double *S = scr + kScrDiag + ns, *sv = S + ns * ns, *X = sv + ns, *xv = X + n1 * ns;
  for (int q = t; q < ns * ns; q += blockDim.x) {
    const int r = q / ns, c = q % ns;
    S[q] = c <= r ? A[(n1 + r) * P + n1 + c] : 0.0;
  }
  for (int l = t; l < ns; l += blockDim.x) sv[l] = -y[n1 + l];
  for (int q = t; q < n1 * ns; q += blockDim.x) X[q] = A[(n1 + q % ns) * P + q / ns];
  for (int j = t; j < n1; j += blockDim.x) xv[j] = -y[j];
  if (t == 0) scr[kScrOk] = ok_s ? 1.0 : 0.0;
}

template <bool SHARE>
__global__ void __launch_bounds__(kLmKpThreads) lm_kp2dg_group_kernel(LmKpArgs a, LmKp2dArgs x2, LmGroupArgs gr) {
  extern __shared__ double A[];         // [ns][ns]: S + the prior and measurement rows, then its factor; then delta_i (n1)
  __shared__ double Js[kLmKpRows][kLmKpMaxP], WJs[kLmKpRows][kLmKpMaxP];   // the staged measurement rows
  __shared__ double rs[kLmKpRows], ws[kLmKpRows], y[kLmKpMaxP];
  __shared__ float lam_s;
  __shared__ int accept_s, ok_s;
  const int g = blockIdx.x, t = threadIdx.x, nb = a.nb, o = 3 * a.n_rot, nr9 = 9 * a.n_rot;
  const int oc = SHARE ? 3 : o, n1 = oc + 3;           // the image block: [delta | c] (SHARE: [delta_0 | c])
  const int ob = SHARE ? o - 3 : 0, ns = ob + nb;      // the shared block's first betas column and its size
  const int i0 = gr.off[g], i1 = gr.off[g + 1];
  const LmMeasArgs &mb = x2.mb;
  if (t == 0) {
    const LmGroupDecision d = lm_group_commit<SHARE>(a, x2, gr, g);
    accept_s = d.accept;
    lam_s = d.lam;
    bool ok = isfinite(d.lnew);         // a group without a finite loss does not move, nor one with a failed block
    for (int i = i0; i < i1; ++i) ok = ok && gr.scr[(size_t)i * gr.stride + kScrOk] != 0.0;
    ok_s = ok;
  }
  __syncthreads();
  const bool accept = accept_s;
  const float *Bst = (accept ? a.tbetas : a.betas) + (size_t)g * nb;
  if (accept) {
    for (int l = t; l < nb; l += blockDim.x) a.betas[(size_t)g * nb + l] = a.tbetas[(size_t)g * nb + l];
    if (mb.weights) lm_meas_take_trial(mb, g, nb);
  }
  // S = sum_i S_i, s = sum_i s_i in image order, then (SHARE) the pose-prior rows, the measurement rows and betas_w beta
  int pr[kLmKpPairs], pc[kLmKpPairs];
  double acc[kLmKpPairs], gs = 0.0;
  lm_kp_pairs(ns, pr, pc, acc);
  for (int i = i0; i < i1; ++i) {
    const double *S = gr.scr + (size_t)i * gr.stride + kScrDiag + ns;
#pragma unroll
    for (int q = 0; q < kLmKpPairs; ++q)
      if (pr[q] >= 0) acc[q] += S[pr[q] * ns + pc[q]];
    if (t < ns) gs += S[ns * ns + t];
  }
  // the group's state rotations are its first image's rows, which launch 2 updated on accept
  if constexpr (SHARE)
    lm_kp2d_prior_rows<3>(x2, o, a.rot + (size_t)i0 * nr9, x2.anchor ? x2.anchor + (size_t)g * nr9 : nullptr, pr, pc,
                          acc, gs);
  if (mb.weights)
    lm_meas_add_rows(mb, g, nb, ob, (accept ? mb.tmeas : mb.meas) + (size_t)g * 5,
                     (accept ? mb.tjac : mb.jac) + (size_t)g * 5 * nb, Js, WJs, ws, rs, pr, pc, acc, gs);
  if (x2.betas_w > 0.f && (SHARE ? t >= ob && t < ns : t < nb)) gs += (double)x2.betas_w * (double)Bst[t - ob];
  lm_kp_store(ns, A, y, pr, pc, acc, gs);
  if (t == 0) {
    const double damp = (double)x2.betas_w + (double)lam_s;
    for (int j = 0; j < ns; ++j) A[j * ns + j] += SHARE && j < ob ? (double)lam_s : damp;
  }
  lm_kp_solve(A, y, ns, ns, ok_s);
  const bool ok = ok_s;
  // the next trial of every image: delta_i = -x_i - X_i dshared, then R Exp(delta), c + delta_c, beta + dbeta; SHARE:
  // R_j Exp(dshared_j) of the group's rotations (its first image's) into every image's rows, j >= 1
  double *dv = A + ns * ns;
  for (int i = i0; i < i1; ++i) {
    const double *X = gr.scr + (size_t)i * gr.stride + kScrDiag + 2 * ns + ns * ns, *xv = X + n1 * ns;
    for (int j = t; j < n1; j += blockDim.x) {
      double v = -xv[j];
      for (int l = 0; l < ns; ++l) v -= X[j * ns + l] * y[l];
      dv[j] = v;
    }
    __syncthreads();
    for (int j = t; j < a.n_rot; j += blockDim.x) {
      float *Rt = a.trot + (size_t)i * nr9 + 9 * j;
      if (SHARE && j > 0)                 // a shared rotation: the group's, from its first image's rows
        lm_rot_next(a.rot + (size_t)i0 * nr9 + 9 * j, y + 3 * j - 3, ok, Rt);
      else
        lm_rot_next(a.rot + (size_t)i * nr9 + 9 * j, dv + 3 * j, ok, Rt);
    }
    if (t < 3) {
      const float x = a.last[(size_t)i * 3 + t];
      a.tlast[(size_t)i * 3 + t] = ok ? (float)((double)x + dv[oc + t]) : x;
    }
    for (int l = t; l < nb; l += blockDim.x)
      gr.tbetas_img[(size_t)i * nb + l] = ok ? (float)((double)Bst[l] + y[ob + l]) : Bst[l];
    __syncthreads();
  }
  for (int l = t; l < nb; l += blockDim.x) {
    const float x = Bst[l];
    a.tbetas[(size_t)g * nb + l] = ok ? (float)((double)x + y[ob + l]) : x;
  }
}

// The grouped entries' checks (check_lm_kp's, then the offsets, read on the host) and the three launches; the offsets
// are copied into the workspace on the stream.  SHARE: the shared-pose entries, with the group anchor; `meas`: the
// _measurements_ entries
template <bool SHARE>
int run_lm_kp2dg(const char *fn, int batch, int G, const int32_t *offsets, LmKpArgs a, LmKp2dArgs x,
                 float *tbetas_img, void *workspace, bool meas, void *stream) {
  const int rc = check_lm_kp(fn, batch, a, lm_kp2d_ptrs(x, meas) && offsets && tbetas_img && workspace,
                             lm_kp2d_factors_ok(x), kLmKp2dFactors);
  if (rc != SHAPY_OK) return rc;
  const int orc = put_group_offsets(fn, "group_offsets", batch, G, offsets, workspace, stream);
  if (orc != SHAPY_OK || batch == 0) return orc;
  const int n1 = SHARE ? 6 : 3 * a.n_rot + 3, ns = a.P - n1;
  LmGroupArgs gr{G, (int *)workspace, (double *)((char *)workspace + lm_group_offsets_bytes(G)),
                 lm_group_stride(n1, ns), tbetas_img};
  const size_t smem = lm_kp_smem(a.P), smem3 = (size_t)(ns * ns + n1) * sizeof(double);
  int e = lm_launch(lm_kp2dg_loss_kernel<SHARE>, batch, 128, 0, stream, a, x, gr);
  if (e == SHAPY_OK) e = lm_launch(lm_kp2dg_image_kernel<SHARE>, batch, kLmKpThreads, smem, stream, a, x, gr);
  if (e == SHAPY_OK) e = lm_launch(lm_kp2dg_group_kernel<SHARE>, G, kLmKpThreads, smem3, stream, a, x, gr);
  return e;
}

// ---------------------------------------------------------------------------------------------------------------
// The calibrated step (shapy_fit_lm_keypoints_2d_calibrated_step, and _measurements_ with MEAS): G bodies in one world
// frame, body g seen by the views [off[g], off[g + 1]) of a synchronised rig with known intrinsics (f_v, px_v, py_v) and
// world-to-camera extrinsics R_v, T_v (camera frame x right, y down, z forward).  One CTA per body, whose parameters are
// its world rotations, betas and world translation t, [delta | beta | t], P = 3 n_rot + NB + 3: the keypoint Jacobian
// is evaluated once per body whatever the number of views.  With X_k = kp_k + t and Y_vk = R_v X_k + T_v (fp64),
// p_vk = f_v (Y_x / Y_z, Y_y / Y_z) + pp_v, and per body, left to right:
//   L = sum_v (view order) [sum_{w_vk > 0} w_vk rho(|p_vk - x_vk|^2) (k order)]
//     + the 2D step's pose prior (against the body's anchor), measurement term (MEAS) and betas prior.
// Keypoint rows: view by view, rows 2k + c of each, weight w_vk q_vk^2 at the state, residual p_vkc - x_vkc, row
// u . J3_k with u = (f_v / Y_z) (R_v[c, :] - (Y_c / Y_z) R_v[2, :]) and J3_k the (3 x P) block of keypoint k (J_t = I:
// u itself on the t columns), staged kLmKpRows at a time (a block may straddle two views).  The prior, measurement and
// betas rows, the first lambda (the keypoint rows' diagonal), damping and solve are the 2D step's, the next trial the
// 3D step's.  Depth rule, per view: a trial with a weighted keypoint at Y_z <= 0 or non-finite in any view, or a view
// whose f is not finite and > 0, has loss +inf; a start that breaks it reports NaN and does not move.
struct LmKp2dCalibArgs : LmKp2dPerspArgs {    // targets (B, K, 2), weights (B, K) and intr (B, 3) per view
  const float *extr;                          // (B, 12) per view: R row-major, then T
  const int *off;                             // (G + 1) view offsets, the device copy in the workspace
};

template <bool MEAS>
__global__ void __launch_bounds__(kLmKpThreads, 2) lm_kp2dc_step_kernel(LmKpArgs a, LmKp2dCalibArgs x2) {
  extern __shared__ double A[];         // [P][P]: the lower triangle of the normal matrix, then its Cholesky factor
  __shared__ double Js[kLmKpRows][kLmKpMaxP], WJs[kLmKpRows][kLmKpMaxP];   // staged rows J_r and w J_r
  __shared__ double rs[kLmKpRows], ws[kLmKpRows], y[kLmKpMaxP], dg[kLmKpMaxP], fz[3 * kLmKpRows];
  __shared__ double lt_s;
  __shared__ int kr[kLmKpRows], ok_s;   // kr: the keypoint of each staged row
  const int b = blockIdx.x, t = threadIdx.x, P = a.P, K = a.K, R2 = 2 * a.K, R3 = 3 * a.K, nb = a.nb;
  const int nr9 = 9 * a.n_rot, o = 3 * a.n_rot, oc = o + nb;     // first betas and first t column
  const int v0 = x2.off[b], v1 = x2.off[b + 1];
  const float *anc = x2.anchor ? x2.anchor + (size_t)b * nr9 : nullptr;
  const bool robust = isfinite(x2.sigma);
  const double s2 = (double)x2.sigma * (double)x2.sigma;
  const float lcur = a.loss[b];
  // 1. trial loss: the keypoint term of each view, then the pose prior once
  if (t == 0) {
    LmKp2dArgs xk = x2;
    xk.pose_w = 0.f;
    double L = 0.0;
    for (int v = v0; v < v1; ++v) {
      const CalibCam tc = calib_cam(x2.intr + (size_t)v * 3, x2.extr + (size_t)v * 12, a.tlast + (size_t)b * 3);
      L += lm_kp2d_trial_loss<true>(a, xk, b, a.targets + (size_t)v * R2, a.weights + (size_t)v * K, nullptr, robust,
                                    s2, &tc);
    }
    if (x2.pose_w > 0.f) L += lm_kp2d_prior_loss(x2, a.trot + (size_t)b * nr9, anc, nr9);
    if constexpr (MEAS) L += lm_meas_loss(x2.mb, b);
    if (x2.betas_w > 0.f) L += (double)x2.betas_w * lm_sq_norm(a.tbetas + (size_t)b * nb, nb);
    lt_s = L;
  }
  __syncthreads();
  // 2. accept or reject
  const double lt = lt_s;
  const bool accept = lm_accept(a.first, lt, lcur);
  const float lnew = lm_loss(accept, lt, lcur);
  const float *J = (accept ? a.tjac : a.jac) + (size_t)b * R3 * P;
  const float *M = (accept ? a.tkp : a.kp) + (size_t)b * R3;
  const float *Rst = (accept ? a.trot : a.rot) + (size_t)b * nr9;
  const float *Bst = (accept ? a.tbetas : a.betas) + (size_t)b * nb;
  const float *Tst = (accept ? a.tlast : a.last) + (size_t)b * 3;
  if (accept) {
    lm_kp_take_trial(a, b, lnew);
    if constexpr (MEAS) lm_meas_take_trial(x2.mb, b, nb);
  }
  // 3. normal equations: the keypoint rows of the views in order, rows 2k + c of each
  int pr[kLmKpPairs], pc[kLmKpPairs];
  double acc[kLmKpPairs], g = 0.0;
  lm_kp_pairs(P, pr, pc, acc);
  const double cxy[2] = {0.0, 0.0};     // the weak-perspective camera of lm_kp2d_row / lm_kp2d_entry: not read
  const int nrows = (v1 - v0) * R2;
  for (int r0 = 0; r0 < nrows; r0 += kLmKpRows) {
    const int nr = min(kLmKpRows, nrows - r0);
    __syncthreads();
    for (int i = t; i < nr; i += blockDim.x) {   // row weight (IRLS at the state), residual and factors
      const int v = v0 + (r0 + i) / R2, q = (r0 + i) % R2;
      const CalibCam sc = calib_cam(x2.intr + (size_t)v * 3, x2.extr + (size_t)v * 12, Tst);
      double wr, res;
      lm_kp2d_row<true>(M, a.targets + (size_t)v * R2, a.weights + (size_t)v * K, 0.0, cxy, robust, s2, q >> 1, q & 1,
                        wr, res, &sc, fz + 3 * i);
      ws[i] = wr;
      rs[i] = res;
      kr[i] = q >> 1;
    }
    __syncthreads();
    for (int i = t; i < nr * P; i += blockDim.x) {
      const int row = i / P, col = i % P;
      const double wr = ws[row];
      if (wr > 0.0) {                    // a dropped keypoint's rows are never read: they may be NaN
        const double x = lm_kp2d_entry<false, true, CalibCam>(J, M, P, oc, kr[row], 0, col, 0.0, 0.0, cxy,
                                                              fz + 3 * row);
        Js[row][col] = x;
        WJs[row][col] = wr * x;
      }
    }
    __syncthreads();
    lm_kp_add_rows(nr, P, Js, WJs, ws, rs, pr, pc, acc, g);
  }
#pragma unroll
  for (int i = 0; i < kLmKpPairs; ++i)
    if (pr[i] >= 0 && pr[i] == pc[i]) dg[pr[i]] = acc[i];     // the diagonal of the keypoint rows: the first lambda
  lm_kp2d_prior_rows(x2, o, Rst, anc, pr, pc, acc, g);
  if constexpr (MEAS)
    lm_meas_add_rows(x2.mb, b, nb, o, (accept ? x2.mb.tmeas : x2.mb.meas) + (size_t)b * 5,
                     (accept ? x2.mb.tjac : x2.mb.jac) + (size_t)b * 5 * nb, Js, WJs, ws, rs, pr, pc, acc, g);
  if (x2.betas_w > 0.f && t >= o && t < oc) g += (double)x2.betas_w * (double)Bst[t - o];
  lm_kp_damp(a, b, accept, lnew, A, y, pr, pc, acc, g, dg, 1, o, oc, x2.betas_w, ok_s);
  // 4. Cholesky and the two triangular solves
  lm_kp_solve(A, y, P, P, ok_s);
  // 5. next trial (ok is uniform: every thread reads it after the last barrier); a failed step keeps the state
  lm_kp_next_trial(a, b, y, ok_s);
}

// The calibrated entries' checks (check_lm_kp's over the G bodies, then the view offsets, read on the host) and the
// launch; the offsets are copied into the workspace on the stream
template <bool MEAS>
int run_lm_kp2dc(const char *fn, int views, int G, const int32_t *offsets, LmKpArgs a, LmKp2dCalibArgs x,
                 void *workspace, void *stream) {
  const int rc = check_lm_kp(fn, G, a, lm_kp2d_ptrs(x, MEAS) && offsets && x.intr && x.extr && workspace,
                             lm_kp2d_factors_ok(x), kLmKp2dFactors);
  if (rc != SHAPY_OK) return rc;
  const int orc = put_group_offsets(fn, "view_offsets", views, G, offsets, workspace, stream);
  if (orc != SHAPY_OK || G == 0) return orc;
  x.off = (const int *)workspace;
  return lm_launch(lm_kp2dc_step_kernel<MEAS>, G, kLmKpThreads, lm_kp_smem(a.P), stream, a, x);
}

// ---------------------------------------------------------------------------------------------------------------
// The sequence step (shapy_fit_lm_keypoints_2d_sequence_step): the frames [off[s], off[s + 1]) of sequence s are one
// person filmed by one camera, in time order.  Frame t keeps its rotations R_t,j and camera-frame translation tau_t
// (n1 = 3 n_rot + 3 columns [delta | tau]) and projects as the perspective step does with its own intrinsics; the
// sequence shares one beta.  Per sequence, in fp64, left to right:
//   L_s = sum_t (frame order) [the perspective step's keypoint term + pose prior of frame t
//                              + 1/2 srot_w sum_{j >= 0} |R_{t+1},j - R_t,j|_F^2 (j order, row-major entries)
//                              + stransl_w |tau_{t+1} - tau_t|^2]  (the last two when t + 1 is in s and the weight > 0)
//       + betas_w |beta|^2.
// The smoothness rows of the pair (t, t + 1) are the pose prior's rows with the anchor replaced by the neighbour: weight
// srot_w / 2, residual R_{t+1},j - R_t,j, Jacobian -R_t,j [e_a]x on frame t's column 3 j + a and +R_{t+1},j [e_a]x on
// frame t + 1's; then weight stransl_w, residual tau_{t+1} - tau_t, Jacobian -I and +I.  The normal matrix of a sequence
// is block tridiagonal in its frames with an arrow of betas columns: the diagonal block D_t, the coupling B_t of frame
// t with beta, and C_t, the block of frame t + 1's rows and frame t's columns, block diagonal: per joint -srot_w / 2
// D_{t+1},j^T D_t,j (D = the 9 x 3 tangent rows), and -stransl_w I on tau.  Three launches after the keypoint Jacobian:
//   1. lm_kp2ds_loss_kernel, per frame: the bracket of the trial's loss into its scratch and, on the first step, the
//      diagonal of its keypoint rows (lm_kp2dg_loss_kernel's slots), so that lm_group_decide<false> decides unchanged;
//   2. lm_kp2ds_frame_kernel, per frame: the decision of its sequence (lm_group_of), on accept the frame's trial
//      becomes its state; the perspective keypoint rows in the column order [delta | tau | beta], the pose-prior rows,
//      then the diagonal blocks and gradient of the smoothness rows of the previous and the next frame (a neighbour read
//      as accept ? trial : state, neither written during the launch); A_t (P x P lower) and -g_t into the frame's
//      scratch;
//   3. lm_kp2ds_sequence_kernel, per sequence: the decision recorded in the sequence's state (lm_group_commit), then a
//      block LDL^T sweep over its frames (block Thomas, the arrow carried along): with Dt_0 = D_0 + lambda I,
//        Dt_t = D_t + lambda I - C_{t-1} Dt_{t-1}^-1 C_{t-1}^T,  Bt_t = B_t - C_{t-1} Dt_{t-1}^-1 Bt_{t-1},
//        rt_t = -g_t - C_{t-1} Dt_{t-1}^-1 rt_{t-1},  Et = E - sum_t Bt_t^T Dt_t^-1 Bt_t,  et = -g_beta - sum_t ...,
//      each frame's [Dt_t | Bt_t] factored by lm_kp_solve with n = n1 in shared memory (the trailing block carries Et),
//      then X_t = Dt_t^-1 Bt_t (lm_kp_solve_rows), Y_t = Dt_t^-1 C_t^T and y_t = Dt_t^-1 rt_t into the frame's
//      scratch; Et (+ betas_w + lambda on its diagonal) dbeta = et - betas_w beta; from the last frame back, x_t = y_t -
//      X_t dbeta - Y_t x_{t+1} and the next trial R Exp(delta) (lm_rot_next), tau + dtau, beta + dbeta (trial betas
//      per sequence and per frame).
// The policy is the grouped step's per sequence: one decision, lambda, loss and accept count, the first lambda from the
// diagonal of the keypoint rows (per frame on [delta | tau], summed over the frames on beta); a sequence whose loss is
// not finite or one of whose pivots fails keeps its state.  Depth rule per frame, as the perspective step's: a trial
// with a weighted keypoint at Y_z <= 0 or a bad f in any frame gives the sequence a loss of +inf.  No atomics; a
// sequence's bits do not depend on the rest of the batch.  A sequence of one frame has the perspective step's loss,
// lambda and decision bit for bit.
struct LmKp2dSeqArgs : LmKp2dPerspArgs {     // intr (B, 3) per frame
  float srot_w, stransl_w;                   // the smoothness weights
};

// A frame's scratch: lm_group_decide's slots (kScrLoss, kScrDmax, then the nb betas diagonal entries), then A_t (P x P,
// lower), -g_t (P), and from launch 3 y_t (n1), X_t (nb x n1, beta-major) and Y_t^T (n1 x n1, row k = column k of Y_t)
constexpr int kSeqA = kScrDiag;               // + nb
__host__ __device__ inline int lm_seq_stride(int n1, int nb) {
  const int P = n1 + nb;
  return kSeqA + nb + P * P + P + n1 + nb * n1 + n1 * n1;
}

// Phase 1: the smoothness term of the pair (b, b + 1) of the trial, rotations then translation
__device__ __forceinline__ double lm_seq_smooth_loss(const LmKpArgs &a, const LmKp2dSeqArgs &x2, int b) {
  const int nr9 = 9 * a.n_rot;
  double L = 0.0;
  if (x2.srot_w > 0.f) {
    const float *r0 = a.trot + (size_t)b * nr9, *r1 = r0 + nr9;
    double q = 0.0;
    for (int i = 0; i < nr9; ++i) {
      const double d = (double)r1[i] - (double)r0[i];
      q += d * d;
    }
    L += 0.5 * (double)x2.srot_w * q;
  }
  if (x2.stransl_w > 0.f) {
    const float *t0 = a.tlast + (size_t)b * 3;
    double q = 0.0;
    for (int c = 0; c < 3; ++c) {
      const double d = (double)t0[3 + c] - (double)t0[c];
      q += d * d;
    }
    L += (double)x2.stransl_w * q;
  }
  return L;
}

// Phase 3: the smoothness rows of the pair of frame b (rotations R, translation T) and one neighbour (Rn, Tn), on b's
// columns [delta | tau]: the diagonal blocks srot_w / 2 D_j^T D_j and stransl_w I, the gradient srot_w / 2 D_j^T (R_j -
// Rn_j) and stransl_w (T - Tn)
__device__ __forceinline__ void lm_seq_smooth_rows(const LmKp2dSeqArgs &x2, int o, const float *R, const float *Rn,
                                                   const float *T, const float *Tn, const int (&pr)[kLmKpPairs],
                                                   const int (&pc)[kLmKpPairs], double (&acc)[kLmKpPairs], double &g) {
  const int t = threadIdx.x;
  if (x2.srot_w > 0.f) {
    const double hw = 0.5 * (double)x2.srot_w;
#pragma unroll
    for (int i = 0; i < kLmKpPairs; ++i) {
      if (pr[i] >= 0 && pr[i] < o && pc[i] / 3 == pr[i] / 3) {
        const float *Rj = R + 9 * (pr[i] / 3);
        for (int e = 0; e < 9; ++e) acc[i] += (hw * rot_tangent(Rj, pr[i] % 3, e)) * rot_tangent(Rj, pc[i] % 3, e);
      }
    }
    if (t < o) {
      const float *Rj = R + 9 * (t / 3), *Nj = Rn + 9 * (t / 3);
      for (int e = 0; e < 9; ++e) g += (hw * rot_tangent(Rj, t % 3, e)) * ((double)Rj[e] - (double)Nj[e]);
    }
  }
  if (x2.stransl_w > 0.f) {
    const double w = x2.stransl_w;
#pragma unroll
    for (int i = 0; i < kLmKpPairs; ++i)
      if (pr[i] >= o && pr[i] < o + 3 && pc[i] == pr[i]) acc[i] += w;
    if (t >= o && t < o + 3) g += w * ((double)T[t - o] - (double)Tn[t - o]);
  }
}

__global__ void __launch_bounds__(128) lm_kp2ds_loss_kernel(LmKpArgs a, LmKp2dSeqArgs x2, LmGroupArgs gr) {
  __shared__ double dg[kLmKpMaxP];
  const int b = blockIdx.x, t = threadIdx.x, P = a.P, K = a.K, nb = a.nb, n1 = 3 * a.n_rot + 3;
  const float *tg = a.targets + (size_t)b * 2 * K, *wt = a.weights + (size_t)b * K;
  const float *anc = x2.anchor ? x2.anchor + (size_t)b * 9 * a.n_rot : nullptr;
  const bool robust = isfinite(x2.sigma);
  const double s2 = (double)x2.sigma * (double)x2.sigma;
  double *scr = gr.scr + (size_t)b * gr.stride;
  const PerspCam tc = persp_cam(x2.intr + (size_t)b * 3, a.tlast + (size_t)b * 3);
  if (t == 0) {
    double L = lm_kp2d_trial_loss<true>(a, x2, b, tg, wt, anc, robust, s2, &tc);
    if (b + 1 < gr.off[lm_group_of(gr, b) + 1]) L += lm_seq_smooth_loss(a, x2, b);
    scr[kScrLoss] = L;
  }
  if (!a.first) return;
  // the first step accepts: the diagonal of the trial's keypoint rows, column t of [delta | tau | beta], in row order
  if (t < P) {
    const float *J = a.tjac + (size_t)b * 3 * K * P, *M = a.tkp + (size_t)b * 3 * K;
    const double cxy[2] = {0.0, 0.0};   // the weak-perspective camera of lm_kp2d_row / lm_kp2d_entry: not read
    double d = 0.0;
    for (int r = 0; r < 2 * K; ++r) {
      double wr, res, fz[2];
      lm_kp2d_row<true>(M, tg, wt, 0.0, cxy, robust, s2, r >> 1, r & 1, wr, res, &tc, fz);
      if (!(wr > 0.0)) continue;
      const double x = lm_kp2d_entry<true, true>(J, M, P, n1 - 3, r >> 1, r & 1, t, 0.0, 0.0, cxy, fz);
      d += (wr * x) * x;
    }
    dg[t] = d;
  }
  __syncthreads();
  if (t == 0) {
    double m = kDiagFloor;
    for (int j = 0; j < n1; ++j) m = fmax(m, dg[j]);
    scr[kScrDmax] = m;
  }
  if (t < nb) scr[kScrDiag + t] = dg[n1 + t];
}

__global__ void __launch_bounds__(kLmKpThreads, 2) lm_kp2ds_frame_kernel(LmKpArgs a, LmKp2dSeqArgs x2, LmGroupArgs gr) {
  __shared__ double Js[kLmKpRows][kLmKpMaxP], WJs[kLmKpRows][kLmKpMaxP];   // staged rows J_r and w J_r
  __shared__ double rs[kLmKpRows], ws[kLmKpRows];
  __shared__ int accept_s, prev_s, next_s;
  const int b = blockIdx.x, t = threadIdx.x, P = a.P, K = a.K, R3 = 3 * a.K, nr9 = 9 * a.n_rot, o = 3 * a.n_rot;
  const float *tg = a.targets + (size_t)b * 2 * K, *wt = a.weights + (size_t)b * K;
  const float *anc = x2.anchor ? x2.anchor + (size_t)b * nr9 : nullptr;
  const bool robust = isfinite(x2.sigma);
  const double s2 = (double)x2.sigma * (double)x2.sigma;
  // 2. the sequence's decision
  if (t == 0) {
    const int s = lm_group_of(gr, b);
    accept_s = lm_group_decide<false>(a, x2, gr, s).accept;
    prev_s = b > gr.off[s];
    next_s = b + 1 < gr.off[s + 1];
  }
  __syncthreads();
  const bool accept = accept_s;
  const float *J = (accept ? a.tjac : a.jac) + (size_t)b * R3 * P;
  const float *M = (accept ? a.tkp : a.kp) + (size_t)b * R3;
  const float *Rs = accept ? a.trot : a.rot, *Ts = accept ? a.tlast : a.last;   // every frame of the sequence's state
  const float *Rst = Rs + (size_t)b * nr9, *Tst = Ts + (size_t)b * 3;
  if (accept) lm_kp_take_trial(a, b, 0.f, false);
  // 3. the frame's rows, columns [delta | tau | beta]
  int pr[kLmKpPairs], pc[kLmKpPairs];
  double acc[kLmKpPairs], g = 0.0;
  lm_kp_pairs(P, pr, pc, acc);
  const double cxy[2] = {0.0, 0.0};     // the weak-perspective camera of lm_kp2d_row / lm_kp2d_entry: not read
  const PerspCam sc = persp_cam(x2.intr + (size_t)b * 3, Tst);
  lm_kp2d_keypoint_rows<true, true>(K, P, J, M, tg, wt, 0.0, 0.0, cxy, robust, s2, o, Js, WJs, ws, rs, pr, pc, acc, g,
                                    &sc);
  lm_kp2d_prior_rows(x2, o, Rst, anc, pr, pc, acc, g);
  if (prev_s) lm_seq_smooth_rows(x2, o, Rst, Rst - nr9, Tst, Tst - 3, pr, pc, acc, g);
  if (next_s) lm_seq_smooth_rows(x2, o, Rst, Rst + nr9, Tst, Tst + 3, pr, pc, acc, g);
  double *At = gr.scr + (size_t)b * gr.stride + kSeqA + a.nb;
  lm_kp_store(P, At, At + P * P, pr, pc, acc, g);
}

__global__ void __launch_bounds__(kLmKpThreads) lm_kp2ds_sequence_kernel(LmKpArgs a, LmKp2dSeqArgs x2,
                                                                          LmGroupArgs gr) {
  extern __shared__ double S[];         // [P][P]: [Dt_t | Bt_t^T ; Et] lower, then its partial factor; then [n1][n1]: Y_t
  __shared__ double y[kLmKpMaxP], xs[2][kLmKpMaxP], db[kLmKpMaxP], Cs[kLmKpMaxP][3];   // Cs: row k of C_t, its block
  __shared__ float lam_s;
  __shared__ int accept_s, ok_s;
  const int s = blockIdx.x, t = threadIdx.x, P = a.P, nb = a.nb, o = 3 * a.n_rot, n1 = o + 3, nr9 = 9 * a.n_rot;
  const int i0 = gr.off[s], i1 = gr.off[s + 1];
  double *Ys = S + P * P;
  if (t == 0) {
    const LmGroupDecision d = lm_group_commit<false>(a, x2, gr, s);
    accept_s = d.accept;
    lam_s = d.lam;
    ok_s = isfinite(d.lnew);            // a sequence without a finite loss does not move, nor one with a failed pivot
  }
  __syncthreads();
  const bool accept = accept_s;
  const double lam = (double)lam_s;
  const float *Bst = (accept ? a.tbetas : a.betas) + (size_t)s * nb;
  if (accept)
    for (int l = t; l < nb; l += blockDim.x) a.betas[(size_t)s * nb + l] = a.tbetas[(size_t)s * nb + l];
  // the forward sweep
  for (int i = i0; i < i1; ++i) {
    double *scr = gr.scr + (size_t)i * gr.stride;
    const double *Ai = scr + kSeqA + nb, *gi = Ai + P * P;
    const double *pv = scr - gr.stride + kSeqA + nb + P * P + P;   // the previous frame's y, X, (Y in shared memory)
    const double *yp = pv, *Xp = pv + n1;
    const bool more = i > i0;
    for (int q = t; q < P * P; q += blockDim.x) {
      const int r = q / P, c = q % P;
      if (c > r) continue;
      double v = Ai[q];
      if (r < n1) {                     // Dt_t: D_t + lambda I - C_{t-1} Y_{t-1}
        if (r == c) v += lam;
        if (more) {
          const int m0 = 3 * (r / 3);
          for (int m = 0; m < 3; ++m) v -= Cs[r][m] * Ys[(m0 + m) * n1 + c];
        }
        S[q] = v;
      } else if (c < n1) {              // Bt_t^T: B_t^T - (C_{t-1} X_{t-1})^T
        if (more) {
          const int m0 = 3 * (c / 3);
          for (int m = 0; m < 3; ++m) v -= Cs[c][m] * Xp[(r - n1) * n1 + m0 + m];
        }
        S[q] = v;
      } else {                          // E, summed in frame order under the Schur updates so far
        S[q] = more ? S[q] + v : v;
      }
    }
    for (int j = t; j < P; j += blockDim.x) {
      double v = gi[j];
      if (j < n1) {
        if (more) {
          const int m0 = 3 * (j / 3);
          for (int m = 0; m < 3; ++m) v -= Cs[j][m] * yp[m0 + m];
        }
        y[j] = v;
      } else {
        y[j] = more ? y[j] + v : v;
      }
    }
    // Dt_t factored: the trailing block becomes Et - Bt_t^T Dt_t^-1 Bt_t, y's tail et - Bt_t^T Dt_t^-1 rt_t, y's head
    // Dt_t^-1 rt_t (lm_kp_solve starts with a barrier)
    lm_kp_solve(S, y, P, n1, ok_s);
    lm_kp_solve_rows(S, P, n1, nb);     // X_t = Dt_t^-1 Bt_t
    double *yo = scr + kSeqA + nb + P * P + P, *Xo = yo + n1, *Yo = Xo + nb * n1;
    for (int j = t; j < n1; j += blockDim.x) yo[j] = y[j];
    for (int q = t; q < nb * n1; q += blockDim.x) Xo[q] = S[(n1 + q / n1) * P + q % n1];
    if (i + 1 < i1) {
      // C_t from the state rotations of frames t and t + 1 (launch 2 made an accepted trial the state)
      for (int k = t; k < n1; k += blockDim.x) {
        for (int m = 0; m < 3; ++m) {
          double v = 0.0;
          if (k < o) {
            if (x2.srot_w > 0.f) {
              const double hw = 0.5 * (double)x2.srot_w;
              const float *Rn = a.rot + (size_t)(i + 1) * nr9 + 9 * (k / 3), *Rc = a.rot + (size_t)i * nr9 + 9 * (k / 3);
              for (int e = 0; e < 9; ++e) v += (hw * rot_tangent(Rn, k % 3, e)) * rot_tangent(Rc, m, e);
            }
          } else if (m == k - o) {
            v = (double)x2.stransl_w;
          }
          Cs[k][m] = -v;
        }
      }
      __syncthreads();
      // Y_t = Dt_t^-1 C_t^T: C_t^T into Ys (row m, column k), then L z = C^T and L^T Y = z, each row scaled by its
      // pivot after the elimination.  Column k of C_t^T is zero above its block, and stays so under L^-1
      for (int q = t; q < n1 * n1; q += blockDim.x) {
        const int m = q / n1, k = q % n1;
        Ys[q] = m / 3 == k / 3 ? Cs[k][m % 3] : 0.0;
      }
      __syncthreads();
      for (int j = 0; j < n1; ++j) {
        const int kmax = 3 * (j / 3) + 3, rows = n1 - j - 1;
        for (int q = t; q < rows * kmax; q += blockDim.x) {
          const int r = j + 1 + q / kmax, k = q % kmax;
          Ys[r * n1 + k] -= (S[r * P + j] / S[j * P + j]) * Ys[j * n1 + k];
        }
        __syncthreads();
      }
      for (int q = t; q < n1 * n1; q += blockDim.x) Ys[q] /= S[(q / n1) * P + q / n1];
      __syncthreads();
      for (int j = n1 - 1; j > 0; --j) {
        for (int q = t; q < j * n1; q += blockDim.x) {
          const int r = q / n1, k = q % n1;
          Ys[r * n1 + k] -= (S[j * P + r] / S[j * P + j]) * Ys[j * n1 + k];
        }
        __syncthreads();
      }
      for (int q = t; q < n1 * n1; q += blockDim.x) Ys[q] /= S[(q / n1) * P + q / n1];
      __syncthreads();
      for (int q = t; q < n1 * n1; q += blockDim.x) Yo[q] = Ys[(q % n1) * n1 + q / n1];
    }
    __syncthreads();
  }
  // Et dbeta = et: the trailing block, betas_w beta and the damping betas_w + lambda
  double *E = Ys;
  for (int q = t; q < nb * nb; q += blockDim.x) {
    const int r = q / nb, c = q % nb;
    E[q] = c <= r ? S[(n1 + r) * P + n1 + c] + (r == c ? (double)x2.betas_w + lam : 0.0) : 0.0;
  }
  for (int l = t; l < nb; l += blockDim.x)
    db[l] = x2.betas_w > 0.f ? y[n1 + l] - (double)x2.betas_w * (double)Bst[l] : y[n1 + l];
  lm_kp_solve(E, db, nb, nb, ok_s);
  const bool ok = ok_s;
  // the back-substitution from the last frame, and each frame's next trial
  for (int i = i1 - 1; i >= i0; --i) {
    const double *yo = gr.scr + (size_t)i * gr.stride + kSeqA + nb + P * P + P, *Xo = yo + n1, *Yo = Xo + nb * n1;
    double *xc = xs[i & 1];
    const double *xn = xs[(i + 1) & 1];
    for (int j = t; j < n1; j += blockDim.x) {
      double v = yo[j];
      for (int l = 0; l < nb; ++l) v -= Xo[l * n1 + j] * db[l];
      if (i + 1 < i1)
        for (int k = 0; k < n1; ++k) v -= Yo[k * n1 + j] * xn[k];
      xc[j] = v;
    }
    __syncthreads();
    for (int j = t; j < a.n_rot; j += blockDim.x)
      lm_rot_next(a.rot + (size_t)i * nr9 + 9 * j, xc + 3 * j, ok, a.trot + (size_t)i * nr9 + 9 * j);
    if (t < 3) {
      const float x = a.last[(size_t)i * 3 + t];
      a.tlast[(size_t)i * 3 + t] = ok ? (float)((double)x + xc[o + t]) : x;
    }
    for (int l = t; l < nb; l += blockDim.x)
      gr.tbetas_img[(size_t)i * nb + l] = ok ? (float)((double)Bst[l] + db[l]) : Bst[l];
  }
  for (int l = t; l < nb; l += blockDim.x) {
    const float x = Bst[l];
    a.tbetas[(size_t)s * nb + l] = ok ? (float)((double)x + db[l]) : x;
  }
}

// The sequence entry's checks (check_lm_kp's, the smoothness weights, then the offsets, read on the host) and the three
// launches; the offsets are copied into the workspace on the stream
int run_lm_kp2ds(const char *fn, int batch, int G, const int32_t *offsets, LmKpArgs a, LmKp2dSeqArgs x,
                 float *tbetas_img, void *workspace, void *stream) {
  const int rc = check_lm_kp(fn, batch, a, lm_kp2d_ptrs(x, false) && offsets && x.intr && tbetas_img && workspace,
                             lm_kp2d_factors_ok(x) && x.srot_w >= 0.f && isfinite(x.srot_w) && x.stransl_w >= 0.f &&
                                 isfinite(x.stransl_w),
                             "robust_sigma must be > 0 (inf: least squares), the prior weights >= 0, the smoothness "
                             "weights finite and >= 0 and lambda_up and lambda_down >= 1");
  if (rc != SHAPY_OK) return rc;
  const int orc = put_group_offsets(fn, "sequence_offsets", batch, G, offsets, workspace, stream);
  if (orc != SHAPY_OK || batch == 0) return orc;
  const int n1 = 3 * a.n_rot + 3;
  LmGroupArgs gr{G, (int *)workspace, (double *)((char *)workspace + lm_group_offsets_bytes(G)),
                 lm_seq_stride(n1, a.nb), tbetas_img};
  const int ny = n1 > a.nb ? n1 : a.nb;
  const size_t smem = (size_t)(a.P * a.P + ny * ny) * sizeof(double);
  int e = lm_launch(lm_kp2ds_loss_kernel, batch, 128, 0, stream, a, x, gr);
  if (e == SHAPY_OK) e = lm_launch(lm_kp2ds_frame_kernel, batch, kLmKpThreads, 0, stream, a, x, gr);
  if (e == SHAPY_OK) e = lm_launch(lm_kp2ds_sequence_kernel, G, kLmKpThreads, smem, stream, a, x, gr);
  return e;
}

// ---------------------------------------------------------------------------------------------------------------
// The single-image 2D step: pose, shape and camera of each body against its 2D keypoints, one body per CTA
// (shapy_fit_lm_keypoints_2d_step; _perspective_ with PERSP; _measurements_ with MEAS; the _expressive_ entries add the
// pose parts past the body and the facial expression of SMPL-X).  Parameters [delta_j (3 n_rot) | beta (nb) | psi (ne)
// | c or t], P = 3 n_rot + nb + ne + 3, the columns of shapy_smplx_keypoint_jacobian_expr (of
// shapy_smplx_keypoint_jacobian with ne = 0); the 22-joint entries have ne = 0 and P <= kLmKpMaxP, the expressive ones
// P <= kLmKp2dMaxP.  The weak-perspective camera c = (c0, c1, c2) takes the columns of transl (which a weak-perspective
// camera cannot see along z, and which duplicates c1, c2 in x and y).  With s = softplus(c0) (threshold 20, as the
// forward) the projection is p_k = s (kp_k,xy + (c1, c2)), and per body, in fp64, left to right:
//   L = sum_{w_k > 0} w_k rho(|p_k - x_k|^2)  (k order)
//     + 1/2 pose_w sum_{j >= 1} |R_j - R0_j|_F^2  (j order, row-major entries; when pose_w > 0)
//     + sum_{u_m > 0} u_m (t_m - meas_m)^2  (MEAS; m order, summed on its own)
//     + betas_w |beta|^2  (l order; when betas_w > 0) + expr_w |psi|^2  (l order; when expr_w > 0)
// rho(e) = e at sigma = inf, else e q with q = sigma^2 / (sigma^2 + e) (Geman-McClure).  With per-joint weights w_j
// (joint_w, n_rot entries, joint 0 not read) the pose prior is sum_{j >= 1, w_j > 0} (1/2 w_j) |R_j - R0_j|_F^2 in j
// order.  Rows of the normal equations, accumulated into A and g in this order:
//   keypoint rows 2k + c (c = 0 x, 1 y), weight w_k q_k^2 (the IRLS weight rho'(e_k), 1 at sigma = inf) at the state,
//     residual p_kc - x_kc, Jacobian staged from the 3D keypoint Jacobian (transl columns skipped): s J_{3k+c} on the
//     rotation, betas and expression columns, ds/dc0 (kp_kc + c_{1+c}) on c0, s on c_{1+c};
//   pose-prior rows (R_j - R0_j)_e, weight pose_w / 2 (w_j / 2), Jacobian R_j [e_a]x in column 3 j + a
//     (d(R Exp d) = R [d]x), j = 1 .. n_rot - 1, e in row-major order: they only reach the 3 x 3 diagonal block of
//     joint j;
//   MEAS: the five measurement rows (plain least squares: rho applies to keypoints only), residual meas_m - t_m, into
//     the betas block of A and g;
//   then g += betas_w beta on the betas columns and expr_w psi on the expression columns.
// The first lambda is 1e-3 max(diag A, 1e-6) of the keypoint rows alone; the diagonal then gets betas_w + lambda on the
// betas columns, expr_w + lambda on the expression columns and lambda elsewhere.  With every measurement weight <= 0
// the loss gains an exact 0 and no row is added, so the MEAS step equals the step without, bit for bit, for any sigma,
// pose prior and betas_w.
//
// PERSP: the projection of a pinhole camera of known intrinsics (f, px, py) per body: camera frame x right, y down, z
// forward, the last three parameters the translation t.  With Y_k = kp_k + t (fp64),
//   p_k = f (Y_k,x / Y_k,z, Y_k,y / Y_k,z) + (px, py);
// the loss is the weak-perspective one term for term with this p_k, and keypoint row 2k + c is (f / Y_z) (J_{3k+c} -
// (Y_c / Y_z) J_{3k+2}) on every column, J_t = I on the t columns.  Depth rule: a trial with a weighted keypoint at
// Y_z <= 0 or non-finite, or a body whose f is not finite and > 0, has loss +inf: it is rejected, and a start that
// breaks the rule reports NaN and does not move.  The other rows, lambda, damping, solve and next trial (t + delta_t)
// are the weak-perspective step's.
//
// One CTA of kLmKpThreads per body: the packed fp64 lower triangle of A (P (P + 1) / 2 entries, 160.8 KB at P = 200)
// and kLmKpRows staged rows of width P live in dynamic shared memory.  Each staged chunk is added into the shared
// triangle (thread t owns the packed entries t + 256 i, each entry summing its rows in row order), then the pose-prior
// and measurement rows into their blocks.  The Cholesky is right-looking (column j scaled, then the trailing triangle
// updated, one warp per trailing row), then L z = -g and L^T delta = z.
constexpr int kLmKp2dMaxP = 200;

struct LmKp2dStepArgs : LmKp2dPerspArgs {   // intr is null in the weak-perspective step
  const float *joint_w;                     // (n_rot) per-joint pose-prior weights, or null: pose_w for every joint
  float expr_w;
  int ne;
  float *expr, *texpr;                      // state and trial expression (B, ne); null when ne = 0
};

// dynamic shared memory of the 2D step, in doubles: the packed triangle, Js and WJs (kLmKpRows x P each), y, z, dg,
// the scaled column and the Cholesky diagonal (P each), ws and rs (kLmKpRows each)
__host__ __device__ inline size_t lm_kp2d_smem_doubles(int P) {
  return (size_t)P * (P + 1) / 2 + (size_t)2 * kLmKpRows * P + (size_t)5 * P + 2 * kLmKpRows;
}

// the packed position of the lower-triangle entry (i, k), k <= i
__device__ __forceinline__ int tri(int i, int k) { return i * (i + 1) / 2 + k; }

// the row r and column c (c <= r) of the packed entry p
__device__ __forceinline__ void tri_rc(int p, int &r, int &c) {
  r = (int)((sqrt(8.0 * p + 1.0) - 1.0) * 0.5);
  while ((r + 1) * (r + 2) / 2 <= p) ++r;
  while (r * (r + 1) / 2 > p) --r;
  c = p - r * (r + 1) / 2;
}

template <bool MEAS, bool PERSP>
__global__ void __launch_bounds__(kLmKpThreads, 1) lm_kp2d_step_kernel(LmKpArgs a, LmKp2dStepArgs x2) {
  extern __shared__ double smem[];
  __shared__ double lt_s, lam_s;
  __shared__ int ok_s;
  const int b = blockIdx.x, t = threadIdx.x, P = a.P, K = a.K, R3 = 3 * a.K, nb = a.nb, ne = x2.ne, nr9 = 9 * a.n_rot;
  const int o = 3 * a.n_rot, oe = o + nb, oc = oe + ne;   // first betas, expression and camera column
  const int npk = P * (P + 1) / 2;
  double *A = smem, *Js = A + npk, *WJs = Js + kLmKpRows * P, *y = WJs + kLmKpRows * P, *z = y + P, *dg = z + P,
         *col = dg + P, *ld = col + P, *ws = ld + P, *rs = ws + kLmKpRows;
  const float *tg = a.targets + (size_t)b * 2 * K, *wt = a.weights + (size_t)b * K;
  const float *anc = x2.anchor ? x2.anchor + (size_t)b * nr9 : nullptr;
  const bool robust = isfinite(x2.sigma), prior = x2.joint_w || x2.pose_w > 0.f;
  const double s2 = (double)x2.sigma * (double)x2.sigma;
  const float lcur = a.loss[b];
  // 1. trial loss
  if (t == 0) {
    LmKp2dArgs xs = x2;
    if (x2.joint_w) xs.pose_w = 0.f;       // the per-joint prior follows the keypoint term
    double L;
    if constexpr (PERSP) {
      const PerspCam tc = persp_cam(x2.intr + (size_t)b * 3, a.tlast + (size_t)b * 3);
      L = lm_kp2d_trial_loss<true>(a, xs, b, tg, wt, anc, robust, s2, &tc);
    } else {
      L = lm_kp2d_trial_loss(a, xs, b, tg, wt, anc, robust, s2);
    }
    if (x2.joint_w) {
      const float *tr = a.trot + (size_t)b * nr9;
      for (int j = 1; j < a.n_rot; ++j) {
        if (!(x2.joint_w[j] > 0.f)) continue;
        double q = 0.0;
        for (int e = 9 * j; e < 9 * j + 9; ++e) {
          const double d = (double)tr[e] - (double)anc[e];
          q += d * d;
        }
        L += (0.5 * (double)x2.joint_w[j]) * q;
      }
    }
    if constexpr (MEAS) L += lm_meas_loss(x2.mb, b);
    if (x2.betas_w > 0.f) L += (double)x2.betas_w * lm_sq_norm(a.tbetas + (size_t)b * nb, nb);
    if (x2.expr_w > 0.f) L += (double)x2.expr_w * lm_sq_norm(x2.texpr + (size_t)b * ne, ne);
    lt_s = L;
  }
  for (int p = t; p < npk; p += blockDim.x) A[p] = 0.0;
  __syncthreads();
  // 2. accept or reject
  const double lt = lt_s;
  const bool accept = lm_accept(a.first, lt, lcur);
  const float lnew = lm_loss(accept, lt, lcur);
  const float *J = (accept ? a.tjac : a.jac) + (size_t)b * R3 * P;
  const float *M = (accept ? a.tkp : a.kp) + (size_t)b * R3;
  const float *Rst = (accept ? a.trot : a.rot) + (size_t)b * nr9;
  const float *Bst = (accept ? a.tbetas : a.betas) + (size_t)b * nb;
  const float *Est = ne ? (accept ? x2.texpr : x2.expr) + (size_t)b * ne : nullptr;
  const float *Cst = (accept ? a.tlast : a.last) + (size_t)b * 3;
  if (accept) {
    lm_kp_take_trial(a, b, lnew);
    for (int i = t; i < ne; i += blockDim.x) x2.expr[(size_t)b * ne + i] = x2.texpr[(size_t)b * ne + i];
    if constexpr (MEAS) lm_meas_take_trial(x2.mb, b, nb);
  }
  double s, ds;
  softplus_d((double)Cst[0], s, ds);
  const double cxy[2] = {(double)Cst[1], (double)Cst[2]};
  PerspCam sc{};
  if constexpr (PERSP) sc = persp_cam(x2.intr + (size_t)b * 3, Cst);
  double *fz = nullptr;
  if constexpr (PERSP) fz = lm_persp_factors();
  // 3. normal equations: the keypoint rows 2k + c, kLmKpRows at a time, into the packed triangle
  int r0e, c0e;                             // this thread's first packed entry
  tri_rc(t, r0e, c0e);
  double g = 0.0;
  for (int r0 = 0; r0 < 2 * K; r0 += kLmKpRows) {
    const int nr = min(kLmKpRows, 2 * K - r0);
    __syncthreads();
    for (int i = t; i < nr; i += blockDim.x) {
      double wr, res;
      lm_kp2d_row<PERSP>(M, tg, wt, s, cxy, robust, s2, (r0 + i) >> 1, (r0 + i) & 1, wr, res, &sc,
                         PERSP ? fz + 2 * i : nullptr);
      ws[i] = wr;
      rs[i] = res;
    }
    __syncthreads();
    for (int i = t; i < nr * P; i += blockDim.x) {
      const int row = i / P, c = i % P;
      const double wr = ws[row];
      if (wr > 0.0) {                       // a dropped keypoint's rows are never read: they may be NaN
        const double v = lm_kp2d_entry<false, PERSP>(J, M, P, oc, (r0 + row) >> 1, (r0 + row) & 1, c, s, ds, cxy,
                                                     PERSP ? fz + 2 * row : nullptr);
        Js[row * P + c] = v;
        WJs[row * P + c] = wr * v;
      }
    }
    __syncthreads();
    int r = r0e, c = c0e;
    for (int p = t; p < npk; p += blockDim.x) {
      double acc = A[p];
      for (int row = 0; row < nr; ++row)
        if (ws[row] > 0.0) acc += WJs[row * P + r] * Js[row * P + c];
      A[p] = acc;
      c += blockDim.x;
      while (c > r) {
        c -= r + 1;
        ++r;
      }
    }
    if (t < P)
      for (int row = 0; row < nr; ++row)
        if (ws[row] > 0.0) g += WJs[row * P + t] * rs[row];
  }
  __syncthreads();
  if (t < P) dg[t] = A[tri(t, t)];          // the diagonal of the keypoint rows: the first lambda
  // the pose-prior rows of joint j (weight w_j / 2) reach only its diagonal block: its six lower entries.  Another
  // thread than t adds the prior to diagonal entry t: every dg read has to come first
  __syncthreads();
  if (prior) {
    for (int q = t; q < 6 * (a.n_rot - 1); q += blockDim.x) {
      const int j = 1 + q / 6, u = q % 6, ar = u < 1 ? 0 : u < 3 ? 1 : 2, ac = u - ar * (ar + 1) / 2;
      const float wj = x2.joint_w ? x2.joint_w[j] : x2.pose_w;
      if (!(wj > 0.f)) continue;
      const double hw = 0.5 * (double)wj;
      const float *R = Rst + 9 * j;
      const int p = tri(3 * j + ar, 3 * j + ac);
      double acc = A[p];
      for (int e = 0; e < 9; ++e) acc += (hw * rot_tangent(R, ar, e)) * rot_tangent(R, ac, e);
      A[p] = acc;
    }
    if (t >= 3 && t < o) {
      const float wj = x2.joint_w ? x2.joint_w[t / 3] : x2.pose_w;
      if (wj > 0.f) {
        const double hw = 0.5 * (double)wj;
        const float *R = Rst + 9 * (t / 3), *R0 = anc + 9 * (t / 3);
        for (int e = 0; e < 9; ++e) g += (hw * rot_tangent(R, t % 3, e)) * ((double)R[e] - (double)R0[e]);
      }
    }
  }
  if constexpr (MEAS) {
    // the five measurement rows at the state (values Mm, Jacobian Jm (5, nb)) into the betas block, in m order, each
    // entry (o + r, o + c) by one thread; a dropped term's row is never read: it may be NaN
    const float *Mm = (accept ? x2.mb.tmeas : x2.mb.meas) + (size_t)b * 5;
    const float *Jm = (accept ? x2.mb.tjac : x2.mb.jac) + (size_t)b * 5 * nb;
    const float *mt = x2.mb.targets + (size_t)b * 5, *mw = x2.mb.weights + (size_t)b * 5;
    for (int q = t; q < nb * (nb + 1) / 2; q += blockDim.x) {
      int r, c;
      tri_rc(q, r, c);
      double acc = A[tri(o + r, o + c)];
      for (int m = 0; m < 5; ++m) {
        const double w = mw[m];
        if (w > 0.0) acc += (w * (double)Jm[m * nb + r]) * (double)Jm[m * nb + c];
      }
      A[tri(o + r, o + c)] = acc;
    }
    if (t >= o && t < oe)
      for (int m = 0; m < 5; ++m) {
        const double w = mw[m];
        if (w > 0.0) g += (w * (double)Jm[m * nb + t - o]) * ((double)Mm[m] - (double)mt[m]);
      }
  }
  if (x2.betas_w > 0.f && t >= o && t < oe) g += (double)x2.betas_w * (double)Bst[t - o];
  if (x2.expr_w > 0.f && t >= oe && t < oc) g += (double)x2.expr_w * (double)Est[t - oe];
  if (t < P) y[t] = -g;
  __syncthreads();
  if (t == 0) {
    double dmax = kDiagFloor;
    if (a.first)
      for (int j = 0; j < P; ++j) dmax = fmax(dmax, dg[j]);
    const float lam = lm_lambda(a.first, accept, a.first ? 0.f : a.lambda[b], dmax, a.up, a.down);
    a.lambda[b] = lam;
    if (accept && !a.first) a.accepted[b] += 1;
    lam_s = lam;
    ok_s = isfinite(lnew);
  }
  __syncthreads();
  if (t < P) {
    const double lam = lam_s;
    A[tri(t, t)] += t >= o && t < oe ? (double)x2.betas_w + lam : t >= oe && t < oc ? (double)x2.expr_w + lam : lam;
  }
  // 4. Cholesky A = L L^T on the packed triangle: column j scaled (its pivot into ld, a copy into col), then the
  // trailing triangle updated, one warp per row
  const int warp = t >> 5, lane = t & 31, nw = blockDim.x >> 5;
  for (int j = 0; j < P; ++j) {
    __syncthreads();
    const double d = A[tri(j, j)];
    const double ljj = sqrt(d);
    if (t == 0) {
      ok_s = ok_s && d > 0.0 && isfinite(d);
      ld[j] = ljj;
    }
    for (int i = j + 1 + t; i < P; i += blockDim.x) {
      const double v = A[tri(i, j)] / ljj;
      A[tri(i, j)] = v;
      col[i] = v;
    }
    __syncthreads();
    for (int i = j + 1 + warp; i < P; i += nw) {
      const double ci = col[i];
      double *Ai = A + tri(i, 0);
      for (int k = j + 1 + lane; k <= i; k += 32) Ai[k] -= ci * col[k];
    }
  }
  // L z = -g (column order), then L^T delta = z (column order, from the last) into y
  for (int j = 0; j < P; ++j) {
    __syncthreads();
    const double yj = y[j] / ld[j];
    if (t == 0) z[j] = yj;
    for (int i = j + 1 + t; i < P; i += blockDim.x) y[i] -= A[tri(i, j)] * yj;
  }
  for (int j = P - 1; j >= 0; --j) {
    __syncthreads();
    const double dj = z[j] / ld[j];
    if (t == 0) y[j] = dj;
    for (int i = t; i < j; i += blockDim.x) z[i] -= A[tri(j, i)] * dj;
  }
  __syncthreads();
  // 5. next trial (ok is uniform: every thread reads it after the last barrier); a failed step keeps the state
  const bool ok = ok_s;
  const float *sr = a.rot + (size_t)b * nr9;
  float *trr = a.trot + (size_t)b * nr9;
  for (int j = t; j < a.n_rot; j += blockDim.x) {
    if (!ok) {
      for (int e = 0; e < 9; ++e) trr[9 * j + e] = sr[9 * j + e];
      continue;
    }
    lm_exp_gs(sr + 9 * j, y[3 * j], y[3 * j + 1], y[3 * j + 2], trr + 9 * j);
  }
  for (int l = t; l < nb; l += blockDim.x) {
    const float v = a.betas[(size_t)b * nb + l];
    a.tbetas[(size_t)b * nb + l] = ok ? (float)((double)v + y[o + l]) : v;
  }
  for (int l = t; l < ne; l += blockDim.x) {
    const float v = x2.expr[(size_t)b * ne + l];
    x2.texpr[(size_t)b * ne + l] = ok ? (float)((double)v + y[oe + l]) : v;
  }
  if (t < 3) {
    const float v = a.last[(size_t)b * 3 + t];
    a.tlast[(size_t)b * 3 + t] = ok ? (float)((double)v + y[oc + t]) : v;
  }
}

// The 2D step's arguments without per-joint weights and expression: what the 22-joint entries pass
inline LmKp2dStepArgs kp2d_args(const float *anchor, float sigma, float pose_w, float betas_w, const LmMeasArgs &mb,
                                const float *intr) {
  LmKp2dStepArgs x{};
  static_cast<LmKp2dPerspArgs &>(x) = LmKp2dPerspArgs{{anchor, sigma, pose_w, betas_w, mb}, intr};
  return x;
}

// The single-image 2D entries' checks and the launch: `persp` and `meas` say which pointers the entry takes, and
// max_p bounds P, kLmKpMaxP for the 22-joint entries (which take no expression and state none in their messages) and
// kLmKp2dMaxP for the expressive ones
int run_lm_kp2d(const char *fn, int batch, LmKpArgs a, LmKp2dStepArgs x, bool persp, bool meas, int max_p,
                void *stream) {
  const bool ptrs = (x.anchor || !(x.pose_w > 0.f || x.joint_w)) && (x.ne == 0 || (x.expr && x.texpr)) &&
                    (!persp || x.intr) && (!meas || lm_meas_ptrs(x.mb));
  SHAPY_REQUIRE(a.targets && a.weights && a.rot && a.betas && a.last && a.kp && a.jac && a.loss && a.lambda &&
                    a.accepted && a.trot && a.tbetas && a.tlast && a.tkp && a.tjac && ptrs,
                "%s: null argument", fn);
  const bool sizes = batch >= 0 && a.K >= 1 && a.n_rot >= 1 && a.n_rot <= 64 && a.nb >= 1 && x.ne >= 0;
  if (max_p == kLmKpMaxP)
    SHAPY_REQUIRE(sizes, "%s: bad size (batch %d, %d keypoints, n_rot %d, %d betas)", fn, batch, a.K, a.n_rot, a.nb);
  SHAPY_REQUIRE(sizes, "%s: bad size (batch %d, %d keypoints, n_rot %d, %d betas, %d expression)", fn, batch, a.K,
                a.n_rot, a.nb, x.ne);
  SHAPY_REQUIRE(a.up >= 1.f && a.down >= 1.f && lm_kp2d_factors_ok(x) && x.expr_w >= 0.f, "%s: %s", fn,
                kLmKp2dFactors);
  a.P = 3 * a.n_rot + a.nb + x.ne + 3;
  if (a.P > max_p) {
    set_error("%s: %d parameters, at most %d are supported", fn, a.P, max_p);
    return SHAPY_ERR_UNSUPPORTED;
  }
  if (batch == 0) return SHAPY_OK;
  const size_t smem = lm_kp2d_smem_doubles(a.P) * sizeof(double);
  auto kernel = meas ? (persp ? lm_kp2d_step_kernel<true, true> : lm_kp2d_step_kernel<true, false>)
                     : (persp ? lm_kp2d_step_kernel<false, true> : lm_kp2d_step_kernel<false, false>);
  return lm_launch(kernel, batch, kLmKpThreads, smem, stream, a, x);
}


// ---------------------------------------------------------------------------------------------------------------
// The step of the fit to 3D scans (shapy_fit_lm_scan_step): parameters [delta_j (3 n_rot) | beta | t], the columns of
// shapy_smplx_vertex_jacobian.  Loss, fp64, left to right: c_s Ls + c_m Lm + pose prior + measurements + betas_w
// |beta|^2, c_s = s2m / sum_{w_i > 0} w_i (1 when that sum is 0), c_m = m2s / V, Ls = sum_i w_i rho(d_i^2) over the kept
// points (d_i = |c_i - p_i|, c_i = sum_k b_ik x_{f_i,k}), Lm = sum_v rho(e_v^2) (e_v = |x_v - s_v|, s_v the vertex's
// nearest kept point).  Two kernels:
//   lm_scan_rows_kernel, one CTA per (chunk of kScanChunk points or vertices, body): the rows of the trial at its held
//     correspondences, staged kScanItems items (3 row slots each) at a time in fp64, accumulated into the packed lower
//     triangle of J^T U J (U the IRLS weights without c_s / c_m), J^T U r and the chunk's loss share; each thread owns
//     one 4 x 4 block of the triangle in registers (SIMT fp64), and the partial sums go to the workspace.  A point with
//     all barycentrics > 0 on a face of non-zero area gives one point-to-plane row n^T (c_i - p_i), n the face's unit
//     normal held constant; any other kept point three point-to-point rows c_i - p_i; a vertex with a nearest point
//     three rows x_v - s_v.  With the penetration term, a second launch (<true>) covers the 6 C points of the pair
//     rows (B, C, 2) in chunks after every body's scan chunks: point k < 3 is vertex k of the intruder in the receiver's cone, k >= 3 vertex k - 3 of the
//     receiver in the intruder's cone; a point with phi != 0 gives one row phi, weight w_p, its Jacobian
//     sum over the point and the cone's three vertices of (d phi / d x)^T J_x, phi and its derivatives in fp64
//     (penetration.cuh).  The chunking depends on N, V and C only; no atomics.
//   lm_scan_step_kernel, one CTA per body: the chunks summed in chunk order into the trial's loss, A = c_s A_s +
//     c_m A_m (+ A_p, the penetration chunks, already weighted) and g, the policy of the other steps, the state's A and g replaced by the trial's on accept (P^2 + P
//     doubles instead of a Jacobian), then the pose-prior and measurement rows at the state, betas_w + lambda on the
//     betas diagonal and lambda elsewhere, lm_kp_solve and the next trial.
constexpr int kScanChunk = 1024;        // points or vertices per CTA of the row kernel
constexpr int kScanItems = 16;          // items staged at a time: 3 row slots each
constexpr int kScanRows = 3 * kScanItems;
constexpr int kScanThreads = 320;       // >= the 4 x 4 blocks of the lower triangle at P = 96 (300)

// doubles per (body, chunk) in the workspace: the packed lower triangle, g and the loss share
__host__ __device__ inline size_t lm_scan_stride(int P) { return (size_t)P * (P + 1) / 2 + P + 1; }

inline int lm_scan_chunks(int n) { return (n + kScanChunk - 1) / kScanChunk; }

// rho(e) and its derivative: Geman-McClure e s2 / (s2 + e) and (s2 / (s2 + e))^2, or e and 1 for least squares
__device__ __forceinline__ void scan_rho(bool robust, double s2, double e, double &rho, double &drho) {
  if (robust) {
    const double q = s2 / (s2 + e);
    rho = e * q;
    drho = q * q;
  } else {
    rho = e;
    drho = 1.0;
  }
}

struct LmScanRowArgs {
  int N, V, P, ns, nm;                  // points, vertices, parameters, point chunks, vertex chunks
  const float *points, *weights;        // (B, N, 3), (B, N)
  const int32_t *faces;                 // (F, 3)
  const float *verts, *jac;             // the trial's (B, V, 3), (B, V, 3, P)
  const int32_t *face_idx, *nearest;    // (B, N), (B, V) or null (no model -> scan term)
  const float *bary;                    // (B, N, 3)
  float sigma, s2m, m2s;
  double *ws;
};

// The penetration rows: pairs (B, C, 2) of shapy_self_collisions on F faces, np chunks of the 6 C points per body,
// weight w; their partial sums at ws, (B, np) chunks after the (B, ns + nm) of the scan terms.
struct LmScanPenArgs {
  const int32_t *pairs;
  int C, np, F;
  float w;
  PenParams pen;
  double *ws;
};

// Penetration point i of body b (pair i / 6, point i % 6): with phi != 0 its row (kind 4, weight w_p, residual phi,
// loss share w_p phi^2) and d phi / d x of the point and the cone's three vertices.
__device__ __forceinline__ void lm_scan_pen_item(const LmScanRowArgs &a, const LmScanPenArgs &pa, int b, int i,
                                                 double (*pg)[3], int *vid, int &kind, double &u, double &r, double &l) {
  int rf[3], qf[3];
  if (!pen::pair_faces(pa.pairs + ((size_t)b * pa.C + i / 6) * 2, a.faces, pa.F, rf, qf)) return;
  const int k = i % 6;
  const int *cv = k < 3 ? rf : qf;       // the cone's face; the point is a vertex of the other face
  const int pv = k < 3 ? qf[k] : rf[k - 3];
  const float *vb = a.verts + (size_t)b * a.V * 3;
  const pen::Cone<double> cone = pen::make_cone(pen::ld<double>(vb + 3 * cv[0]), pen::ld<double>(vb + 3 * cv[1]),
                                                pen::ld<double>(vb + 3 * cv[2]));
  const pen::V3<double> p = pen::ld<double>(vb + 3 * pv);
  const pen::PointTerms<double> e = pen::point_terms(p, cone, pa.pen);
  if (e.phi == 0.0) return;
  pen::V3<double> gp{0.0, 0.0, 0.0}, gc = gp, gn = gp, gx[3] = {gp, gp, gp};
  double gr = 0.0;
  pen::point_backward(p, cone, e, pa.pen, 1.0, gp, gc, gn, gr);
  pen::cone_backward(cone, gc, gn, gr, gx);
  const pen::V3<double> gv[4] = {gp, gx[0], gx[1], gx[2]};
  const int vv[4] = {pv, cv[0], cv[1], cv[2]};
  for (int m = 0; m < 4; ++m) {
    vid[m] = vv[m];
    pg[m][0] = gv[m].x; pg[m][1] = gv[m].y; pg[m][2] = gv[m].z;
  }
  const double w = pa.w;
  kind = 4;
  u = w;
  r = e.phi;
  l = w * (e.phi * e.phi);
}

// PEN: the penetration chunks (blockIdx.x the chunk of pa), otherwise the point then vertex chunks of the scan terms.
template <bool PEN>
__global__ void __launch_bounds__(kScanThreads) lm_scan_rows_kernel(LmScanRowArgs a, LmScanPenArgs pa) {
  __shared__ double Js[kScanRows][kLmKpMaxP];
  __shared__ double us[kScanRows], rs[kScanRows], ls[kScanItems], cf[kScanItems][3], nrm[kScanItems][3];
  __shared__ double pg[PEN ? kScanItems : 1][4][3];     // d phi / d x of a penetration point's four vertices
  __shared__ int vid[kScanItems][PEN ? 4 : 3], kind[kScanItems];  // 1 point-to-plane, 2 point-to-point, 3 vertex, 4 pen
  const int b = blockIdx.y, c = blockIdx.x, t = threadIdx.x, P = a.P, Pp = (P + 3) & ~3, nbw = Pp / 4;
  const bool pts = !PEN && c < a.ns;
  const int i0 = (PEN ? c : pts ? c : c - a.ns) * kScanChunk, n = min(kScanChunk, (PEN ? 6 * pa.C : pts ? a.N : a.V) - i0);
  const bool active = PEN ? pa.w > 0.f : pts ? a.s2m > 0.f : (a.m2s > 0.f && a.nearest);
  const bool robust = isfinite(a.sigma);
  const double s2 = (double)a.sigma * (double)a.sigma;
  int bi = 0, bj = 0;
  tri_rc(t, bi, bj);
  const bool own = t < nbw * (nbw + 1) / 2;
  double acc[4][4], g = 0.0, L = 0.0;
  for (int x = 0; x < 4; ++x)
    for (int y = 0; y < 4; ++y) acc[x][y] = 0.0;
  const float *J = a.jac + (size_t)b * a.V * 3 * P;
  for (int s0 = 0; active && s0 < n; s0 += kScanItems) {
    const int ni = min(kScanItems, n - s0);
    __syncthreads();
    if (t < ni) {                       // item t: its rows' weights, residuals and what their entries need
      for (int r = 0; r < 3; ++r) us[3 * t + r] = rs[3 * t + r] = 0.0;
      ls[t] = 0.0;
      kind[t] = 0;
      const int i = i0 + s0 + t;
      double d[3];
      if constexpr (PEN) {
        lm_scan_pen_item(a, pa, b, i, pg[t], vid[t], kind[t], us[3 * t], rs[3 * t], ls[t]);
      } else if (pts) {
        const double w = a.weights[(size_t)b * a.N + i];
        if (w > 0.0) {                  // a dropped point is never read
          const int f = a.face_idx[(size_t)b * a.N + i];
          const float *p = a.points + ((size_t)b * a.N + i) * 3, *bc = a.bary + ((size_t)b * a.N + i) * 3;
          double X[3][3];
          for (int k = 0; k < 3; ++k) {
            const int v = a.faces[3 * f + k];
            vid[t][k] = v;
            cf[t][k] = bc[k];
            for (int q = 0; q < 3; ++q) X[k][q] = a.verts[((size_t)b * a.V + v) * 3 + q];
          }
          for (int q = 0; q < 3; ++q) d[q] = cf[t][0] * X[0][q] + cf[t][1] * X[1][q] + cf[t][2] * X[2][q] - (double)p[q];
          double rho, drho;
          scan_rho(robust, s2, d[0] * d[0] + d[1] * d[1] + d[2] * d[2], rho, drho);
          ls[t] = w * rho;
          const double u = w * drho;
          const double e1[3] = {X[1][0] - X[0][0], X[1][1] - X[0][1], X[1][2] - X[0][2]};
          const double e2[3] = {X[2][0] - X[0][0], X[2][1] - X[0][1], X[2][2] - X[0][2]};
          const double nv[3] = {e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2],
                                e1[0] * e2[1] - e1[1] * e2[0]};
          const double nn = sqrt(nv[0] * nv[0] + nv[1] * nv[1] + nv[2] * nv[2]);
          if (cf[t][0] > 0.0 && cf[t][1] > 0.0 && cf[t][2] > 0.0 && nn > 0.0) {
            for (int q = 0; q < 3; ++q) nrm[t][q] = nv[q] / nn;
            kind[t] = 1;
            us[3 * t] = u;
            rs[3 * t] = nrm[t][0] * d[0] + nrm[t][1] * d[1] + nrm[t][2] * d[2];
          } else {
            kind[t] = 2;
            for (int q = 0; q < 3; ++q) {
              us[3 * t + q] = u;
              rs[3 * t + q] = d[q];
            }
          }
        }
      } else {
        const int q = a.nearest[(size_t)b * a.V + i];
        if (q >= 0) {
          const float *s = a.points + ((size_t)b * a.N + q) * 3;
          for (int k = 0; k < 3; ++k) d[k] = (double)a.verts[((size_t)b * a.V + i) * 3 + k] - (double)s[k];
          double rho, drho;
          scan_rho(robust, s2, d[0] * d[0] + d[1] * d[1] + d[2] * d[2], rho, drho);
          ls[t] = rho;
          kind[t] = 3;
          vid[t][0] = i;
          for (int k = 0; k < 3; ++k) {
            us[3 * t + k] = drho;
            rs[3 * t + k] = d[k];
          }
        }
      }
    }
    __syncthreads();
    for (int e = t; e < 3 * ni * Pp; e += blockDim.x) {
      const int row = e / Pp, col = e % Pp, it = row / 3, cc = row % 3;
      if (!(us[row] > 0.0)) continue;
      double x = 0.0;
      if (col < P) {
        const int k = kind[it];
        auto mix = [&](int q) {       // sum_k b_k J_{v_k}, row q
          const float *j0 = J + ((size_t)vid[it][0] * 3 + q) * P + col, *j1 = J + ((size_t)vid[it][1] * 3 + q) * P + col,
                      *j2 = J + ((size_t)vid[it][2] * 3 + q) * P + col;
          return cf[it][0] * (double)*j0 + cf[it][1] * (double)*j1 + cf[it][2] * (double)*j2;
        };
        if (k == 1) x = nrm[it][0] * mix(0) + nrm[it][1] * mix(1) + nrm[it][2] * mix(2);
        else if (k == 2) x = mix(cc);
        else if (PEN)
          for (int m = 0; m < 4; ++m)
            for (int q = 0; q < 3; ++q) x += pg[it][m][q] * (double)J[((size_t)vid[it][m] * 3 + q) * P + col];
        else x = (double)J[((size_t)vid[it][0] * 3 + cc) * P + col];
      }
      Js[row][col] = x;
    }
    __syncthreads();
    if (t == 0)
      for (int it = 0; it < ni; ++it) L += ls[it];
    for (int row = 0; row < 3 * ni; ++row) {
      const double u = us[row];
      if (!(u > 0.0)) continue;
      if (own) {
        double ja[4], jb[4];
        for (int x = 0; x < 4; ++x) {
          ja[x] = u * Js[row][4 * bi + x];
          jb[x] = Js[row][4 * bj + x];
        }
        for (int x = 0; x < 4; ++x)
          for (int y = 0; y < 4; ++y) acc[x][y] += ja[x] * jb[y];
      }
      if (t < P) g += (u * Js[row][t]) * rs[row];
    }
  }
  const int npk = P * (P + 1) / 2;
  double *o = PEN ? pa.ws + ((size_t)b * pa.np + c) * lm_scan_stride(P)
                  : a.ws + ((size_t)b * (a.ns + a.nm) + c) * lm_scan_stride(P);
  if (own)
    for (int x = 0; x < 4; ++x)
      for (int y = 0; y < 4; ++y) {
        const int i = 4 * bi + x, j = 4 * bj + y;
        if (i < P && j <= i) o[tri(i, j)] = acc[x][y];
      }
  if (t < P) o[npk + t] = g;
  if (t == 0) o[npk + P] = L;
}

struct LmScanStepArgs {
  int N, V, ns, nm;
  const float *weights;                 // (B, N): sum_{w_i > 0} w_i normalises the scan -> model term
  float s2m, m2s;
  LmKp2dArgs x2;                        // anchor, pose_w and betas_w, and the measurement block with MEAS
  double *A, *g;                        // the state's undamped data rows: (B, P, P) symmetric, (B, P)
  const double *ws;
  int np;                               // penetration chunks per body (0 without the term) and their partial sums
  const double *wsp;
};

template <bool MEAS>
__global__ void __launch_bounds__(kLmKpThreads) lm_scan_step_kernel(LmKpArgs a, LmScanStepArgs x) {
  extern __shared__ double A[];         // [P][P]: the lower triangle of the normal matrix, then its Cholesky factor
  __shared__ double y[kLmKpMaxP], dg[kLmKpMaxP], part[kLmKpThreads];
  __shared__ double lt_s, cs_s, cm_s, lam_s;
  __shared__ int ok_s;
  const int b = blockIdx.x, t = threadIdx.x, P = a.P, nb = a.nb, nr9 = 9 * a.n_rot, o = 3 * a.n_rot;
  const int npk = P * (P + 1) / 2, nc = x.ns + x.nm;
  const size_t S = lm_scan_stride(P);
  const double *wsb = x.ws + (size_t)b * nc * S, *wpb = x.wsp + (size_t)b * x.np * S;
  const float *anc = x.x2.anchor ? x.x2.anchor + (size_t)b * nr9 : nullptr;
  const float lcur = a.loss[b];
  // 1. trial loss: sum_{w_i > 0} w_i strided over the threads, the threads' sums in thread order, then the chunks
  double sw = 0.0;
  for (int i = t; i < x.N; i += blockDim.x) {
    const double w = x.weights[(size_t)b * x.N + i];
    if (w > 0.0) sw += w;
  }
  part[t] = sw;
  __syncthreads();
  if (t == 0) {
    double W = 0.0;
    for (int q = 0; q < (int)blockDim.x; ++q) W += part[q];
    const double cs = (double)x.s2m / (W > 0.0 ? W : 1.0), cm = (double)x.m2s / (double)x.V;
    double Ls = 0.0, Lm = 0.0;
    for (int c = 0; c < x.ns; ++c) Ls += wsb[c * S + npk + P];
    for (int c = x.ns; c < nc; ++c) Lm += wsb[c * S + npk + P];
    double L = cs * Ls + cm * Lm;
    if (x.np) {
      double Lp = 0.0;
      for (int c = 0; c < x.np; ++c) Lp += wpb[c * S + npk + P];
      L += Lp;
    }
    if (x.x2.pose_w > 0.f) L += lm_kp2d_prior_loss(x.x2, a.trot + (size_t)b * nr9, anc, nr9);
    if constexpr (MEAS) L += lm_meas_loss(x.x2.mb, b);
    if (x.x2.betas_w > 0.f) L += (double)x.x2.betas_w * lm_sq_norm(a.tbetas + (size_t)b * nb, nb);
    lt_s = L;
    cs_s = cs;
    cm_s = cm;
  }
  __syncthreads();
  // 2. accept or reject; an accepted trial's data rows become the state's
  const double lt = lt_s;
  const bool accept = lm_accept(a.first, lt, lcur);
  const float lnew = lm_loss(accept, lt, lcur);
  const float *Rst = (accept ? a.trot : a.rot) + (size_t)b * nr9;
  const float *Bst = (accept ? a.tbetas : a.betas) + (size_t)b * nb;
  if (accept) {
    lm_kp_take_trial(a, b, lnew);
    if constexpr (MEAS) lm_meas_take_trial(x.x2.mb, b, nb);
  }
  double *Ab = x.A + (size_t)b * P * P, *gb = x.g + (size_t)b * P;
  if (accept) {
    const double cs = cs_s, cm = cm_s;
    for (int p = t; p < npk + P; p += blockDim.x) {
      double s1 = 0.0, s2 = 0.0;
      for (int c = 0; c < x.ns; ++c) s1 += wsb[c * S + p];
      for (int c = x.ns; c < nc; ++c) s2 += wsb[c * S + p];
      const double v = cs * s1 + cm * s2;
      if (p < npk) {
        int r, k;
        tri_rc(p, r, k);
        A[r * P + k] = v;
        Ab[r * P + k] = v;
        Ab[k * P + r] = v;
      } else {
        y[p - npk] = v;
        gb[p - npk] = v;
      }
    }
    for (int p = t; x.np && p < npk + P; p += blockDim.x) {  // the penetration rows, by the thread that wrote p
      double s3 = 0.0;
      for (int c = 0; c < x.np; ++c) s3 += wpb[c * S + p];
      if (p < npk) {
        int r, k;
        tri_rc(p, r, k);
        const double v = A[r * P + k] + s3;
        A[r * P + k] = v;
        Ab[r * P + k] = v;
        Ab[k * P + r] = v;
      } else {
        y[p - npk] += s3;
        gb[p - npk] += s3;
      }
    }
  } else {
    for (int p = t; p < npk; p += blockDim.x) {
      int r, k;
      tri_rc(p, r, k);
      A[r * P + k] = Ab[r * P + k];
    }
    for (int i = t; i < P; i += blockDim.x) y[i] = gb[i];
  }
  __syncthreads();
  if (t < P) dg[t] = A[t * P + t];      // the data rows' diagonal: the first lambda
  __syncthreads();
  // 3. the pose-prior rows of joint j (weight pose_w / 2) reach only its diagonal block, the measurement rows the betas
  // block; each entry by one thread, and g_t by thread t
  if (x.x2.pose_w > 0.f) {
    const double hw = 0.5 * (double)x.x2.pose_w;
    for (int q = t; q < 6 * (a.n_rot - 1); q += blockDim.x) {
      const int j = 1 + q / 6, u = q % 6, ar = u < 1 ? 0 : u < 3 ? 1 : 2, ac = u - ar * (ar + 1) / 2;
      const float *R = Rst + 9 * j;
      double acc = A[(3 * j + ar) * P + 3 * j + ac];
      for (int e = 0; e < 9; ++e) acc += (hw * rot_tangent(R, ar, e)) * rot_tangent(R, ac, e);
      A[(3 * j + ar) * P + 3 * j + ac] = acc;
    }
  }
  if constexpr (MEAS) {
    const LmMeasArgs &mb = x.x2.mb;
    const float *Jm = (accept ? mb.tjac : mb.jac) + (size_t)b * 5 * nb;
    const float *mw = mb.weights + (size_t)b * 5;
    for (int q = t; q < nb * (nb + 1) / 2; q += blockDim.x) {
      int r, c;
      tri_rc(q, r, c);
      double acc = A[(o + r) * P + o + c];
      for (int m = 0; m < 5; ++m) {
        const double w = mw[m];
        if (w > 0.0) acc += (w * (double)Jm[m * nb + r]) * (double)Jm[m * nb + c];
      }
      A[(o + r) * P + o + c] = acc;
    }
  }
  if (t < P) {
    double g = y[t];
    if (x.x2.pose_w > 0.f && t >= 3 && t < o) {
      const double hw = 0.5 * (double)x.x2.pose_w;
      const float *R = Rst + 9 * (t / 3), *R0 = anc + 9 * (t / 3);
      for (int e = 0; e < 9; ++e) g += (hw * rot_tangent(R, t % 3, e)) * ((double)R[e] - (double)R0[e]);
    }
    if constexpr (MEAS) {
      const LmMeasArgs &mb = x.x2.mb;
      const float *Mm = (accept ? mb.tmeas : mb.meas) + (size_t)b * 5;
      const float *Jm = (accept ? mb.tjac : mb.jac) + (size_t)b * 5 * nb;
      const float *mt = mb.targets + (size_t)b * 5, *mw = mb.weights + (size_t)b * 5;
      if (t >= o && t < o + nb)
        for (int m = 0; m < 5; ++m) {
          const double w = mw[m];
          if (w > 0.0) g += (w * (double)Jm[m * nb + t - o]) * ((double)Mm[m] - (double)mt[m]);
        }
    }
    if (x.x2.betas_w > 0.f && t >= o && t < o + nb) g += (double)x.x2.betas_w * (double)Bst[t - o];
    y[t] = -g;
  }
  __syncthreads();
  if (t == 0) {
    double dmax = kDiagFloor;
    if (a.first)
      for (int j = 0; j < P; ++j) dmax = fmax(dmax, dg[j]);
    const float lam = lm_lambda(a.first, accept, a.first ? 0.f : a.lambda[b], dmax, a.up, a.down);
    a.lambda[b] = lam;
    if (accept && !a.first) a.accepted[b] += 1;
    lam_s = lam;
    ok_s = isfinite(lnew);
  }
  __syncthreads();
  if (t < P) A[t * P + t] += t >= o && t < o + nb ? (double)x.x2.betas_w + lam_s : lam_s;
  // 4. Cholesky and the two solves; 5. the next trial (a failed step keeps the state)
  lm_kp_solve(A, y, P, P, ok_s);
  lm_kp_next_trial(a, b, y, ok_s);
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
  LmKpArgs a{num_keypoints, n_rot, nb, 0, targets, weights, lambda_up, lambda_down, first ? 1 : 0, rot, betas, transl,
             keypoints, jac, loss, lambda, accepted, trial_rot, trial_betas, trial_transl, trial_keypoints, trial_jac};
  return run_lm_kp("shapy_fit_lm_keypoints_step", lm_kp_step_kernel<false>, batch, a, LmMeasArgs{}, true, true,
                   "lambda_up and lambda_down must be >= 1", stream);
}

extern "C" int shapy_fit_lm_keypoints_measurements_step(
    int batch, int num_keypoints, int n_rot, int nb, const float *targets, const float *weights,
    const float *meas_targets, const float *meas_weights, float betas_weight, float lambda_up, float lambda_down,
    int first, float *rot, float *betas, float *transl, float *keypoints, float *jac, float *meas, float *meas_jac,
    float *loss, float *lambda, int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_transl,
    const float *trial_keypoints, const float *trial_jac, const float *trial_meas, const float *trial_meas_jac,
    void *stream) {
  LmKpArgs a{num_keypoints, n_rot, nb, 0, targets, weights, lambda_up, lambda_down, first ? 1 : 0, rot, betas, transl,
             keypoints, jac, loss, lambda, accepted, trial_rot, trial_betas, trial_transl, trial_keypoints, trial_jac};
  LmMeasArgs m{meas_targets, meas_weights, betas_weight, meas, meas_jac, trial_meas, trial_meas_jac};
  return run_lm_kp("shapy_fit_lm_keypoints_measurements_step", lm_kp_step_kernel<true>, batch, a, m, lm_meas_ptrs(m),
                   betas_weight >= 0.f, "lambda_up and lambda_down must be >= 1 and betas_weight >= 0", stream);
}

extern "C" int shapy_fit_lm_keypoints_2d_step(int batch, int num_keypoints, int n_rot, int nb, const float *targets,
                                              const float *weights, const float *pose_anchor, float robust_sigma,
                                              float pose_prior_weight, float betas_weight, float lambda_up,
                                              float lambda_down, int first, float *rot, float *betas, float *camera,
                                              float *keypoints, float *jac, float *loss, float *lambda,
                                              int32_t *accepted, float *trial_rot, float *trial_betas,
                                              float *trial_camera, const float *trial_keypoints, const float *trial_jac,
                                              void *stream) {
  LmKpArgs a{num_keypoints, n_rot, nb, 0, targets, weights, lambda_up, lambda_down, first ? 1 : 0, rot, betas, camera,
             keypoints, jac, loss, lambda, accepted, trial_rot, trial_betas, trial_camera, trial_keypoints, trial_jac};
  return run_lm_kp2d("shapy_fit_lm_keypoints_2d_step", batch, a,
                     kp2d_args(pose_anchor, robust_sigma, pose_prior_weight, betas_weight, LmMeasArgs{}, nullptr), false,
                     false, kLmKpMaxP, stream);
}

extern "C" int shapy_fit_lm_keypoints_2d_measurements_step(
    int batch, int num_keypoints, int n_rot, int nb, const float *targets, const float *weights,
    const float *pose_anchor, float robust_sigma, float pose_prior_weight, float betas_weight,
    const float *meas_targets, const float *meas_weights, float lambda_up, float lambda_down, int first, float *rot,
    float *betas, float *camera, float *keypoints, float *jac, float *meas, float *meas_jac, float *loss, float *lambda,
    int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_camera, const float *trial_keypoints,
    const float *trial_jac, const float *trial_meas, const float *trial_meas_jac, void *stream) {
  LmKpArgs a{num_keypoints, n_rot, nb, 0, targets, weights, lambda_up, lambda_down, first ? 1 : 0, rot, betas, camera,
             keypoints, jac, loss, lambda, accepted, trial_rot, trial_betas, trial_camera, trial_keypoints, trial_jac};
  const LmMeasArgs m{meas_targets, meas_weights, 0.f, meas, meas_jac, trial_meas, trial_meas_jac};
  return run_lm_kp2d("shapy_fit_lm_keypoints_2d_measurements_step", batch, a,
                     kp2d_args(pose_anchor, robust_sigma, pose_prior_weight, betas_weight, m, nullptr), false, true,
                     kLmKpMaxP, stream);
}

extern "C" int shapy_fit_lm_keypoints_2d_perspective_step(
    int batch, int num_keypoints, int n_rot, int nb, const float *targets, const float *weights,
    const float *intrinsics, const float *pose_anchor, float robust_sigma, float pose_prior_weight, float betas_weight,
    float lambda_up, float lambda_down, int first, float *rot, float *betas, float *transl, float *keypoints,
    float *jac, float *loss, float *lambda, int32_t *accepted, float *trial_rot, float *trial_betas,
    float *trial_transl, const float *trial_keypoints, const float *trial_jac, void *stream) {
  LmKpArgs a{num_keypoints, n_rot, nb, 0, targets, weights, lambda_up, lambda_down, first ? 1 : 0, rot, betas, transl,
             keypoints, jac, loss, lambda, accepted, trial_rot, trial_betas, trial_transl, trial_keypoints, trial_jac};
  return run_lm_kp2d("shapy_fit_lm_keypoints_2d_perspective_step", batch, a,
                     kp2d_args(pose_anchor, robust_sigma, pose_prior_weight, betas_weight, LmMeasArgs{}, intrinsics),
                     true, false, kLmKpMaxP, stream);
}

extern "C" int shapy_fit_lm_keypoints_2d_perspective_measurements_step(
    int batch, int num_keypoints, int n_rot, int nb, const float *targets, const float *weights,
    const float *intrinsics, const float *pose_anchor, float robust_sigma, float pose_prior_weight, float betas_weight,
    const float *meas_targets, const float *meas_weights, float lambda_up, float lambda_down, int first, float *rot,
    float *betas, float *transl, float *keypoints, float *jac, float *meas, float *meas_jac, float *loss, float *lambda,
    int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_transl, const float *trial_keypoints,
    const float *trial_jac, const float *trial_meas, const float *trial_meas_jac, void *stream) {
  LmKpArgs a{num_keypoints, n_rot, nb, 0, targets, weights, lambda_up, lambda_down, first ? 1 : 0, rot, betas, transl,
             keypoints, jac, loss, lambda, accepted, trial_rot, trial_betas, trial_transl, trial_keypoints, trial_jac};
  const LmMeasArgs m{meas_targets, meas_weights, 0.f, meas, meas_jac, trial_meas, trial_meas_jac};
  return run_lm_kp2d("shapy_fit_lm_keypoints_2d_perspective_measurements_step", batch, a,
                     kp2d_args(pose_anchor, robust_sigma, pose_prior_weight, betas_weight, m, intrinsics), true, true,
                     kLmKpMaxP, stream);
}

extern "C" size_t shapy_fit_lm_groups_workspace_bytes(int batch, int num_groups, int n_rot, int nb) {
  if (batch < 0 || num_groups < 0 || n_rot < 1 || nb < 1) return 0;
  return lm_group_offsets_bytes(num_groups) + (size_t)batch * lm_group_stride(3 * n_rot + 3, nb) * sizeof(double);
}

extern "C" int shapy_fit_lm_keypoints_2d_groups_step(
    int batch, int num_groups, const int32_t *group_offsets, int num_keypoints, int n_rot, int nb,
    const float *targets, const float *weights, const float *pose_anchor, float robust_sigma, float pose_prior_weight,
    float betas_weight, float lambda_up, float lambda_down, int first, float *rot, float *betas, float *camera,
    float *keypoints, float *jac, float *loss, float *lambda, int32_t *accepted, float *trial_rot, float *trial_betas,
    float *trial_betas_images, float *trial_camera, const float *trial_keypoints, const float *trial_jac,
    void *workspace, void *stream) {
  LmKpArgs a{num_keypoints, n_rot, nb, 0, targets, weights, lambda_up, lambda_down, first ? 1 : 0, rot, betas, camera,
             keypoints, jac, loss, lambda, accepted, trial_rot, trial_betas, trial_camera, trial_keypoints, trial_jac};
  LmKp2dArgs x{pose_anchor, robust_sigma, pose_prior_weight, betas_weight, LmMeasArgs{}};
  return run_lm_kp2dg<false>("shapy_fit_lm_keypoints_2d_groups_step", batch, num_groups, group_offsets, a, x,
                             trial_betas_images, workspace, false, stream);
}

extern "C" int shapy_fit_lm_keypoints_2d_groups_measurements_step(
    int batch, int num_groups, const int32_t *group_offsets, int num_keypoints, int n_rot, int nb,
    const float *targets, const float *weights, const float *pose_anchor, float robust_sigma, float pose_prior_weight,
    float betas_weight, const float *meas_targets, const float *meas_weights, float lambda_up, float lambda_down,
    int first, float *rot, float *betas, float *camera, float *keypoints, float *jac, float *meas, float *meas_jac,
    float *loss, float *lambda, int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_betas_images,
    float *trial_camera, const float *trial_keypoints, const float *trial_jac, const float *trial_meas,
    const float *trial_meas_jac, void *workspace, void *stream) {
  LmKpArgs a{num_keypoints, n_rot, nb, 0, targets, weights, lambda_up, lambda_down, first ? 1 : 0, rot, betas, camera,
             keypoints, jac, loss, lambda, accepted, trial_rot, trial_betas, trial_camera, trial_keypoints, trial_jac};
  LmKp2dArgs x{pose_anchor, robust_sigma, pose_prior_weight, betas_weight,
               LmMeasArgs{meas_targets, meas_weights, 0.f, meas, meas_jac, trial_meas, trial_meas_jac}};
  return run_lm_kp2dg<false>("shapy_fit_lm_keypoints_2d_groups_measurements_step", batch, num_groups, group_offsets,
                             a, x, trial_betas_images, workspace, true, stream);
}

extern "C" size_t shapy_fit_lm_shared_pose_workspace_bytes(int batch, int num_groups, int n_rot, int nb) {
  if (batch < 0 || num_groups < 0 || n_rot < 1 || nb < 1) return 0;
  return lm_group_offsets_bytes(num_groups) + (size_t)batch * lm_group_stride(6, 3 * (n_rot - 1) + nb) * sizeof(double);
}

extern "C" int shapy_fit_lm_keypoints_2d_shared_pose_step(
    int batch, int num_groups, const int32_t *group_offsets, int num_keypoints, int n_rot, int nb,
    const float *targets, const float *weights, const float *pose_anchor, float robust_sigma, float pose_prior_weight,
    float betas_weight, float lambda_up, float lambda_down, int first, float *rot, float *betas, float *camera,
    float *keypoints, float *jac, float *loss, float *lambda, int32_t *accepted, float *trial_rot, float *trial_betas,
    float *trial_betas_images, float *trial_camera, const float *trial_keypoints, const float *trial_jac,
    void *workspace, void *stream) {
  LmKpArgs a{num_keypoints, n_rot, nb, 0, targets, weights, lambda_up, lambda_down, first ? 1 : 0, rot, betas, camera,
             keypoints, jac, loss, lambda, accepted, trial_rot, trial_betas, trial_camera, trial_keypoints, trial_jac};
  LmKp2dArgs x{pose_anchor, robust_sigma, pose_prior_weight, betas_weight, LmMeasArgs{}};
  return run_lm_kp2dg<true>("shapy_fit_lm_keypoints_2d_shared_pose_step", batch, num_groups, group_offsets, a, x,
                            trial_betas_images, workspace, false, stream);
}

extern "C" int shapy_fit_lm_keypoints_2d_shared_pose_measurements_step(
    int batch, int num_groups, const int32_t *group_offsets, int num_keypoints, int n_rot, int nb,
    const float *targets, const float *weights, const float *pose_anchor, float robust_sigma, float pose_prior_weight,
    float betas_weight, const float *meas_targets, const float *meas_weights, float lambda_up, float lambda_down,
    int first, float *rot, float *betas, float *camera, float *keypoints, float *jac, float *meas, float *meas_jac,
    float *loss, float *lambda, int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_betas_images,
    float *trial_camera, const float *trial_keypoints, const float *trial_jac, const float *trial_meas,
    const float *trial_meas_jac, void *workspace, void *stream) {
  LmKpArgs a{num_keypoints, n_rot, nb, 0, targets, weights, lambda_up, lambda_down, first ? 1 : 0, rot, betas, camera,
             keypoints, jac, loss, lambda, accepted, trial_rot, trial_betas, trial_camera, trial_keypoints, trial_jac};
  LmKp2dArgs x{pose_anchor, robust_sigma, pose_prior_weight, betas_weight,
               LmMeasArgs{meas_targets, meas_weights, 0.f, meas, meas_jac, trial_meas, trial_meas_jac}};
  return run_lm_kp2dg<true>("shapy_fit_lm_keypoints_2d_shared_pose_measurements_step", batch, num_groups,
                            group_offsets, a, x, trial_betas_images, workspace, true, stream);
}

extern "C" size_t shapy_fit_lm_calibrated_workspace_bytes(int num_views, int num_bodies) {
  if (num_views < 0 || num_bodies < 0) return 0;
  return lm_group_offsets_bytes(num_bodies);
}

extern "C" int shapy_fit_lm_keypoints_2d_calibrated_step(
    int num_views, int num_bodies, const int32_t *view_offsets, int num_keypoints, int n_rot, int nb,
    const float *targets, const float *weights, const float *intrinsics, const float *extrinsics,
    const float *pose_anchor, float robust_sigma, float pose_prior_weight, float betas_weight, float lambda_up,
    float lambda_down, int first, float *rot, float *betas, float *transl, float *keypoints, float *jac, float *loss,
    float *lambda, int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_transl,
    const float *trial_keypoints, const float *trial_jac, void *workspace, void *stream) {
  LmKpArgs a{num_keypoints, n_rot, nb, 0, targets, weights, lambda_up, lambda_down, first ? 1 : 0, rot, betas, transl,
             keypoints, jac, loss, lambda, accepted, trial_rot, trial_betas, trial_transl, trial_keypoints, trial_jac};
  LmKp2dCalibArgs x{{{pose_anchor, robust_sigma, pose_prior_weight, betas_weight, LmMeasArgs{}}, intrinsics},
                    extrinsics, nullptr};
  return run_lm_kp2dc<false>("shapy_fit_lm_keypoints_2d_calibrated_step", num_views, num_bodies, view_offsets, a, x,
                             workspace, stream);
}

extern "C" int shapy_fit_lm_keypoints_2d_calibrated_measurements_step(
    int num_views, int num_bodies, const int32_t *view_offsets, int num_keypoints, int n_rot, int nb,
    const float *targets, const float *weights, const float *intrinsics, const float *extrinsics,
    const float *pose_anchor, float robust_sigma, float pose_prior_weight, float betas_weight,
    const float *meas_targets, const float *meas_weights, float lambda_up, float lambda_down, int first, float *rot,
    float *betas, float *transl, float *keypoints, float *jac, float *meas, float *meas_jac, float *loss, float *lambda,
    int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_transl, const float *trial_keypoints,
    const float *trial_jac, const float *trial_meas, const float *trial_meas_jac, void *workspace, void *stream) {
  LmKpArgs a{num_keypoints, n_rot, nb, 0, targets, weights, lambda_up, lambda_down, first ? 1 : 0, rot, betas, transl,
             keypoints, jac, loss, lambda, accepted, trial_rot, trial_betas, trial_transl, trial_keypoints, trial_jac};
  LmKp2dCalibArgs x{{{pose_anchor, robust_sigma, pose_prior_weight, betas_weight,
                      LmMeasArgs{meas_targets, meas_weights, 0.f, meas, meas_jac, trial_meas, trial_meas_jac}},
                     intrinsics},
                    extrinsics, nullptr};
  return run_lm_kp2dc<true>("shapy_fit_lm_keypoints_2d_calibrated_measurements_step", num_views, num_bodies,
                            view_offsets, a, x, workspace, stream);
}

extern "C" size_t shapy_fit_lm_sequence_workspace_bytes(int batch, int num_sequences, int n_rot, int nb) {
  if (batch < 0 || num_sequences < 0 || n_rot < 1 || nb < 1) return 0;
  return lm_group_offsets_bytes(num_sequences) + (size_t)batch * lm_seq_stride(3 * n_rot + 3, nb) * sizeof(double);
}

extern "C" int shapy_fit_lm_keypoints_2d_sequence_step(
    int batch, int num_sequences, const int32_t *sequence_offsets, int num_keypoints, int n_rot, int nb,
    const float *targets, const float *weights, const float *intrinsics, const float *pose_anchor, float robust_sigma,
    float pose_prior_weight, float betas_weight, float smooth_rot_weight, float smooth_transl_weight, float lambda_up,
    float lambda_down, int first, float *rot, float *betas, float *transl, float *keypoints, float *jac, float *loss,
    float *lambda, int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_betas_images,
    float *trial_transl, const float *trial_keypoints, const float *trial_jac, void *workspace, void *stream) {
  LmKpArgs a{num_keypoints, n_rot, nb, 0, targets, weights, lambda_up, lambda_down, first ? 1 : 0, rot, betas, transl,
             keypoints, jac, loss, lambda, accepted, trial_rot, trial_betas, trial_transl, trial_keypoints, trial_jac};
  LmKp2dSeqArgs x{{{pose_anchor, robust_sigma, pose_prior_weight, betas_weight, LmMeasArgs{}}, intrinsics},
                  smooth_rot_weight, smooth_transl_weight};
  return run_lm_kp2ds("shapy_fit_lm_keypoints_2d_sequence_step", batch, num_sequences, sequence_offsets, a, x,
                      trial_betas_images, workspace, stream);
}

extern "C" int shapy_fit_lm_keypoints_2d_expressive_step(
    int batch, int num_keypoints, int n_rot, int nb, int ne, const float *targets, const float *weights,
    const float *pose_anchor, const float *joint_weights, float robust_sigma, float pose_prior_weight,
    float betas_weight, float expression_weight, float lambda_up, float lambda_down, int first, float *rot,
    float *betas, float *expression, float *camera, float *keypoints, float *jac, float *loss, float *lambda,
    int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_expression, float *trial_camera,
    const float *trial_keypoints, const float *trial_jac, void *stream) {
  LmKpArgs a{num_keypoints, n_rot, nb, 0, targets, weights, lambda_up, lambda_down, first ? 1 : 0, rot, betas, camera,
             keypoints, jac, loss, lambda, accepted, trial_rot, trial_betas, trial_camera, trial_keypoints, trial_jac};
  LmKp2dStepArgs x = kp2d_args(pose_anchor, robust_sigma, pose_prior_weight, betas_weight, LmMeasArgs{}, nullptr);
  x.joint_w = joint_weights;
  x.expr_w = expression_weight;
  x.ne = ne;
  x.expr = expression;
  x.texpr = trial_expression;
  return run_lm_kp2d("shapy_fit_lm_keypoints_2d_expressive_step", batch, a, x, false, false, kLmKp2dMaxP, stream);
}

extern "C" int shapy_fit_lm_keypoints_2d_expressive_perspective_step(
    int batch, int num_keypoints, int n_rot, int nb, int ne, const float *targets, const float *weights,
    const float *intrinsics, const float *pose_anchor, const float *joint_weights, float robust_sigma,
    float pose_prior_weight, float betas_weight, float expression_weight, float lambda_up, float lambda_down, int first,
    float *rot, float *betas, float *expression, float *transl, float *keypoints, float *jac, float *loss,
    float *lambda, int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_expression,
    float *trial_transl, const float *trial_keypoints, const float *trial_jac, void *stream) {
  LmKpArgs a{num_keypoints, n_rot, nb, 0, targets, weights, lambda_up, lambda_down, first ? 1 : 0, rot, betas, transl,
             keypoints, jac, loss, lambda, accepted, trial_rot, trial_betas, trial_transl, trial_keypoints, trial_jac};
  LmKp2dStepArgs x = kp2d_args(pose_anchor, robust_sigma, pose_prior_weight, betas_weight, LmMeasArgs{}, intrinsics);
  x.joint_w = joint_weights;
  x.expr_w = expression_weight;
  x.ne = ne;
  x.expr = expression;
  x.texpr = trial_expression;
  return run_lm_kp2d("shapy_fit_lm_keypoints_2d_expressive_perspective_step", batch, a, x, true, false, kLmKp2dMaxP,
                     stream);
}

extern "C" size_t shapy_fit_lm_scan_workspace_bytes(int batch, int num_points, int num_verts, int num_params) {
  if (batch < 0 || num_points < 1 || num_verts < 1 || num_params < 1) return 0;
  return (size_t)batch * (lm_scan_chunks(num_points) + lm_scan_chunks(num_verts)) * lm_scan_stride(num_params) *
         sizeof(double);
}

extern "C" size_t shapy_fit_lm_scan_penetration_workspace_bytes(int batch, int num_points, int num_verts,
                                                                int num_params, int num_pairs) {
  if (batch < 0 || num_points < 1 || num_verts < 1 || num_params < 1 || num_pairs < 0) return 0;
  return (size_t)batch * (lm_scan_chunks(num_points) + lm_scan_chunks(num_verts) + lm_scan_chunks(6 * num_pairs)) *
         lm_scan_stride(num_params) * sizeof(double);
}

namespace shapy {
// the penetration rows of shapy_fit_lm_scan_penetration_step; null: shapy_fit_lm_scan_step
struct LmScanPen {
  const int32_t *pairs;
  int C, F;
  float weight, sigma;
};

static int lm_scan_step_run(
    const char *fn, int batch, int num_points, int num_verts, int n_rot, int nb, const float *points,
    const float *weights, const int32_t *faces, const float *pose_anchor, float robust_sigma,
    float scan_to_model_weight, float model_to_scan_weight, float pose_prior_weight, float betas_weight,
    const float *meas_targets, const float *meas_weights, float lambda_up, float lambda_down, int first, float *rot,
    float *betas, float *transl, double *normal_matrix, double *gradient, float *meas, float *meas_jac, float *loss,
    float *lambda, int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_transl,
    const float *trial_vertices, const float *trial_jac, const int32_t *trial_face_idx, const float *trial_bary,
    const int32_t *trial_nearest, const float *trial_meas, const float *trial_meas_jac, const LmScanPen *pen,
    void *workspace, size_t workspace_bytes, void *stream) {
  const LmMeasArgs mb{meas_targets, meas_weights, 0.f, meas, meas_jac, trial_meas, trial_meas_jac};
  const bool with_meas = meas_targets || meas_weights || meas || meas_jac || trial_meas || trial_meas_jac;
  const float s2m = scan_to_model_weight, m2s = model_to_scan_weight;
  SHAPY_REQUIRE(points && weights && faces && rot && betas && transl && normal_matrix && gradient && loss && lambda &&
                    accepted && trial_rot && trial_betas && trial_transl && trial_vertices && trial_jac &&
                    trial_face_idx && trial_bary && workspace && (trial_nearest || !(m2s > 0.f)) &&
                    (pose_anchor || !(pose_prior_weight > 0.f)) && (!with_meas || lm_meas_ptrs(mb)) &&
                    (!pen || pen->pairs || pen->C == 0),
                "%s: null argument", fn);
  SHAPY_REQUIRE(batch >= 0 && batch <= 65535 && num_points >= 1 && num_verts >= 1 && n_rot >= 1 && n_rot <= 64 &&
                    nb >= 1,
                "%s: bad size (batch %d, %d points, %d vertices, n_rot %d, %d betas)", fn, batch, num_points, num_verts,
                n_rot, nb);
  SHAPY_REQUIRE(robust_sigma > 0.f && s2m >= 0.f && m2s >= 0.f && isfinite(s2m) && isfinite(m2s) &&
                    pose_prior_weight >= 0.f && betas_weight >= 0.f && lambda_up >= 1.f && lambda_down >= 1.f,
                "%s: robust_sigma must be > 0 (inf: least squares), the term and prior weights finite and >= 0 and "
                "lambda_up and lambda_down >= 1",
                fn);
  SHAPY_REQUIRE(!pen || (pen->C >= 0 && pen->F >= 1 && pen->weight >= 0.f && isfinite(pen->weight) &&
                         pen->sigma > 0.f && isfinite(pen->sigma)),
                "%s: the penetration pairs, faces, weight (finite, >= 0) or sigma (finite, > 0) are bad", fn);
  const int P = 3 * n_rot + nb + 3;
  if (P > kLmKpMaxP) {
    set_error("%s: %d parameters, at most %d are supported", fn, P, kLmKpMaxP);
    return SHAPY_ERR_UNSUPPORTED;
  }
  const size_t need = pen ? shapy_fit_lm_scan_penetration_workspace_bytes(batch, num_points, num_verts, P, pen->C)
                          : shapy_fit_lm_scan_workspace_bytes(batch, num_points, num_verts, P);
  SHAPY_REQUIRE(workspace_bytes >= need, "%s: workspace of %zu bytes, %zu needed", fn, workspace_bytes, need);
  if (batch == 0) return SHAPY_OK;
  const int ns = lm_scan_chunks(num_points), nm = lm_scan_chunks(num_verts), np = pen ? lm_scan_chunks(6 * pen->C) : 0;
  LmScanRowArgs r{num_points, num_verts, P,  ns, nm, points, weights, faces, trial_vertices, trial_jac, trial_face_idx,
                  trial_nearest, trial_bary, robust_sigma, s2m, m2s, (double *)workspace};
  LmScanPenArgs pa{};
  lm_scan_rows_kernel<false><<<dim3(ns + nm, batch), kScanThreads, 0, (cudaStream_t)stream>>>(r, pa);
  SHAPY_LAUNCH_CHECK();
  if (np > 0) {
    pa = LmScanPenArgs{pen->pairs, pen->C, np, pen->F, pen->weight, PenParams{pen->sigma, 1000.f, true},
                       (double *)workspace + (size_t)batch * (ns + nm) * lm_scan_stride(P)};
    lm_scan_rows_kernel<true><<<dim3(np, batch), kScanThreads, 0, (cudaStream_t)stream>>>(r, pa);
    SHAPY_LAUNCH_CHECK();
  }
  LmKpArgs a{0, n_rot, nb, P, nullptr, nullptr, lambda_up, lambda_down, first ? 1 : 0, rot, betas, transl, nullptr,
             nullptr, loss, lambda, accepted, trial_rot, trial_betas, trial_transl, nullptr, nullptr};
  LmScanStepArgs x{num_points, num_verts, ns, nm, weights, s2m, m2s,
                   LmKp2dArgs{pose_anchor, robust_sigma, pose_prior_weight, betas_weight, mb}, normal_matrix,
                   gradient, (const double *)workspace, np, pa.ws};
  return lm_launch(with_meas ? lm_scan_step_kernel<true> : lm_scan_step_kernel<false>, batch, kLmKpThreads,
                   lm_kp_smem(P), stream, a, x);
}
}  // namespace shapy

extern "C" int shapy_fit_lm_scan_step(
    int batch, int num_points, int num_verts, int n_rot, int nb, const float *points, const float *weights,
    const int32_t *faces, const float *pose_anchor, float robust_sigma, float scan_to_model_weight,
    float model_to_scan_weight, float pose_prior_weight, float betas_weight, const float *meas_targets,
    const float *meas_weights, float lambda_up, float lambda_down, int first, float *rot, float *betas, float *transl,
    double *normal_matrix, double *gradient, float *meas, float *meas_jac, float *loss, float *lambda,
    int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_transl, const float *trial_vertices,
    const float *trial_jac, const int32_t *trial_face_idx, const float *trial_bary, const int32_t *trial_nearest,
    const float *trial_meas, const float *trial_meas_jac, void *workspace, size_t workspace_bytes, void *stream) {
  return lm_scan_step_run("shapy_fit_lm_scan_step", batch, num_points, num_verts, n_rot, nb, points, weights, faces,
                          pose_anchor, robust_sigma, scan_to_model_weight, model_to_scan_weight, pose_prior_weight,
                          betas_weight, meas_targets, meas_weights, lambda_up, lambda_down, first, rot, betas, transl,
                          normal_matrix, gradient, meas, meas_jac, loss, lambda, accepted, trial_rot, trial_betas,
                          trial_transl, trial_vertices, trial_jac, trial_face_idx, trial_bary, trial_nearest,
                          trial_meas, trial_meas_jac, nullptr, workspace, workspace_bytes, stream);
}

extern "C" int shapy_fit_lm_scan_penetration_step(
    int batch, int num_points, int num_verts, int n_rot, int nb, const float *points, const float *weights,
    const int32_t *faces, int num_faces, const float *pose_anchor, float robust_sigma, float scan_to_model_weight,
    float model_to_scan_weight, float pose_prior_weight, float betas_weight, const float *meas_targets,
    const float *meas_weights, const int32_t *pen_pairs, int num_pairs, float penetration_weight,
    float penetration_sigma, float lambda_up, float lambda_down, int first, float *rot, float *betas, float *transl,
    double *normal_matrix, double *gradient, float *meas, float *meas_jac, float *loss, float *lambda,
    int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_transl, const float *trial_vertices,
    const float *trial_jac, const int32_t *trial_face_idx, const float *trial_bary, const int32_t *trial_nearest,
    const float *trial_meas, const float *trial_meas_jac, void *workspace, size_t workspace_bytes, void *stream) {
  const LmScanPen pen{pen_pairs, num_pairs, num_faces, penetration_weight, penetration_sigma};
  return lm_scan_step_run("shapy_fit_lm_scan_penetration_step", batch, num_points, num_verts, n_rot, nb, points,
                          weights, faces, pose_anchor, robust_sigma, scan_to_model_weight, model_to_scan_weight,
                          pose_prior_weight, betas_weight, meas_targets, meas_weights, lambda_up, lambda_down, first,
                          rot, betas, transl, normal_matrix, gradient, meas, meas_jac, loss, lambda, accepted,
                          trial_rot, trial_betas, trial_transl, trial_vertices, trial_jac, trial_face_idx, trial_bary,
                          trial_nearest, trial_meas, trial_meas_jac, &pen, workspace, workspace_bytes, stream);
}
