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
  // 4. Cholesky A = L L^T, right-looking: column j scaled, then the trailing lower triangle updated
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

template <bool MEAS>
int launch_lm_kp(int batch, const LmKpArgs &a, const LmMeasArgs &m, void *stream) {
  const size_t smem = (size_t)a.P * a.P * sizeof(double);
  // past 48 KB of static plus dynamic shared memory the launch has to opt in
  cudaFuncAttributes attr;
  SHAPY_CUDA_TRY(cudaFuncGetAttributes(&attr, lm_kp_step_kernel<MEAS>));
  if (smem + attr.sharedSizeBytes > 48 * 1024)
    SHAPY_CUDA_TRY(cudaFuncSetAttribute(lm_kp_step_kernel<MEAS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)smem));
  lm_kp_step_kernel<MEAS><<<batch, kLmKpThreads, smem, (cudaStream_t)stream>>>(a, m);
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
  return launch_lm_kp<false>(batch, a, LmMeasArgs{}, stream);
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
  return launch_lm_kp<true>(batch, a, m, stream);
}
