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
