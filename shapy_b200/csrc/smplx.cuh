// Shared declarations of the SMPL-X kernels (smplx.cu).
#pragma once
#include <map>
#include <mutex>

#include "common.cuh"

namespace shapy {

constexpr int kMaxJoints = 64;
constexpr int kMaxCoef = 32;

struct SmplxDev {
  int V, J, NB, NE, NC, F, L, D, rows, K, n_chain, n_levels, ell_w_n, n_extra, n_over;
  float *v_template, *posedirs /* [(J-1)*9][3V], the source of the pose-blend GEMM weights */;
  float *basis;   /* [NC][V3p]: shape then expression blend-shape rows, 16-byte aligned rows */
  int V3p;
  float *J_template /* [3J] */, *J_dirs /* [3J][NC] */;
  int *ell_idx;   /* [W][V] */
  float *ell_w;   /* [W][V] */
  int *parents, *level_joints, *level_off; /* level_off[n_levels+1] */
  int *faces;     /* [F][3] */
  int *lmk_vidx;  /* [L][3] */
  float *lmk_bc;  /* [L][3] */
  int *dyn_vidx;  /* [rows][D][3] */
  float *dyn_bc;  /* [rows][D][3] */
  int *neck;      /* [n_chain] */
  int *ex_ptr, *ex_col;
  float *ex_val;
  int *over_src, *over_tgt;
  // backward only: per-joint skinning lists (CSR over joints, vertices ascending) for the skinning-transform adjoint,
  // and per-vertex keypoint entries (CSR over vertices) that gather the landmark and J14 cotangents onto a vertex;
  // an entry's slot indexes [static landmarks | dynamic landmarks | J14 rows], row >= 0 only for a dynamic landmark
  // of that LUT row
  int *jv_ptr, *jv_idx;
  float *jv_w;
  int *vk_ptr, *vk_slot, *vk_row;
  float *vk_w;
};

}  // namespace shapy

struct shapy_smplx {
  shapy::SmplxDev d;
  std::vector<void *> allocs;
  // pose blend on the tensor cores (wgmma), the only place the pose blend runs: posedirs^T x kPoseScale as split-fp16
  // [V3g][Kpad] weights, built on first use per padded pose-feature width Kpad (joints >= n_rot contribute exact
  // zeros, so a call's GEMM stops at its Kpad), and a zero bias
  struct PoseW { __half *hi = nullptr, *lo = nullptr; };
  mutable std::mutex pw_mu;
  mutable std::map<int, PoseW> pw;
  float *zero_bias = nullptr;   // [V3g]
  int extra_nnz = 0;            // non-zeros of the J14 regressor (host copy of ex_ptr[n_extra])
};

namespace shapy {
constexpr float kPoseScale = 1024.0f;   // posedirs entries (~1e-3) are scaled into fp16's normal range
constexpr int kPoseKAlign = 16;         // pose-feature width padding (wgmma K granularity)
constexpr int kPoseV3Align = 384;       // 3V padding: a multiple of every cout tile of the wgmma engine
}  // namespace shapy

