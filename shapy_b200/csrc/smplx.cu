// Fused SMPL-X body-model evaluation for sm_90a.
//
// Replaces the ~90-launch reference chain (blend_shapes -> vertices2joints -> pose blend ->
// batch_rigid_transform (54 serial bmm) -> skinning -> landmarks -> J14), reference
// regressor/human_shape/models/body_models/lbs.py:99-295 and body_models.py:628-767, by four
// launches:
//   smplx_pose_kernel    per body: joints from the (pre-contracted, exact) J_template + J_dirs . beta,
//                        level-parallel kinematic chain, A = G - [0 | G . J], the pose feature as the
//                        split-fp16 input of the pose-blend GEMM, contour LUT row
//   pose-blend GEMM      (R[1:] - I) . posedirs of all bodies on the wgmma engine (pose_blend_gemm)
//   smplx_vertex_kernel  tile of 32 vertices x 32 bodies: shape (+ expression) blend (constants staged
//                        through shared memory once per tile, reused by all 32 bodies), plus the GEMM's
//                        pose offsets, sparse skinning
//   smplx_joints_kernel  per body: landmarks, sparse J14 regressor + overwrite, weak-perspective camera
// plus smplx_shape_kernel for the T-pose path (SMPL.forward_shape, body_models.py:292-302), and the adjoints of both
// (shapy_smplx_backward, shapy_smplx_backward_shape, shapy_decode_rot6d_backward; see "posed backward" below).
//
// Exact structure that is exploited (changes summation order only):
//   * J = J_regressor . (T + S.beta) = J_regressor.T + (J_regressor.S).beta  (contracted once, in fp64)
//   * joints >= n_rot are identity => their pose-feature columns are exactly 0 and are left out of the GEMM
//   * lbs_weights and the J14 regressor are stored sparse (ELL / CSR); zero entries contribute exactly 0
#include <algorithm>
#include <cmath>
#include <cstring>

#include "conv.cuh"
#include "smplx.cuh"

namespace shapy {

constexpr int TV = 32;  // vertices per tile (one per lane)
constexpr int TB = 32;  // bodies per tile (8 per warp, 4 warps)
constexpr int KC = 32;  // blend-shape rows staged per chunk

// ----------------------------------------------------------------------------------------------
__global__ void decode_rot6d_kernel(const float *__restrict__ raw, int n, float *__restrict__ rot) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float *x = raw + 6 * (size_t)i;
  // row-major 3x2: column 0 = x[0], x[2], x[4]; column 1 = x[1], x[3], x[5]  (pose_utils.py:138-153)
  float a0 = x[0], a1 = x[2], a2 = x[4], c0 = x[1], c1 = x[3], c2 = x[5];
  float n1 = fmaxf(sqrtf(a0 * a0 + a1 * a1 + a2 * a2), 1e-12f);
  float b10 = a0 / n1, b11 = a1 / n1, b12 = a2 / n1;
  float d = b10 * c0 + b11 * c1 + b12 * c2;
  float u0 = c0 - d * b10, u1 = c1 - d * b11, u2 = c2 - d * b12;
  float n2 = fmaxf(sqrtf(u0 * u0 + u1 * u1 + u2 * u2), 1e-12f);
  float b20 = u0 / n2, b21 = u1 / n2, b22 = u2 / n2;
  float b30 = b11 * b22 - b12 * b21, b31 = b12 * b20 - b10 * b22, b32 = b10 * b21 - b11 * b20;
  float *R = rot + 9 * (size_t)i;  // columns b1 b2 b3
  R[0] = b10; R[1] = b20; R[2] = b30;
  R[3] = b11; R[4] = b21; R[5] = b31;
  R[6] = b12; R[7] = b22; R[8] = b32;
}

// ----------------------------------------------------------------------------------------------
struct PoseArgs {
  SmplxDev m;
  const float *betas, *expr, *rot;
  int n_rot, B, Bpad, Kp, Kpad;
  float *A, *pfT, *joints;  // joints may be null
  int *lut;
  __half *x_hi, *x_lo;      // pose-blend GEMM input [B][Kpad]; null when no GEMM runs
};

// Per body: blend coefficients [betas | expression], rotations (identity past n_rot), rest joints
// J = J_template + J_dirs . coef and the world transforms G = [G.R | G.t] of the kinematic chain, level by level.
// Shared by smplx_pose_kernel and smplx_chain_bwd_kernel, so the backward walks the same G bit for bit.
__device__ __forceinline__ void body_chain(const SmplxDev &m, const float *betas, const float *expr, const float *rot,
                                           int n_rot, int b, float (*R)[9], float (*Jr)[3], float (*G)[12],
                                           float *coef) {
  const int t = threadIdx.x;
  const int J = m.J;
  if (t < m.NC) coef[t] = t < m.NB ? betas[(size_t)b * m.NB + t] : (expr ? expr[(size_t)b * m.NE + (t - m.NB)] : 0.f);
  for (int i = t; i < J * 9; i += blockDim.x) {
    int j = i / 9, e = i % 9;
    R[j][e] = j < n_rot ? rot[((size_t)b * n_rot + j) * 9 + e] : ((e == 0 || e == 4 || e == 8) ? 1.f : 0.f);
  }
  __syncthreads();
  for (int i = t; i < J * 3; i += blockDim.x) {
    float s = m.J_template[i];
    const float *jd = m.J_dirs + (size_t)i * m.NC;
    for (int l = 0; l < m.NC; ++l) s += jd[l] * coef[l];
    Jr[i / 3][i % 3] = s;
  }
  __syncthreads();
  if (t < 12) {
    int r = t / 4, c = t % 4;
    G[0][t] = c < 3 ? R[0][r * 3 + c] : Jr[0][r];
  }
  __syncthreads();
  for (int lv = 1; lv < m.n_levels; ++lv) {
    int off = m.level_off[lv], cnt = m.level_off[lv + 1] - off;
    for (int i = t; i < cnt * 12; i += blockDim.x) {
      int j = m.level_joints[off + i / 12], e = i % 12, r = e / 4, c = e % 4;
      int p = m.parents[j];
      float g0 = G[p][r * 4 + 0], g1 = G[p][r * 4 + 1], g2 = G[p][r * 4 + 2];
      float v;
      if (c < 3) {
        v = g0 * R[j][c] + g1 * R[j][3 + c] + g2 * R[j][6 + c];
      } else {
        float r0 = Jr[j][0] - Jr[p][0], r1 = Jr[j][1] - Jr[p][1], r2 = Jr[j][2] - Jr[p][2];
        v = g0 * r0 + g1 * r1 + g2 * r2 + G[p][r * 4 + 3];
      }
      G[j][e] = v;
    }
    __syncthreads();
  }
}

// Dynamic-contour LUT row of a body from its rotations (lbs.py:30-41, rotation_utils.py:86-92).  Shared by
// smplx_pose_kernel and smplx_kp_jac_kernel, so both pick the same row.
__device__ __forceinline__ int contour_lut_row(const SmplxDev &m, const float (*R)[9]) {
  float rel[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  for (int q = 0; q < m.n_chain; ++q) {
    const float *Rq = R[m.neck[q]];
    float o[9];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) o[r * 3 + c] = Rq[r * 3] * rel[c] + Rq[r * 3 + 1] * rel[3 + c] + Rq[r * 3 + 2] * rel[6 + c];
    for (int e = 0; e < 9; ++e) rel[e] = o[e];
  }
  float sy = sqrtf(rel[0] * rel[0] + rel[3] * rel[3]);
  float ang = atan2f(-rel[6], sy);
  float deg = fminf(-ang * 180.0f / 3.14159265358979323846f, 39.0f);
  int y = (int)rintf(deg);  // torch.round == round-half-even
  int row = y < 0 ? (y < -39 ? 78 : 39 - y) : y;
  return min(max(row, 0), m.rows - 1);
}

__global__ void __launch_bounds__(128) smplx_pose_kernel(PoseArgs a) {
  const SmplxDev &m = a.m;
  const int b = blockIdx.x, t = threadIdx.x;
  __shared__ float R[kMaxJoints][9];
  __shared__ float Jr[kMaxJoints][3];
  __shared__ float G[kMaxJoints][12];
  __shared__ float coef[kMaxCoef];
  const int J = m.J;
  body_chain(m, a.betas, a.expr, a.rot, a.n_rot, b, R, Jr, G, coef);
  // relative transforms A = G - [0 | G.R . J_rest]   (lbs.py:289-293)
  for (int i = t; i < J * 12; i += blockDim.x) {
    int j = i / 12, e = i % 12, r = e / 4, c = e % 4;
    float v = G[j][e];
    if (c == 3) v -= G[j][r * 4 + 0] * Jr[j][0] + G[j][r * 4 + 1] * Jr[j][1] + G[j][r * 4 + 2] * Jr[j][2];
    a.A[((size_t)b * J + j) * 12 + e] = v;
  }
  if (a.joints) {
    for (int i = t; i < J * 3; i += blockDim.x) a.joints[((size_t)b * m.K) * 3 + i] = G[i / 3][(i % 3) * 4 + 3];
  }
  // blend coefficients of this body, one row per basis row [betas | expression], transposed: a body tile is contiguous
  if (t < m.NC) a.pfT[(size_t)t * a.Bpad + b] = coef[t];
  // pose feature (R[1:] - I) / kPoseScale as the split-fp16 GEMM input row of this body, zero-padded to Kpad
  if (a.x_hi) {
    __half *xh = a.x_hi + (size_t)b * a.Kpad, *xl = a.x_lo + (size_t)b * a.Kpad;
    for (int k = t; k < a.Kpad; k += blockDim.x) {
      int j = 1 + k / 9, e = k % 9;
      const float x = k < a.Kp ? (R[j][e] - ((e == 0 || e == 4 || e == 8) ? 1.f : 0.f)) * (1.0f / kPoseScale) : 0.f;
      split_store(x, xh[k], xl[k]);
    }
  }
  if (t == 0 && m.D > 0) a.lut[b] = contour_lut_row(m, R);
}

// ----------------------------------------------------------------------------------------------
struct VertexArgs {
  SmplxDev m;
  const float *betas, *expr;
  const float *A, *pfT;
  int B, Bpad;
  float *vertices, *v_shaped;  // either may be null
  const __half *pb_hi, *pb_lo;  // pose blend [B][pb_ld] as hi + lo / 2048 (wgmma GEMM); null: none (n_rot 1, or no vertices)
  int pb_ld;
};

__device__ __forceinline__ void cp_async16_zfill(void *smem_dst, const void *src, int src_bytes) {
  unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(src), "r"(src_bytes) : "memory");
}

// posedirs [KP][V3] fp32 -> split-fp16 GEMM weights [V3g][Kpad] (the [cout][cin] layout of a 1x1 convolution), x kPoseScale.
// Every real posedirs row below Kpad is packed (KP = 9 (J - 1), all of them), not only the Kp rows of the call that
// builds the entry: the weights are cached per Kpad, and every pose width that rounds to this Kpad reuses them.
__global__ void pack_pose_weights_kernel(const float *__restrict__ posedirs, int V3, int KP, int Kpad, int V3g,
                                         __half *__restrict__ hi, __half *__restrict__ lo) {
  const size_t n = (size_t)V3g * Kpad;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i / Kpad), k = (int)(i % Kpad);
    const float x = (c < V3 && k < KP) ? posedirs[(size_t)k * V3 + c] * kPoseScale : 0.f;
    split_store(x, hi[i], lo[i]);
  }
}

// One tile = 32 vertices (one per lane) x 32 bodies (8 per warp).  The shape and expression blend-shape rows
// are one [rows][V3p] basis; a chunk of 32 rows (96 floats each) and the matching [rows][32 bodies] coefficient
// block are staged in shared memory with 16-byte cp.async, double buffered, so every constant crosses L2 once
// per tile and the loads of chunk i+1 overlap the FMAs of chunk i.
//
// v_posed of one tile, in acc[body][xyz]: the shape (+ expression) blend and, when posed, the pose-blend GEMM's
// offsets; v_shaped is written after the shape rows when asked.  The forward vertex kernel and the backward
// (smplx_vertex_bwd_kernel) both compute v_posed here, so they see the same bits.  Every thread of the CTA calls it.
__device__ __forceinline__ void tile_v_posed(const VertexArgs &a, bool posed, float (&acc)[8][3],
                                             float (&Ps)[2][KC][TV * 3], float (&pfs)[2][KC][TB]) {
  const SmplxDev &m = a.m;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, t = threadIdx.x;
  const int v0 = blockIdx.x * TV, b0 = blockIdx.y * TB;
  const int c0 = v0 * 3;
  const int v = v0 + lane;
  const bool vok = v < m.V;
  {
    float tx = 0.f, ty = 0.f, tz = 0.f;
    if (vok) { tx = m.v_template[3 * v]; ty = m.v_template[3 * v + 1]; tz = m.v_template[3 * v + 2]; }
#pragma unroll
    for (int i = 0; i < 8; ++i) { acc[i][0] = tx; acc[i][1] = ty; acc[i][2] = tz; }
  }
  // row schedule: [0, NB) shape | [NB, NC) expression (only when given, and only for vertices)
  const int n_rows = (a.expr && posed) ? m.NC : m.NB;
  // chunk boundaries: the first chunk ends exactly after the NB shape rows (v_shaped snapshot)
  auto chunk_begin = [&](int ch) { return ch == 0 ? 0 : m.NB + (ch - 1) * KC; };
  const int n_chunks = 1 + (n_rows > m.NB ? (n_rows - m.NB + KC - 1) / KC : 0);
  auto load_chunk = [&](int ch, int buf) {
    const int r0 = chunk_begin(ch), r1 = min(n_rows, ch == 0 ? m.NB : r0 + KC);
    const int nr = r1 - r0;
    for (int i = t; i < nr * 24; i += 128) {            // 96 floats = 24 x 16 bytes per row
      const int k = i / 24, q = i % 24;
      const int col = c0 + q * 4;
      const int nb = max(0, min(16, (m.V3p - col) * 4));
      const float *src = m.basis + (size_t)(r0 + k) * m.V3p + (nb ? col : 0);
      cp_async16_zfill(&Ps[buf][k][q * 4], src, nb);
    }
    for (int i = t; i < nr * 8; i += 128) {             // 32 bodies = 8 x 16 bytes per row
      const int k = i / 8, q = i % 8;
      cp_async16_zfill(&pfs[buf][k][q * 4], a.pfT + (size_t)(r0 + k) * a.Bpad + b0 + q * 4, 16);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  load_chunk(0, 0);
  for (int ch = 0; ch < n_chunks; ++ch) {
    const int buf = ch & 1;
    if (ch + 1 < n_chunks) {
      load_chunk(ch + 1, buf ^ 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    const int r0 = chunk_begin(ch), nr = min(n_rows, ch == 0 ? m.NB : r0 + KC) - r0;
#pragma unroll 4
    for (int k = 0; k < nr; ++k) {
      const float px = Ps[buf][k][3 * lane], py = Ps[buf][k][3 * lane + 1], pz = Ps[buf][k][3 * lane + 2];
      const float4 f0 = *reinterpret_cast<const float4 *>(&pfs[buf][k][warp * 8]);
      const float4 f1 = *reinterpret_cast<const float4 *>(&pfs[buf][k][warp * 8 + 4]);
      const float f[8] = {f0.x, f0.y, f0.z, f0.w, f1.x, f1.y, f1.z, f1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        acc[i][0] += f[i] * px; acc[i][1] += f[i] * py; acc[i][2] += f[i] * pz;
      }
    }
    if (ch == 0 && a.v_shaped && vok) {
      // v_shaped = v_template + shapedirs[:, :, :NB] . betas  (body_models.py:763-765)
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int b = b0 + warp * 8 + i;
        if (b < a.B) {
          float *o = a.v_shaped + ((size_t)b * m.V + v) * 3;
          o[0] = acc[i][0]; o[1] = acc[i][1]; o[2] = acc[i][2];
        }
      }
    }
    __syncthreads();
  }
  if (posed && vok && a.pb_hi) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int b = b0 + warp * 8 + i;
      if (b >= a.B) break;
      const size_t o = (size_t)b * a.pb_ld + 3 * v;
#pragma unroll
      for (int c = 0; c < 3; ++c) acc[i][c] += __half2float(a.pb_hi[o + c]) + __half2float(a.pb_lo[o + c]) * kLoInv;
    }
  }
}

__global__ void __launch_bounds__(128) smplx_vertex_kernel(VertexArgs a) {
  const SmplxDev &m = a.m;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int v = blockIdx.x * TV + lane, b0 = blockIdx.y * TB;
  __shared__ __align__(16) float Ps[2][KC][TV * 3];
  __shared__ __align__(16) float pfs[2][KC][TB];
  float acc[8][3];
  const bool posed = a.vertices != nullptr;
  tile_v_posed(a, posed, acc, Ps, pfs);
  if (!posed || v >= m.V) return;
  // ---- sparse linear blend skinning: out = sum_j w_vj (A_j . [v_posed; 1])
  float out[8][3];
#pragma unroll
  for (int i = 0; i < 8; ++i) out[i][0] = out[i][1] = out[i][2] = 0.f;
  for (int s = 0; s < m.ell_w_n; ++s) {
    float w = m.ell_w[(size_t)s * m.V + v];
    if (w == 0.f) continue;
    int j = m.ell_idx[(size_t)s * m.V + v];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      int b = b0 + warp * 8 + i;
      if (b >= a.B) break;
      const float4 *Ab = reinterpret_cast<const float4 *>(a.A + ((size_t)b * m.J + j) * 12);
      float4 r0 = __ldg(Ab), r1 = __ldg(Ab + 1), r2 = __ldg(Ab + 2);
      float x = acc[i][0], y = acc[i][1], z = acc[i][2];
      out[i][0] += w * (r0.x * x + r0.y * y + r0.z * z + r0.w);
      out[i][1] += w * (r1.x * x + r1.y * y + r1.z * z + r1.w);
      out[i][2] += w * (r2.x * x + r2.y * y + r2.z * z + r2.w);
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int b = b0 + warp * 8 + i;
    if (b < a.B) {
      float *o = a.vertices + ((size_t)b * m.V + v) * 3;
      o[0] = out[i][0]; o[1] = out[i][1]; o[2] = out[i][2];
    }
  }
}

// ----------------------------------------------------------------------------------------------
struct JointsArgs {
  SmplxDev m;
  const float *vertices, *camera;
  const int *lut;
  int B;
  float *joints, *proj;
};

__global__ void __launch_bounds__(512) smplx_joints_kernel(JointsArgs a) {
  // launched as a programmatic dependent of the kernel that writes the vertices: its launch latency overlaps that
  // kernel's tail; everything below reads the predecessor's output, so wait for its completion first
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const SmplxDev &m = a.m;
  const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  extern __shared__ float sm[];
  float *jt = sm;               // [K][3]
  float *reg = sm + m.K * 3;    // [n_extra][3]
  const float *vb = a.vertices + (size_t)b * m.V * 3;
  float *jout = a.joints + (size_t)b * m.K * 3;
  for (int i = t; i < m.J * 3; i += blockDim.x) jt[i] = jout[i];  // posed joints from the pose kernel
  for (int i = t; i < m.L + m.D; i += blockDim.x) {
    const int *vi;
    const float *bc;
    if (i < m.L) { vi = m.lmk_vidx + 3 * i; bc = m.lmk_bc + 3 * i; }
    else {
      size_t o = ((size_t)a.lut[b] * m.D + (i - m.L)) * 3;
      vi = m.dyn_vidx + o; bc = m.dyn_bc + o;
    }
    for (int c = 0; c < 3; ++c)
      jt[(m.J + i) * 3 + c] = vb[3 * vi[0] + c] * bc[0] + vb[3 * vi[1] + c] * bc[1] + vb[3 * vi[2] + c] * bc[2];
  }
  for (int r = warp; r < m.n_extra; r += blockDim.x / 32) {
    float sx = 0.f, sy = 0.f, sz = 0.f;
    for (int e = m.ex_ptr[r] + lane; e < m.ex_ptr[r + 1]; e += 32) {
      int c = m.ex_col[e];
      float w = m.ex_val[e];
      sx += w * vb[3 * c]; sy += w * vb[3 * c + 1]; sz += w * vb[3 * c + 2];
    }
    for (int o = 16; o; o >>= 1) {
      sx += __shfl_xor_sync(0xffffffffu, sx, o);
      sy += __shfl_xor_sync(0xffffffffu, sy, o);
      sz += __shfl_xor_sync(0xffffffffu, sz, o);
    }
    if (lane == 0) { reg[3 * r] = sx; reg[3 * r + 1] = sy; reg[3 * r + 2] = sz; }
  }
  __syncthreads();
  for (int i = t; i < m.n_over * 3; i += blockDim.x) {
    int q = i / 3, c = i % 3;
    jt[m.over_src[q] * 3 + c] = reg[m.over_tgt[q] * 3 + c];
  }
  __syncthreads();
  for (int i = t; i < m.K * 3; i += blockDim.x) jout[i] = jt[i];
  if (a.proj && a.camera) {
    float c0 = a.camera[3 * b];
    float s = c0 > 20.f ? c0 : log1pf(expf(c0));  // F.softplus (beta=1, threshold=20)
    float tx = a.camera[3 * b + 1], ty = a.camera[3 * b + 2];
    for (int i = t; i < m.K; i += blockDim.x) {
      a.proj[((size_t)b * m.K + i) * 2 + 0] = s * (jt[3 * i] + tx);
      a.proj[((size_t)b * m.K + i) * 2 + 1] = s * (jt[3 * i + 1] + ty);
    }
  }
}

// ----------------------------------------------------------------------------------------------
// T-pose path: v_shaped[b][c] = T[c] + sum_l beta[b][l] S[l][c], S = the shape rows of the basis (row pitch ld).
// One thread per coordinate, the NB shape coefficients of that coordinate live in registers and are reused for SB
// bodies, so the only HBM traffic is the (B, 3V) output stream (S and T are 1.4 MB and stay in L2).
constexpr int SB = 64;
constexpr int SBP = 12;   // padded beta row (float4 x 3) so a body's coefficients are 3 broadcast LDS.128
template <int NB>
__global__ void __launch_bounds__(256) smplx_shape_kernel(const float *__restrict__ T, const float *__restrict__ S,
                                                          int ld, const float *__restrict__ betas, int V3, int B,
                                                          float *__restrict__ out) {
  static_assert(NB <= SBP, "beta row padding");
  __shared__ __align__(16) float bs[SB][SBP];
  // two coordinates per thread (c and c + 256): the same 3 LDS.128 of betas feed 20 FMAs
  const int c0 = blockIdx.x * 512 + threadIdx.x, c1 = c0 + 256;
  const int b0 = blockIdx.y * SB;
  for (int i = threadIdx.x; i < SB * SBP; i += blockDim.x) {
    int b = b0 + i / SBP, l = i % SBP;
    bs[i / SBP][l] = (b < B && l < NB) ? betas[(size_t)b * NB + l] : 0.f;
  }
  float s0[SBP], s1[SBP], t0 = 0.f, t1 = 0.f;
#pragma unroll
  for (int l = 0; l < SBP; ++l) { s0[l] = 0.f; s1[l] = 0.f; }
  if (c0 < V3) {
    t0 = T[c0];
#pragma unroll
    for (int l = 0; l < NB; ++l) s0[l] = S[(size_t)l * ld + c0];
  }
  if (c1 < V3) {
    t1 = T[c1];
#pragma unroll
    for (int l = 0; l < NB; ++l) s1[l] = S[(size_t)l * ld + c1];
  }
  __syncthreads();
  const int nb = min(SB, B - b0);
  float *o = out + (size_t)b0 * V3;
#pragma unroll 2
  for (int i = 0; i < nb; ++i) {
    const float4 q0 = *reinterpret_cast<const float4 *>(&bs[i][0]);
    const float4 q1 = *reinterpret_cast<const float4 *>(&bs[i][4]);
    const float4 q2 = *reinterpret_cast<const float4 *>(&bs[i][8]);
    const float bb[SBP] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w, q2.x, q2.y, q2.z, q2.w};
    float v0 = t0, v1 = t1;
#pragma unroll
    for (int l = 0; l < NB; ++l) { v0 += bb[l] * s0[l]; v1 += bb[l] * s1[l]; }
    if (c0 < V3) __stcs(o + (size_t)i * V3 + c0, v0);
    if (c1 < V3) __stcs(o + (size_t)i * V3 + c1, v1);
  }
}

__global__ void smplx_shape_kernel_generic(const float *__restrict__ T, const float *__restrict__ S, int ld,
                                           const float *__restrict__ betas, int NB, int V3, int B,
                                           float *__restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (c >= V3) return;
  float v = T[c];
  for (int l = 0; l < NB; ++l) v += betas[(size_t)b * NB + l] * S[(size_t)l * ld + c];
  out[(size_t)b * V3 + c] = v;
}

// Adjoint of the blend shapes: part of grad_coef[b][l] = sum_c S[l][c] g[b][c] over the NB shape rows and the NE
// expression rows that follow them in the basis.  g = gv for every row, plus gv2 (when given) for the shape rows only:
// the posed backward passes the cotangent of v_posed as gv and that of v_shaped, which carries no expression
// (body_models.py:763-765), as gv2; the T-pose path passes gv alone with NE = 0.  The 3V coordinates are cut into
// kShapeSplit fixed chunks; CTA (tile, chunk) writes the partial sums of its bodies over its chunk (per thread over a
// fixed stride, then a fixed xor tree and a fixed order over warps) and smplx_shape_bwd_sum_kernel adds the chunks in
// order.  Neither the chunking nor the order depends on B or on a body's place in the batch, so a body's gradient is
// bit-identical alone and in any batch.  HBM traffic is the (B, 3V) gradient read once (S stays in L2, read once per
// TILE bodies).
constexpr int kShapeSplit = 16;
constexpr int kShapeTile = 8;
template <int NB, int NE, int TILE>
__global__ void __launch_bounds__(256) smplx_shape_bwd_kernel(const float *__restrict__ S, int ld,
                                                              const float *__restrict__ gv,
                                                              const float *__restrict__ gv2, int V3, int B,
                                                              float *__restrict__ part) {
  constexpr int NR = NB + NE;
  const int b0 = blockIdx.x * TILE, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int nb = min(TILE, B - b0);
  const int chunk = (V3 + kShapeSplit - 1) / kShapeSplit, c_lo = blockIdx.y * chunk, c_hi = min(V3, c_lo + chunk);
  float acc[TILE][NR];
#pragma unroll
  for (int i = 0; i < TILE; ++i)
#pragma unroll
    for (int l = 0; l < NR; ++l) acc[i][l] = 0.f;
  for (int c = c_lo + t; c < c_hi; c += 256) {
    float s[NR];
#pragma unroll
    for (int l = 0; l < NR; ++l) s[l] = __ldg(S + (size_t)l * ld + c);
#pragma unroll
    for (int i = 0; i < TILE; ++i) {
      if (i < nb) {
        const float g = __ldcs(gv + (size_t)(b0 + i) * V3 + c);
        const float gs = gv2 ? g + __ldcs(gv2 + (size_t)(b0 + i) * V3 + c) : g;
#pragma unroll
        for (int l = 0; l < NR; ++l) acc[i][l] += (l < NB ? gs : g) * s[l];
      }
    }
  }
  __shared__ float red[8][TILE * NR];
#pragma unroll
  for (int i = 0; i < TILE; ++i)
#pragma unroll
    for (int l = 0; l < NR; ++l) {
      float v = acc[i][l];
      for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) red[warp][i * NR + l] = v;
    }
  __syncthreads();
  for (int r = t; r < nb * NR; r += 256) {
    float v = 0.f;
    for (int w = 0; w < 8; ++w) v += red[w][r];
    part[((size_t)(b0 + r / NR) * kShapeSplit + blockIdx.y) * NR + r % NR] = v;
  }
}

// any row count: CTA (body, chunk, l), l < NR; gv2 adds to the rows below NB
__global__ void __launch_bounds__(256) smplx_shape_bwd_kernel_generic(const float *__restrict__ S, int ld,
                                                                      const float *__restrict__ gv,
                                                                      const float *__restrict__ gv2, int NB, int NR,
                                                                      int V3, float *__restrict__ part) {
  const int b = blockIdx.x, l = blockIdx.z, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int chunk = (V3 + kShapeSplit - 1) / kShapeSplit, c_lo = blockIdx.y * chunk, c_hi = min(V3, c_lo + chunk);
  const float *g2 = (gv2 && l < NB) ? gv2 : nullptr;
  float v = 0.f;
  for (int c = c_lo + t; c < c_hi; c += 256) {
    const float g = __ldg(gv + (size_t)b * V3 + c);
    v += (g2 ? g + __ldg(g2 + (size_t)b * V3 + c) : g) * __ldg(S + (size_t)l * ld + c);
  }
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __shared__ float red[8];
  if (lane == 0) red[warp] = v;
  __syncthreads();
  if (t == 0) {
    float s = 0.f;
    for (int w = 0; w < 8; ++w) s += red[w];
    part[((size_t)b * kShapeSplit + blockIdx.y) * NR + l] = s;
  }
}

__global__ void smplx_shape_bwd_sum_kernel(const float *__restrict__ part, int NB, int B, float *__restrict__ gb) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= B * NB) return;
  const int b = r / NB, l = r % NB;
  float v = 0.f;
  for (int s = 0; s < kShapeSplit; ++s) v += part[((size_t)b * kShapeSplit + s) * NB + l];
  gb[r] = v;
}

// ============================================================================================== posed backward
// Adjoint of shapy_smplx_forward, first order, with the reference's autograd semantics (DESIGN.md §6b).  It recomputes
// the forward from its inputs (smplx_pose_kernel and the pose-blend GEMM give A, the LUT rows and the pose offsets bit
// for bit; tile_v_posed gives v_posed), then runs the adjoints below.  No float atomics: every sum has a fixed order
// that does not depend on B or on a body's place in the batch.

// 6D decoder: the adjoint of decode_rot6d_kernel's Gram-Schmidt.  clamp_min(norm, 1e-12) passes the gradient to the
// norm only where norm >= 1e-12, as torch's clamp_min does under autograd.
__global__ void decode_rot6d_bwd_kernel(const float *__restrict__ raw, int n, const float *__restrict__ grot,
                                        float *__restrict__ graw) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float *x = raw + 6 * (size_t)i;
  const float *G = grot + 9 * (size_t)i;
  float a[3] = {x[0], x[2], x[4]}, c[3] = {x[1], x[3], x[5]};
  const float n1r = sqrtf(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]), n1 = fmaxf(n1r, 1e-12f);
  float b1[3], u[3], b2[3];
  for (int k = 0; k < 3; ++k) b1[k] = a[k] / n1;
  const float d = b1[0] * c[0] + b1[1] * c[1] + b1[2] * c[2];
  for (int k = 0; k < 3; ++k) u[k] = c[k] - d * b1[k];
  const float n2r = sqrtf(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]), n2 = fmaxf(n2r, 1e-12f);
  for (int k = 0; k < 3; ++k) b2[k] = u[k] / n2;
  // R = [b1 b2 b3] by columns
  float g1[3] = {G[0], G[3], G[6]}, g2[3] = {G[1], G[4], G[7]}, g3[3] = {G[2], G[5], G[8]};
  // b3 = b1 x b2
  g1[0] += b2[1] * g3[2] - b2[2] * g3[1]; g1[1] += b2[2] * g3[0] - b2[0] * g3[2]; g1[2] += b2[0] * g3[1] - b2[1] * g3[0];
  g2[0] += g3[1] * b1[2] - g3[2] * b1[1]; g2[1] += g3[2] * b1[0] - g3[0] * b1[2]; g2[2] += g3[0] * b1[1] - g3[1] * b1[0];
  // b2 = u / n2
  float gu[3];
  const float gn2 = -(g2[0] * u[0] + g2[1] * u[1] + g2[2] * u[2]) / (n2 * n2);
  for (int k = 0; k < 3; ++k) gu[k] = g2[k] / n2 + (n2r >= 1e-12f ? gn2 * u[k] / n2r : 0.f);
  // u = c - d b1, d = b1 . c
  const float gd = -(gu[0] * b1[0] + gu[1] * b1[1] + gu[2] * b1[2]);
  float gc[3];
  for (int k = 0; k < 3; ++k) {
    gc[k] = gu[k] + gd * b1[k];
    g1[k] += -d * gu[k] + gd * c[k];
  }
  // b1 = a / n1
  float ga[3];
  const float gn1 = -(g1[0] * a[0] + g1[1] * a[1] + g1[2] * a[2]) / (n1 * n1);
  for (int k = 0; k < 3; ++k) ga[k] = g1[k] / n1 + (n1r >= 1e-12f ? gn1 * a[k] / n1r : 0.f);
  float *o = graw + 6 * (size_t)i;
  o[0] = ga[0]; o[1] = gc[0]; o[2] = ga[1]; o[3] = gc[1]; o[4] = ga[2]; o[5] = gc[2];
}

// Joints backward, per body: the cotangent of the keypoints (joints + the proj_joints term), the camera gradient, the
// J14 routing (an overwritten keypoint's cotangent goes to its J14 row, the joint or landmark it replaced gets none),
// and the split into posed-joint cotangents gP [B][J][3] and landmark / J14 cotangents gkp [B][nkp][3].
struct JointsBwdArgs {
  SmplxDev m;
  const float *joints;            // forward joints [B][K][3]; read only for the camera gradient
  const float *camera, *g_joints, *g_proj;
  float *gP, *gkp, *g_camera;
};

__global__ void __launch_bounds__(128) smplx_joints_bwd_kernel(JointsBwdArgs a) {
  const SmplxDev &m = a.m;
  const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  extern __shared__ float sm[];
  float *gj = sm;                 // [K][3]
  float *greg = sm + m.K * 3;     // [n_extra][3]
  const int nkp = m.L + m.D + m.n_extra;
  const float *gproj = a.camera ? a.g_proj : nullptr;
  float s = 0.f, c0 = 0.f;
  if (a.camera) {
    c0 = a.camera[3 * b];
    s = c0 > 20.f ? c0 : log1pf(expf(c0));
  }
  for (int i = t; i < m.K * 3; i += blockDim.x) {
    float g = a.g_joints ? a.g_joints[(size_t)b * m.K * 3 + i] : 0.f;
    if (gproj && i % 3 < 2) g += s * gproj[((size_t)b * m.K + i / 3) * 2 + i % 3];
    gj[i] = g;
  }
  for (int i = t; i < m.n_extra * 3; i += blockDim.x) greg[i] = 0.f;
  if (a.g_camera && warp == 0) {
    // proj = s (xy + t): d/ds = sum g (xy + t), d/dt = sum s g; ds/dc0 = sigmoid(c0), or 1 past softplus' threshold
    float gs = 0.f, gx = 0.f, gy = 0.f;
    if (gproj) {
      const float tx = a.camera[3 * b + 1], ty = a.camera[3 * b + 2];
      const float *jt = a.joints + (size_t)b * m.K * 3;
      for (int i = lane; i < m.K; i += 32) {
        const float px = gproj[((size_t)b * m.K + i) * 2], py = gproj[((size_t)b * m.K + i) * 2 + 1];
        gs += px * (jt[3 * i] + tx) + py * (jt[3 * i + 1] + ty);
        gx += s * px;
        gy += s * py;
      }
    }
    for (int o = 16; o; o >>= 1) {
      gs += __shfl_xor_sync(0xffffffffu, gs, o);
      gx += __shfl_xor_sync(0xffffffffu, gx, o);
      gy += __shfl_xor_sync(0xffffffffu, gy, o);
    }
    if (lane == 0) {
      a.g_camera[3 * b] = gs * (c0 > 20.f ? 1.f : 1.f / (1.f + expf(-c0)));
      a.g_camera[3 * b + 1] = gx;
      a.g_camera[3 * b + 2] = gy;
    }
  }
  __syncthreads();
  if (t == 0) {
    for (int q = 0; q < m.n_over; ++q)
      for (int c = 0; c < 3; ++c) greg[m.over_tgt[q] * 3 + c] += gj[m.over_src[q] * 3 + c];
    for (int q = 0; q < m.n_over; ++q)
      for (int c = 0; c < 3; ++c) gj[m.over_src[q] * 3 + c] = 0.f;
  }
  __syncthreads();
  if (!a.gP) return;
  for (int i = t; i < m.J * 3; i += blockDim.x) a.gP[(size_t)b * m.J * 3 + i] = gj[i];
  float *gk = a.gkp + (size_t)b * nkp * 3;
  for (int i = t; i < (m.L + m.D) * 3; i += blockDim.x) gk[i] = gj[m.J * 3 + i];
  for (int i = t; i < m.n_extra * 3; i += blockDim.x) gk[(m.L + m.D) * 3 + i] = greg[i];
}

// Vertex backward on the forward's tile of 32 vertices x 32 bodies: v_posed (tile_v_posed), the total vertex
// cotangent gv = grad_vertices + the landmark and J14 cotangents gathered through the per-vertex keypoint entries, and
// its pull-back through the skinning, gvp = sum_s w_s R_{A_s}^T gv.  Writes v_posed, gv and gvp, each [B][V][3].
struct VertexBwdArgs {
  VertexArgs f;                   // recompute of v_posed; f.vertices and f.v_shaped are unused
  const float *g_vertices, *gkp;  // either may be null (zero)
  const int *lut;
  float *vp, *gv, *gvp;
};

__global__ void __launch_bounds__(128) smplx_vertex_bwd_kernel(VertexBwdArgs a) {
  const SmplxDev &m = a.f.m;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int v = blockIdx.x * TV + lane, b0 = blockIdx.y * TB;
  __shared__ __align__(16) float Ps[2][KC][TV * 3];
  __shared__ __align__(16) float pfs[2][KC][TB];
  float acc[8][3];
  tile_v_posed(a.f, true, acc, Ps, pfs);
  if (v >= m.V) return;
  const int nkp = m.L + m.D + m.n_extra;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int b = b0 + warp * 8 + i;
    if (b >= a.f.B) break;
    const size_t o = ((size_t)b * m.V + v) * 3;
    a.vp[o] = acc[i][0]; a.vp[o + 1] = acc[i][1]; a.vp[o + 2] = acc[i][2];
    float g0 = 0.f, g1 = 0.f, g2 = 0.f;
    if (a.g_vertices) { g0 = a.g_vertices[o]; g1 = a.g_vertices[o + 1]; g2 = a.g_vertices[o + 2]; }
    if (a.gkp) {
      const int row = m.D ? a.lut[b] : -1;
      for (int e = m.vk_ptr[v]; e < m.vk_ptr[v + 1]; ++e) {
        const int r = m.vk_row[e];
        if (r >= 0 && r != row) continue;
        const float w = m.vk_w[e];
        const float *q = a.gkp + ((size_t)b * nkp + m.vk_slot[e]) * 3;
        g0 += w * q[0]; g1 += w * q[1]; g2 += w * q[2];
      }
    }
    a.gv[o] = g0; a.gv[o + 1] = g1; a.gv[o + 2] = g2;
    float h0 = 0.f, h1 = 0.f, h2 = 0.f;
    for (int s = 0; s < m.ell_w_n; ++s) {
      const float w = m.ell_w[(size_t)s * m.V + v];
      if (w == 0.f) continue;
      const int j = m.ell_idx[(size_t)s * m.V + v];
      const float4 *Ab = reinterpret_cast<const float4 *>(a.f.A + ((size_t)b * m.J + j) * 12);
      const float4 r0 = __ldg(Ab), r1 = __ldg(Ab + 1), r2 = __ldg(Ab + 2);
      h0 += w * (r0.x * g0 + r1.x * g1 + r2.x * g2);
      h1 += w * (r0.y * g0 + r1.y * g1 + r2.y * g2);
      h2 += w * (r0.z * g0 + r1.z * g1 + r2.z * g2);
    }
    a.gvp[o] = h0; a.gvp[o + 1] = h1; a.gvp[o + 2] = h2;
  }
}

// Skinning-transform adjoint: gA[b][j] = sum_v w_vj gv[b][v] (x) [v_posed[b][v]; 1], over the per-joint vertex list
// built in shapy_smplx_create.  One CTA per body, one warp per joint at a time: lanes stride the list, then a fixed
// xor tree.
__global__ void __launch_bounds__(256) smplx_skin_bwd_kernel(SmplxDev m, const float *__restrict__ gv,
                                                             const float *__restrict__ vp, float *__restrict__ gA) {
  const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float *gvb = gv + (size_t)b * m.V * 3, *vpb = vp + (size_t)b * m.V * 3;
  for (int j = warp; j < m.J; j += 8) {
    float acc[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) acc[k] = 0.f;
    for (int e = m.jv_ptr[j] + lane; e < m.jv_ptr[j + 1]; e += 32) {
      const int v = m.jv_idx[e];
      const float w = m.jv_w[e];
      const float g[3] = {w * gvb[3 * v], w * gvb[3 * v + 1], w * gvb[3 * v + 2]};
      const float p[3] = {vpb[3 * v], vpb[3 * v + 1], vpb[3 * v + 2]};
#pragma unroll
      for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[r * 4 + c] += g[r] * p[c];
        acc[r * 4 + 3] += g[r];
      }
    }
#pragma unroll
    for (int k = 0; k < 12; ++k) {
      float v = acc[k];
      for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      acc[k] = v;
    }
    if (lane < 12) {
      float v = acc[0];
#pragma unroll
      for (int k = 1; k < 12; ++k) v = lane == k ? acc[k] : v;
      gA[((size_t)b * m.J + j) * 12 + lane] = v;
    }
  }
}

// Pose-feature adjoint: part[b][split][k] = sum over chunk `split` of the 3V coordinates of P[k][c] gvp[b][c], k < Kp,
// from the fp32 posedirs rows (the rows past Kp multiply exact zeros).  A SIMT GEMM with a fixed split-K: the 3V
// coordinates are cut into kPfSplit chunks whatever B is, a CTA computes a 64-body x 64-row tile over one chunk in
// steps of 32 coordinates (4 x 4 outputs per thread), and smplx_chain_bwd_kernel adds the chunks in order.
constexpr int kPfSplit = 16;
constexpr int kPfTB = 64, kPfTK = 64, kPfTC = 32;
__global__ void __launch_bounds__(256) smplx_posefeat_bwd_kernel(const float *__restrict__ P, const float *__restrict__ gvp,
                                                                 int V3, int Kp, int B, float *__restrict__ part) {
  __shared__ __align__(16) float Gs[kPfTC][kPfTB + 4];
  __shared__ float Pk[kPfTC][kPfTK + 1];
  const int t = threadIdx.x, tb = t / 16, tk = t % 16;
  const int k0 = blockIdx.x * kPfTK, b0 = blockIdx.y * kPfTB;
  const int chunk = (V3 + kPfSplit - 1) / kPfSplit, c_lo = blockIdx.z * chunk, c_hi = min(V3, c_lo + chunk);
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[i][q] = 0.f;
  for (int cb = c_lo; cb < c_hi; cb += kPfTC) {
    for (int i = t; i < kPfTB * kPfTC; i += 256) {
      const int bb = i / kPfTC, cc = i % kPfTC, c = cb + cc;
      Gs[cc][bb] = (b0 + bb < B && c < c_hi) ? __ldcs(gvp + (size_t)(b0 + bb) * V3 + c) : 0.f;
    }
    for (int i = t; i < kPfTK * kPfTC; i += 256) {
      const int kk = i / kPfTC, cc = i % kPfTC, c = cb + cc;
      Pk[cc][kk] = (k0 + kk < Kp && c < c_hi) ? __ldg(P + (size_t)(k0 + kk) * V3 + c) : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int cc = 0; cc < kPfTC; ++cc) {
      const float4 g = *reinterpret_cast<const float4 *>(&Gs[cc][tb * 4]);
      const float gg[4] = {g.x, g.y, g.z, g.w};
      float p[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) p[q] = Pk[cc][tk + 16 * q];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[i][q] += gg[i] * p[q];
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int b = b0 + tb * 4 + i;
    if (b >= B) break;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int k = k0 + tk + 16 * q;
      if (k < Kp) part[((size_t)b * kPfSplit + blockIdx.z) * Kp + k] = acc[i][q];
    }
  }
}

// Chain backward, per body: recompute G (body_chain), seed its cotangent from A = G - [0 | G.R . J_rest] and the
// posed joints, walk the joints in reverse topological order (one joint per step, so a parent's cotangent is summed
// over its children in a fixed order), add the pose-feature cotangent to R[1:], and finish the coefficient gradient
// with J_dirs^T g_J_rest.
struct ChainBwdArgs {
  SmplxDev m;
  const float *betas, *expr, *rot;
  int n_rot, Kp;
  const float *gA, *gP, *pf_part, *gcoef;   // gP, pf_part, gcoef may be null (zero)
  int n_gcoef;                              // rows of gcoef per body
  float *g_rot, *g_betas, *g_expr;          // any may be null
};

__global__ void __launch_bounds__(128) smplx_chain_bwd_kernel(ChainBwdArgs a) {
  const SmplxDev &m = a.m;
  const int b = blockIdx.x, t = threadIdx.x;
  __shared__ float R[kMaxJoints][9];
  __shared__ float Jr[kMaxJoints][3];
  __shared__ float G[kMaxJoints][12];
  __shared__ float coef[kMaxCoef];
  __shared__ float gG[kMaxJoints][12];
  __shared__ float gR[kMaxJoints][9];
  __shared__ float gJ[kMaxJoints][3];
  const int J = m.J;
  body_chain(m, a.betas, a.expr, a.rot, a.n_rot, b, R, Jr, G, coef);
  const float *gAb = a.gA + (size_t)b * J * 12;
  for (int i = t; i < J * 12; i += blockDim.x) {
    const int j = i / 12, e = i % 12, r = e / 4, c = e % 4;
    float g = gAb[i];
    if (c < 3) g -= gAb[j * 12 + r * 4 + 3] * Jr[j][c];
    else if (a.gP) g += a.gP[((size_t)b * J + j) * 3 + r];
    gG[j][e] = g;
  }
  for (int i = t; i < J * 3; i += blockDim.x) {
    const int j = i / 3, c = i % 3;
    gJ[j][c] = -(G[j][c] * gAb[j * 12 + 3] + G[j][4 + c] * gAb[j * 12 + 7] + G[j][8 + c] * gAb[j * 12 + 11]);
  }
  __syncthreads();
  for (int j = J - 1; j >= 1; --j) {
    const int p = m.parents[j];
    if (t < 12) {
      const int r = t / 4, c = t % 4;
      if (c < 3)
        gG[p][t] += gG[j][r * 4] * R[j][c * 3] + gG[j][r * 4 + 1] * R[j][c * 3 + 1] + gG[j][r * 4 + 2] * R[j][c * 3 + 2] +
                    gG[j][r * 4 + 3] * (Jr[j][c] - Jr[p][c]);
      else
        gG[p][t] += gG[j][t];
    } else if (t < 21) {
      const int k = (t - 12) / 3, c = (t - 12) % 3;
      gR[j][k * 3 + c] = G[p][k] * gG[j][c] + G[p][4 + k] * gG[j][4 + c] + G[p][8 + k] * gG[j][8 + c];
    } else if (t < 24) {
      const int c = t - 21;
      const float rel = G[p][c] * gG[j][3] + G[p][4 + c] * gG[j][7] + G[p][8 + c] * gG[j][11];
      gJ[j][c] += rel;
      gJ[p][c] -= rel;
    }
    __syncthreads();
  }
  if (t < 9) gR[0][t] = gG[0][(t / 3) * 4 + t % 3];
  if (t < 3) gJ[0][t] += gG[0][t * 4 + 3];
  __syncthreads();
  if (a.g_rot) {
    for (int i = t; i < a.n_rot * 9; i += blockDim.x) {
      float g = gR[i / 9][i % 9];
      const int k = i - 9;                   // pose feature (R[1:] - I), k = 9 (j - 1) + e
      if (a.pf_part && k >= 0 && k < a.Kp)
        for (int s = 0; s < kPfSplit; ++s) g += a.pf_part[((size_t)b * kPfSplit + s) * a.Kp + k];
      a.g_rot[(size_t)b * a.n_rot * 9 + i] = g;
    }
  }
  if (t < m.NC && (t < m.NB ? a.g_betas != nullptr : a.g_expr != nullptr)) {
    float g = (a.gcoef && t < a.n_gcoef) ? a.gcoef[(size_t)b * a.n_gcoef + t] : 0.f;
    for (int i = 0; i < J * 3; ++i) g += m.J_dirs[(size_t)i * m.NC + t] * gJ[i / 3][i % 3];
    if (t < m.NB) a.g_betas[(size_t)b * m.NB + t] = g;
    else a.g_expr[(size_t)b * m.NE + (t - m.NB)] = g;
  }
}

// ============================================================================================== keypoint Jacobian
// The keypoints (joints + transl, expression zero) and their Jacobian (3K, P) with respect to the parameters
// [delta_j (3 n_rot) | beta (NB) | t (3)], R_j(delta) = R_j Exp(delta_j), at delta = 0, with the backward's semantics
// (constant LUT row, J14 overwrite, constant model buffers; DESIGN.md §6b).  One CTA per body.  Only the vertices the
// keypoints reference are evaluated: a keypoint entry is one (vertex, weight) pair of a landmark or a J14 row, indexed
// [static landmarks (3 L) | dynamic landmarks of the body's LUT row (3 D) | J14 rows (CSR order)].  Each entry's
// vertex state (v_posed, M = sum_s w_s G_s.R and the posed vertex) is computed once into shared memory when the entries
// fit there, else recomputed where it is used (same function, same bits).  A thread owns one (keypoint, column block)
// and sums that block's entries in entry order: no atomics, and nothing depends on the rest of the batch.
constexpr int kKpJacThreads = 256;
constexpr int kKpState = 15;              // v_posed (3), M (9), posed vertex (3)
constexpr int kKpCacheEntries = 2048;     // entries cached in shared memory (120 KB)

struct KpJacArgs {
  SmplxDev m;
  const float *betas, *rot, *transl;      // transl may be null (zero)
  int n_rot, Kp, P, n_entries, cached;
  float *kp, *jac;
};

__device__ __forceinline__ void kp_entry(const SmplxDev &m, int row, int e, int &v, float &w) {
  if (e < 3 * m.L) { v = m.lmk_vidx[e]; w = m.lmk_bc[e]; return; }
  e -= 3 * m.L;
  if (e < 3 * m.D) {
    const size_t o = (size_t)row * m.D * 3 + e;
    v = m.dyn_vidx[o]; w = m.dyn_bc[o];
    return;
  }
  e -= 3 * m.D;
  v = m.ex_col[e]; w = m.ex_val[e];
}

// entries [e0, e1) of keypoint k; false for a skeleton joint (not overwritten by a J14 row)
__device__ __forceinline__ bool kp_range(const SmplxDev &m, int k, int &e0, int &e1) {
  int r = -1;
  for (int q = 0; q < m.n_over; ++q)
    if (m.over_src[q] == k) r = m.over_tgt[q];
  if (r >= 0) {
    e0 = 3 * (m.L + m.D) + m.ex_ptr[r]; e1 = 3 * (m.L + m.D) + m.ex_ptr[r + 1];
    return true;
  }
  if (k < m.J) return false;
  e0 = 3 * (k - m.J); e1 = e0 + 3;
  return true;
}

__device__ __forceinline__ float kp_jdir(const SmplxDev &m, int j, int c, int l) {
  return m.J_dirs[((size_t)j * 3 + c) * m.NC + l];
}

// v_posed of vertex v (template, the NB shape rows, the fp32 posedirs rows below Kp, in that order), M and the posed
// vertex sum_s w_s (G_s.R (v_posed - J_s) + G_s.t), the skinning weights in ELL order.  EXPR: the NE expression rows
// follow the shape rows (all NC basis rows)
template <bool EXPR = false>
__device__ __forceinline__ void kp_vertex_state(const SmplxDev &m, int v, int Kp, const float *coef, const float *pf,
                                                const float (*G)[12], const float (*Jr)[3], float *st) {
  const int V3 = m.V * 3;
  float p0 = m.v_template[3 * v], p1 = m.v_template[3 * v + 1], p2 = m.v_template[3 * v + 2];
  for (int l = 0; l < (EXPR ? m.NC : m.NB); ++l) {
    const float *S = m.basis + (size_t)l * m.V3p + 3 * v;
    p0 += S[0] * coef[l]; p1 += S[1] * coef[l]; p2 += S[2] * coef[l];
  }
#pragma unroll 8
  for (int k = 0; k < Kp; ++k) {
    const float *P = m.posedirs + (size_t)k * V3 + 3 * v;
    p0 += P[0] * pf[k]; p1 += P[1] * pf[k]; p2 += P[2] * pf[k];
  }
  float M[9], x[3];
  for (int i = 0; i < 9; ++i) M[i] = 0.f;
  x[0] = x[1] = x[2] = 0.f;
  for (int s = 0; s < m.ell_w_n; ++s) {
    const float w = m.ell_w[(size_t)s * m.V + v];
    if (w == 0.f) continue;
    const int j = m.ell_idx[(size_t)s * m.V + v];
    const float q0 = p0 - Jr[j][0], q1 = p1 - Jr[j][1], q2 = p2 - Jr[j][2];
    for (int r = 0; r < 3; ++r) {
      x[r] += w * (G[j][r * 4] * q0 + G[j][r * 4 + 1] * q1 + G[j][r * 4 + 2] * q2 + G[j][r * 4 + 3]);
      for (int c = 0; c < 3; ++c) M[r * 3 + c] += w * G[j][r * 4 + c];
    }
  }
  st[0] = p0; st[1] = p1; st[2] = p2;
  for (int i = 0; i < 9; ++i) st[3 + i] = M[i];
  st[12] = x[0]; st[13] = x[1]; st[14] = x[2];
}

// d x_v / d delta_{j,a} into d[a][c]: the skinning term omega_a x (sum_{s in sub(j)} w_s (G_s.R (v_p - J_s) + G_s.t)
// - W o_j), W = sum_{s in sub(j)} w_s, plus the pose-feature term M . P_v^(j) . vec(R_j [e_a]x) for j >= 1
__device__ __forceinline__ void kp_vertex_drot(const SmplxDev &m, int v, int j, const float *st, const float (*G)[12],
                                               const float (*Jr)[3], const float (*R)[9],
                                               const unsigned long long *sub, float (&d)[3][3]) {
  float Y0 = 0.f, Y1 = 0.f, Y2 = 0.f, W = 0.f;
  for (int s = 0; s < m.ell_w_n; ++s) {
    const float w = m.ell_w[(size_t)s * m.V + v];
    if (w == 0.f) continue;
    const int i = m.ell_idx[(size_t)s * m.V + v];
    if (!((sub[i] >> j) & 1ull)) continue;
    const float q0 = st[0] - Jr[i][0], q1 = st[1] - Jr[i][1], q2 = st[2] - Jr[i][2];
    Y0 += w * (G[i][0] * q0 + G[i][1] * q1 + G[i][2] * q2 + G[i][3]);
    Y1 += w * (G[i][4] * q0 + G[i][5] * q1 + G[i][6] * q2 + G[i][7]);
    Y2 += w * (G[i][8] * q0 + G[i][9] * q1 + G[i][10] * q2 + G[i][11]);
    W += w;
  }
  const float q0 = Y0 - W * G[j][3], q1 = Y1 - W * G[j][7], q2 = Y2 - W * G[j][11];
  for (int a = 0; a < 3; ++a) {
    const float w0 = G[j][a], w1 = G[j][4 + a], w2 = G[j][8 + a];
    d[a][0] = w1 * q2 - w2 * q1; d[a][1] = w2 * q0 - w0 * q2; d[a][2] = w0 * q1 - w1 * q0;
  }
  if (j == 0) return;
  float P[9][3];
  const float *Pj = m.posedirs + (size_t)9 * (j - 1) * m.V * 3 + 3 * v;
  for (int e = 0; e < 9; ++e)
    for (int c = 0; c < 3; ++c) P[e][c] = Pj[(size_t)e * m.V * 3 + c];
  for (int a = 0; a < 3; ++a) {
    // R_j [e_a]x: column c is R_j (e_a x e_c), the column of R_j at (a + 2) % 3 or (a + 1) % 3, signed
    float D[9];
    const int a1 = (a + 1) % 3, a2 = (a + 2) % 3;
    for (int r = 0; r < 3; ++r) {
      D[r * 3 + a] = 0.f;
      D[r * 3 + a1] = R[j][r * 3 + a2];
      D[r * 3 + a2] = -R[j][r * 3 + a1];
    }
    float dv[3];
    for (int c = 0; c < 3; ++c) {
      float s = 0.f;
      for (int e = 0; e < 9; ++e) s += P[e][c] * D[e];
      dv[c] = s;
    }
    for (int r = 0; r < 3; ++r) d[a][r] += st[3 + r * 3] * dv[0] + st[4 + r * 3] * dv[1] + st[5 + r * 3] * dv[2];
  }
}

// d x_v / d beta_l = M S_l[v] + sum_s w_s (dG_s.t/dbeta_l - G_s.R dJ_s/dbeta_l)
__device__ __forceinline__ void kp_vertex_dbeta(const SmplxDev &m, int v, int l, const float *st,
                                                const float (*G)[12], const float (*dGt)[3][kMaxCoef],
                                                float (&d)[3]) {
  const float *S = m.basis + (size_t)l * m.V3p + 3 * v;
  const float s0 = S[0], s1 = S[1], s2 = S[2];
  for (int c = 0; c < 3; ++c) d[c] = st[3 + c * 3] * s0 + st[4 + c * 3] * s1 + st[5 + c * 3] * s2;
  for (int s = 0; s < m.ell_w_n; ++s) {
    const float w = m.ell_w[(size_t)s * m.V + v];
    if (w == 0.f) continue;
    const int i = m.ell_idx[(size_t)s * m.V + v];
    const float j0 = kp_jdir(m, i, 0, l), j1 = kp_jdir(m, i, 1, l), j2 = kp_jdir(m, i, 2, l);
    for (int c = 0; c < 3; ++c)
      d[c] += w * (dGt[i][c][l] - (G[i][c * 4] * j0 + G[i][c * 4 + 1] * j1 + G[i][c * 4 + 2] * j2));
  }
}

// The expression-aware Jacobian's arguments: the expression (B, NE) rides after KpJacArgs, which keeps its layout
struct KpJacExprArgs : KpJacArgs {
  const float *expr;
};

// The body of both Jacobian kernels.  EXPR (smplx_kp_jac_expr_kernel): the chain and the vertex states at the
// expression a.expr, and NE more columns after the betas: the expression rows are shape rows l in [NB, NC) of basis and
// J_dirs, so their columns are the betas columns' formula over all NC coefficients (P = 3 n_rot + NC + 3)
template <bool EXPR, typename Args>
__device__ __forceinline__ void kp_jac_body(const Args &a) {
  const SmplxDev &m = a.m;
  const int b = blockIdx.x, t = threadIdx.x;
  __shared__ float R[kMaxJoints][9];
  __shared__ float Jr[kMaxJoints][3];
  __shared__ float G[kMaxJoints][12];
  __shared__ float coef[kMaxCoef];
  __shared__ float pf[(kMaxJoints - 1) * 9];
  __shared__ float dGt[kMaxJoints][3][kMaxCoef];    // dG_j.t / dbeta
  __shared__ unsigned long long sub[kMaxJoints];    // bit i of sub[s]: i is s or one of its ancestors
  __shared__ int lut_row;
  extern __shared__ float cache[];                  // [n_entries][kKpState] when cached
  const int NB = EXPR ? m.NC : m.NB;                // the shape-like columns: betas, then the expression with EXPR
  const float *expr = nullptr;
  if constexpr (EXPR) expr = a.expr;
  body_chain(m, a.betas, expr, a.rot, a.n_rot, b, R, Jr, G, coef);
  if (t == 0) {
    for (int s = 0; s < m.J; ++s) sub[s] = (s ? sub[m.parents[s]] : 0ull) | (1ull << s);
    lut_row = m.D > 0 ? contour_lut_row(m, R) : 0;
  }
  for (int k = t; k < a.Kp; k += blockDim.x) {
    const int j = 1 + k / 9, e = k % 9;
    pf[k] = R[j][e] - ((e == 0 || e == 4 || e == 8) ? 1.f : 0.f);
  }
  // dG_j.t / dbeta level by level: dG_0.t = dJ_0, dG_j.t = G_p.R (dJ_j - dJ_p) + dG_p.t
  for (int i = t; i < 3 * NB; i += blockDim.x) dGt[0][i / NB][i % NB] = kp_jdir(m, 0, i / NB, i % NB);
  __syncthreads();
  for (int lv = 1; lv < m.n_levels; ++lv) {
    const int off = m.level_off[lv], cnt = m.level_off[lv + 1] - off;
    for (int i = t; i < cnt * 3 * NB; i += blockDim.x) {
      const int j = m.level_joints[off + i / (3 * NB)], c = (i / NB) % 3, l = i % NB, p = m.parents[j];
      const float r0 = kp_jdir(m, j, 0, l) - kp_jdir(m, p, 0, l), r1 = kp_jdir(m, j, 1, l) - kp_jdir(m, p, 1, l),
                  r2 = kp_jdir(m, j, 2, l) - kp_jdir(m, p, 2, l);
      dGt[j][c][l] = G[p][c * 4] * r0 + G[p][c * 4 + 1] * r1 + G[p][c * 4 + 2] * r2 + dGt[p][c][l];
    }
    __syncthreads();
  }
  const int row = lut_row;
  if (a.cached) {
    for (int e = t; e < a.n_entries; e += blockDim.x) {
      int v;
      float w;
      kp_entry(m, row, e, v, w);
      kp_vertex_state<EXPR>(m, v, a.Kp, coef, pf, G, Jr, cache + (size_t)e * kKpState);
    }
    __syncthreads();
  }
  // work items (keypoint k, column block g): g < n_rot the 3 x 3 block of delta_g, g = n_rot the betas, g = n_rot + 1
  // the translation and the keypoint itself
  const int NG = a.n_rot + 2, P = a.P, K = m.K;
  const float *tr = a.transl ? a.transl + (size_t)b * 3 : nullptr;
  float *jb = a.jac + (size_t)b * 3 * K * P;
  float local[kKpState];
  for (int i = t; i < K * NG; i += blockDim.x) {
    const int k = i / NG, g = i % NG;
    int e0 = 0, e1 = 0;
    const bool mix = kp_range(m, k, e0, e1);
    float *o = jb + (size_t)3 * k * P;          // row 3 k + c at o + c P
    auto state = [&](int e, int &v, float &w) -> const float * {
      kp_entry(m, row, e, v, w);
      if (a.cached) return cache + (size_t)e * kKpState;
      kp_vertex_state<EXPR>(m, v, a.Kp, coef, pf, G, Jr, local);
      return local;
    };
    if (g < a.n_rot) {
      float acc[3][3];                           // [a][c]
      for (int x = 0; x < 3; ++x) acc[x][0] = acc[x][1] = acc[x][2] = 0.f;
      if (!mix) {
        if (g != k && ((sub[k] >> g) & 1ull)) {  // omega_a x (J_k - o_g) for a proper ancestor g
          const float q0 = G[k][3] - G[g][3], q1 = G[k][7] - G[g][7], q2 = G[k][11] - G[g][11];
          for (int x = 0; x < 3; ++x) {
            const float w0 = G[g][x], w1 = G[g][4 + x], w2 = G[g][8 + x];
            acc[x][0] = w1 * q2 - w2 * q1; acc[x][1] = w2 * q0 - w0 * q2; acc[x][2] = w0 * q1 - w1 * q0;
          }
        }
      } else {
        for (int e = e0; e < e1; ++e) {
          int v;
          float w;
          const float *st = state(e, v, w);
          float d[3][3];
          kp_vertex_drot(m, v, g, st, G, Jr, R, sub, d);
          for (int x = 0; x < 3; ++x)
            for (int c = 0; c < 3; ++c) acc[x][c] += w * d[x][c];
        }
      }
      for (int c = 0; c < 3; ++c)
        for (int x = 0; x < 3; ++x) o[(size_t)c * P + 3 * g + x] = acc[x][c];
    } else if (g == a.n_rot) {
      for (int l = 0; l < NB; ++l) {
        float acc[3] = {0.f, 0.f, 0.f};
        if (!mix) {
          for (int c = 0; c < 3; ++c) acc[c] = dGt[k][c][l];
        } else {
          for (int e = e0; e < e1; ++e) {
            int v;
            float w;
            const float *st = state(e, v, w);
            float d[3];
            kp_vertex_dbeta(m, v, l, st, G, dGt, d);
            for (int c = 0; c < 3; ++c) acc[c] += w * d[c];
          }
        }
        for (int c = 0; c < 3; ++c) o[(size_t)c * P + 3 * a.n_rot + l] = acc[c];
      }
    } else {
      float x[3];
      if (!mix) {
        for (int c = 0; c < 3; ++c) x[c] = G[k][c * 4 + 3];
      } else {
        x[0] = x[1] = x[2] = 0.f;
        for (int e = e0; e < e1; ++e) {
          int v;
          float w;
          const float *st = state(e, v, w);
          for (int c = 0; c < 3; ++c) x[c] += w * st[12 + c];
        }
      }
      for (int c = 0; c < 3; ++c) {
        a.kp[((size_t)b * K + k) * 3 + c] = tr ? x[c] + tr[c] : x[c];
        for (int x2 = 0; x2 < 3; ++x2) o[(size_t)c * P + 3 * a.n_rot + NB + x2] = c == x2 ? 1.f : 0.f;
      }
    }
  }
}

__global__ void __launch_bounds__(kKpJacThreads) smplx_kp_jac_kernel(KpJacArgs a) { kp_jac_body<false>(a); }

__global__ void __launch_bounds__(kKpJacThreads) smplx_kp_jac_expr_kernel(KpJacExprArgs a) { kp_jac_body<true>(a); }

// ============================================================================================== vertex Jacobian
// Every posed vertex (+ transl) and its Jacobian (3, P) with the columns of the keypoint Jacobian, for the dense fits
// (the LM scan fit): one CTA per (tile of kVjTile vertices, body), grid (ceil(V / kVjTile), B).  Each CTA recomputes
// its body's chain (jac_chain, a few microseconds of the CTA's time), then the tile's vertex states (kp_vertex_state),
// then one work item per (vertex, column block) as in the keypoint Jacobian, into a shared-memory tile [vertex][xyz][P]
// that is written out contiguously.  Same device functions, so a barycentric mix of these rows is the keypoint
// Jacobian's landmark row up to fp32 rounding.  No atomics; a body's bits do not depend on the rest of the batch.
constexpr int kVjTile = 32;

// The per-body chain the vertex Jacobian starts from, in shared memory: kp_jac_body's prologue without the contour LUT
// row (written apart so that the keypoint kernels keep their code): body_chain, the ancestor masks sub (bit i of
// sub[s]: i is s or one of its ancestors), the pose feature pf (Kp entries) and dG_j.t / dbeta of the betas columns
// level by level.  Ends on a barrier
__device__ __forceinline__ void jac_chain(const SmplxDev &m, const float *betas, const float *rot, int n_rot,
                                          int Kp, int NB, int b, float (*R)[9], float (*Jr)[3],
                                          float (*G)[12], float *coef, float *pf, float (*dGt)[3][kMaxCoef],
                                          unsigned long long *sub) {
  const int t = threadIdx.x;
  body_chain(m, betas, nullptr, rot, n_rot, b, R, Jr, G, coef);
  if (t == 0)
    for (int s = 0; s < m.J; ++s) sub[s] = (s ? sub[m.parents[s]] : 0ull) | (1ull << s);
  for (int k = t; k < Kp; k += blockDim.x) {
    const int j = 1 + k / 9, e = k % 9;
    pf[k] = R[j][e] - ((e == 0 || e == 4 || e == 8) ? 1.f : 0.f);
  }
  // dG_j.t / dbeta level by level: dG_0.t = dJ_0, dG_j.t = G_p.R (dJ_j - dJ_p) + dG_p.t
  for (int i = t; i < 3 * NB; i += blockDim.x) dGt[0][i / NB][i % NB] = kp_jdir(m, 0, i / NB, i % NB);
  __syncthreads();
  for (int lv = 1; lv < m.n_levels; ++lv) {
    const int off = m.level_off[lv], cnt = m.level_off[lv + 1] - off;
    for (int i = t; i < cnt * 3 * NB; i += blockDim.x) {
      const int j = m.level_joints[off + i / (3 * NB)], c = (i / NB) % 3, l = i % NB, p = m.parents[j];
      const float r0 = kp_jdir(m, j, 0, l) - kp_jdir(m, p, 0, l), r1 = kp_jdir(m, j, 1, l) - kp_jdir(m, p, 1, l),
                  r2 = kp_jdir(m, j, 2, l) - kp_jdir(m, p, 2, l);
      dGt[j][c][l] = G[p][c * 4] * r0 + G[p][c * 4 + 1] * r1 + G[p][c * 4 + 2] * r2 + dGt[p][c][l];
    }
    __syncthreads();
  }
}

struct VertJacArgs {
  SmplxDev m;
  const float *betas, *rot, *transl;      // transl may be null (zero)
  int n_rot, Kp, P;
  float *verts, *jac;
};

__global__ void __launch_bounds__(kKpJacThreads) smplx_vertex_jac_kernel(VertJacArgs a) {
  const SmplxDev &m = a.m;
  const int b = blockIdx.y, v0 = blockIdx.x * kVjTile, t = threadIdx.x;
  __shared__ float R[kMaxJoints][9];
  __shared__ float Jr[kMaxJoints][3];
  __shared__ float G[kMaxJoints][12];
  __shared__ float coef[kMaxCoef];
  __shared__ float pf[(kMaxJoints - 1) * 9];
  __shared__ float dGt[kMaxJoints][3][kMaxCoef];
  __shared__ unsigned long long sub[kMaxJoints];
  __shared__ float st[kVjTile][kKpState];
  extern __shared__ float tile[];                   // [nv][3][P]
  jac_chain(m, a.betas, a.rot, a.n_rot, a.Kp, m.NB, b, R, Jr, G, coef, pf, dGt, sub);
  const int nv = min(kVjTile, m.V - v0), P = a.P, NB = m.NB, NG = a.n_rot + 2;
  for (int i = t; i < nv; i += blockDim.x) kp_vertex_state(m, v0 + i, a.Kp, coef, pf, G, Jr, st[i]);
  __syncthreads();
  // work items (vertex q, column block g): g < n_rot the 3 x 3 block of delta_g, g = n_rot the betas, then transl
  for (int i = t; i < nv * NG; i += blockDim.x) {
    const int q = i / NG, g = i % NG, v = v0 + q;
    float *o = tile + (size_t)q * 3 * P;          // row c at o + c P
    if (g < a.n_rot) {
      float d[3][3];
      kp_vertex_drot(m, v, g, st[q], G, Jr, R, sub, d);
      for (int c = 0; c < 3; ++c)
        for (int x = 0; x < 3; ++x) o[c * P + 3 * g + x] = d[x][c];
    } else if (g == a.n_rot) {
      for (int l = 0; l < NB; ++l) {
        float d[3];
        kp_vertex_dbeta(m, v, l, st[q], G, dGt, d);
        for (int c = 0; c < 3; ++c) o[c * P + 3 * a.n_rot + l] = d[c];
      }
    } else {
      for (int c = 0; c < 3; ++c)
        for (int x = 0; x < 3; ++x) o[c * P + 3 * a.n_rot + NB + x] = c == x ? 1.f : 0.f;
    }
  }
  __syncthreads();
  const float *tr = a.transl ? a.transl + (size_t)b * 3 : nullptr;
  const size_t base = (size_t)b * m.V + v0;
  for (int i = t; i < nv * 3; i += blockDim.x) {
    const float x = st[i / 3][12 + i % 3];
    a.verts[base * 3 + i] = tr ? x + tr[i % 3] : x;
  }
  float *jb = a.jac + base * 3 * P;
  for (int i = t; i < nv * 3 * P; i += blockDim.x) jb[i] = tile[i];
}

}  // namespace shapy

using namespace shapy;

extern "C" int shapy_smplx_create(shapy_smplx_t **out, const shapy_smplx_desc_t *d) {
  SHAPY_REQUIRE(out && d, "shapy_smplx_create: null argument");
  SHAPY_REQUIRE(d->num_joints >= 1 && d->num_joints <= kMaxJoints, "num_joints %d unsupported", d->num_joints);
  SHAPY_REQUIRE(d->num_betas >= 1 && d->num_betas + d->num_expr <= kMaxCoef, "too many shape coefficients");
  SHAPY_REQUIRE(d->v_template && d->shapedirs && d->posedirs && d->J_regressor && d->lbs_weights && d->parents &&
                    d->faces, "shapy_smplx_create: missing model tensor");
  const int V = d->num_verts, J = d->num_joints, NB = d->num_betas, NE = d->expr_dirs ? d->num_expr : 0;
  const int NC = NB + NE, F = d->num_faces;
  auto *m = new shapy_smplx();
  SmplxDev &s = m->d;
  memset(&s, 0, sizeof(s));
  s.V = V; s.J = J; s.NB = NB; s.NE = NE; s.NC = NC; s.F = F;
  cudaError_t err = cudaSuccess;
  s.v_template = upload(m->allocs, std::vector<float>(d->v_template, d->v_template + (size_t)V * 3), err);
  // shapedirs -> [NC][3V]
  std::vector<float> S((size_t)NC * V * 3);
  for (int c = 0; c < V * 3; ++c) {
    for (int l = 0; l < NB; ++l) S[(size_t)l * V * 3 + c] = d->shapedirs[(size_t)c * NB + l];
    for (int l = 0; l < NE; ++l) S[(size_t)(NB + l) * V * 3 + c] = d->expr_dirs[(size_t)c * NE + l];
  }
  s.posedirs = upload(m->allocs, std::vector<float>(d->posedirs, d->posedirs + (size_t)(J - 1) * 9 * V * 3), err);
  {
    // shape and expression blend-shape basis with rows padded to a multiple of 4 floats (16-byte cp.async)
    const int V3 = V * 3, V3p = (V3 + 3) / 4 * 4;
    std::vector<float> basis((size_t)NC * V3p, 0.f);
    for (int l = 0; l < NC; ++l) memcpy(&basis[(size_t)l * V3p], &S[(size_t)l * V3], (size_t)V3 * sizeof(float));
    s.V3p = V3p;
    s.basis = upload(m->allocs, basis, err);
    m->zero_bias = upload(m->allocs, std::vector<float>((size_t)(V3 + kPoseV3Align - 1) / kPoseV3Align * kPoseV3Align, 0.f), err);
  }
  // joint regression contracted with the template and the shape basis (fp64 accumulate)
  std::vector<float> Jt((size_t)J * 3), Jd((size_t)J * 3 * NC);
  for (int j = 0; j < J; ++j) {
    std::vector<double> at(3, 0.0), ad((size_t)3 * NC, 0.0);
    for (int v = 0; v < V; ++v) {
      double w = d->J_regressor[(size_t)j * V + v];
      if (w == 0.0) continue;
      for (int c = 0; c < 3; ++c) {
        at[c] += w * d->v_template[(size_t)v * 3 + c];
        for (int l = 0; l < NC; ++l) ad[(size_t)c * NC + l] += w * S[(size_t)l * V * 3 + v * 3 + c];
      }
    }
    for (int c = 0; c < 3; ++c) {
      Jt[j * 3 + c] = (float)at[c];
      for (int l = 0; l < NC; ++l) Jd[((size_t)j * 3 + c) * NC + l] = (float)ad[(size_t)c * NC + l];
    }
  }
  s.J_template = upload(m->allocs, Jt, err);
  s.J_dirs = upload(m->allocs, Jd, err);
  // ELL skinning weights
  int W = 1;
  for (int v = 0; v < V; ++v) {
    int n = 0;
    for (int j = 0; j < J; ++j) n += d->lbs_weights[(size_t)v * J + j] != 0.f;
    W = std::max(W, n);
  }
  std::vector<int> eidx((size_t)W * V, 0);
  std::vector<float> ew((size_t)W * V, 0.f);
  for (int v = 0; v < V; ++v) {
    int n = 0;
    for (int j = 0; j < J; ++j) {
      float w = d->lbs_weights[(size_t)v * J + j];
      if (w != 0.f) { eidx[(size_t)n * V + v] = j; ew[(size_t)n * V + v] = w; ++n; }
    }
  }
  s.ell_w_n = W;
  s.ell_idx = upload(m->allocs, eidx, err);
  s.ell_w = upload(m->allocs, ew, err);
  // kinematic levels
  std::vector<int> par(J), depth(J, 0);
  for (int j = 0; j < J; ++j) par[j] = j == 0 ? -1 : (int)d->parents[j];
  int maxd = 0;
  for (int j = 1; j < J; ++j) {
    if (par[j] < 0 || par[j] >= j) { delete m; set_error("parents[%d] = %d is not a topologically ordered tree", j, par[j]); return SHAPY_ERR_ARG; }
    depth[j] = depth[par[j]] + 1;
    maxd = std::max(maxd, depth[j]);
  }
  std::vector<int> lj, lo;
  for (int lv = 0; lv <= maxd; ++lv) {
    lo.push_back((int)lj.size());
    for (int j = 0; j < J; ++j) if (depth[j] == lv) lj.push_back(j);
  }
  lo.push_back((int)lj.size());
  s.n_levels = maxd + 1;
  s.parents = upload(m->allocs, par, err);
  s.level_joints = upload(m->allocs, lj, err);
  s.level_off = upload(m->allocs, lo, err);
  std::vector<int> faces((size_t)F * 3);
  for (size_t i = 0; i < faces.size(); ++i) faces[i] = (int)d->faces[i];
  s.faces = upload(m->allocs, faces, err);
  // landmarks resolved to vertex triples
  s.L = d->lmk_faces_idx ? d->num_static_lmk : 0;
  std::vector<int> lv((size_t)s.L * 3);
  for (int i = 0; i < s.L; ++i)
    for (int c = 0; c < 3; ++c) lv[i * 3 + c] = faces[(size_t)d->lmk_faces_idx[i] * 3 + c];
  s.lmk_vidx = upload(m->allocs, lv, err);
  s.lmk_bc = upload(m->allocs, std::vector<float>(d->lmk_bary_coords, d->lmk_bary_coords + (size_t)s.L * 3), err);
  s.D = d->dynamic_lmk_faces_idx ? d->num_dyn_lmk : 0;
  s.rows = s.D ? d->num_dyn_rows : 0;
  std::vector<int> dv((size_t)s.rows * s.D * 3);
  for (size_t i = 0; i < (size_t)s.rows * s.D; ++i)
    for (int c = 0; c < 3; ++c) dv[i * 3 + c] = faces[(size_t)d->dynamic_lmk_faces_idx[i] * 3 + c];
  s.dyn_vidx = upload(m->allocs, dv, err);
  s.dyn_bc = upload(m->allocs, std::vector<float>(d->dynamic_lmk_bary_coords,
                                          d->dynamic_lmk_bary_coords + (s.D ? (size_t)s.rows * s.D * 3 : 0)), err);
  s.n_chain = s.D ? d->neck_chain_len : 0;
  std::vector<int> neck(s.n_chain);
  for (int i = 0; i < s.n_chain; ++i) neck[i] = (int)d->neck_kin_chain[i];
  s.neck = upload(m->allocs, neck, err);
  s.K = J + s.L + s.D;
  // J14 regressor -> CSR
  s.n_extra = d->extra_joint_regressor ? d->num_extra : 0;
  std::vector<int> ep(1, 0), ec;
  std::vector<float> ev;
  for (int r = 0; r < s.n_extra; ++r) {
    for (int v = 0; v < V; ++v) {
      float w = d->extra_joint_regressor[(size_t)r * V + v];
      if (w != 0.f) { ec.push_back(v); ev.push_back(w); }
    }
    ep.push_back((int)ec.size());
  }
  s.ex_ptr = upload(m->allocs, ep, err);
  s.ex_col = upload(m->allocs, ec, err);
  s.ex_val = upload(m->allocs, ev, err);
  m->extra_nnz = (int)ec.size();
  s.n_over = s.n_extra ? d->num_overwrite : 0;
  std::vector<int> os(s.n_over), ot(s.n_over);
  for (int i = 0; i < s.n_over; ++i) { os[i] = (int)d->source_idxs[i]; ot[i] = (int)d->target_idxs[i]; }
  s.over_src = upload(m->allocs, os, err);
  s.over_tgt = upload(m->allocs, ot, err);
  {
    // backward tables: the vertices of every joint's skinning weights, ascending
    std::vector<int> jp(1, 0), jvi;
    std::vector<float> jvw;
    for (int j = 0; j < J; ++j) {
      for (int v = 0; v < V; ++v) {
        const float w = d->lbs_weights[(size_t)v * J + j];
        if (w != 0.f) { jvi.push_back(v); jvw.push_back(w); }
      }
      jp.push_back((int)jvi.size());
    }
    s.jv_ptr = upload(m->allocs, jp, err);
    s.jv_idx = upload(m->allocs, jvi, err);
    s.jv_w = upload(m->allocs, jvw, err);
    // ... and the keypoint entries of every vertex: static landmarks, dynamic landmarks (per LUT row), J14 rows
    std::vector<std::vector<int>> slot(V), row(V);
    std::vector<std::vector<float>> wt(V);
    auto add = [&](int v, int sl, int r, float w) { slot[v].push_back(sl); row[v].push_back(r); wt[v].push_back(w); };
    for (int i = 0; i < s.L; ++i)
      for (int c = 0; c < 3; ++c) add(lv[i * 3 + c], i, -1, d->lmk_bary_coords[i * 3 + c]);
    for (int r = 0; r < s.rows; ++r)
      for (int i = 0; i < s.D; ++i)
        for (int c = 0; c < 3; ++c) {
          const size_t o = ((size_t)r * s.D + i) * 3 + c;
          add(dv[o], s.L + i, r, d->dynamic_lmk_bary_coords[o]);
        }
    for (int r = 0; r < s.n_extra; ++r)
      for (int e = ep[r]; e < ep[r + 1]; ++e) add(ec[e], s.L + s.D + r, -1, ev[e]);
    std::vector<int> vp(1, 0), vs, vr;
    std::vector<float> vw;
    for (int v = 0; v < V; ++v) {
      vs.insert(vs.end(), slot[v].begin(), slot[v].end());
      vr.insert(vr.end(), row[v].begin(), row[v].end());
      vw.insert(vw.end(), wt[v].begin(), wt[v].end());
      vp.push_back((int)vs.size());
    }
    s.vk_ptr = upload(m->allocs, vp, err);
    s.vk_slot = upload(m->allocs, vs, err);
    s.vk_row = upload(m->allocs, vr, err);
    s.vk_w = upload(m->allocs, vw, err);
  }
  if (err != cudaSuccess) {
    set_error("shapy_smplx_create: %s", cudaGetErrorString(err));
    shapy_smplx_destroy(m);
    return (int)err;
  }
  *out = m;
  return SHAPY_OK;
}

extern "C" void shapy_smplx_destroy(shapy_smplx_t *m) {
  if (!m) return;
  for (void *p : m->allocs) cudaFree(p);
  for (auto &kv : m->pw) { cudaFree(kv.second.hi); cudaFree(kv.second.lo); }
  delete m;
}

extern "C" int shapy_smplx_num_keypoints(const shapy_smplx_t *m) { return m ? m->d.K : 0; }
extern "C" const int32_t *shapy_smplx_faces_i32(const shapy_smplx_t *m) { return m ? m->d.faces : nullptr; }

static inline int bpad(int B) { return (B + 31) / 32 * 32; }

static inline int pose_kpad(int Kp) { return (Kp + kPoseKAlign - 1) / kPoseKAlign * kPoseKAlign; }
static inline int pose_v3g(const SmplxDev &d) { return (d.V * 3 + kPoseV3Align - 1) / kPoseV3Align * kPoseV3Align; }

// Workspace of shapy_smplx_forward, 256-byte aligned pieces.  The GEMM activations are sized for the widest pose
// feature ((J - 1) * 9); a call uses the first B * Kpad of them.
struct SmplxWorkspace {
  float *A;              // [B][J][12] relative transforms
  float *pfT;            // [NC][Bpad] blend coefficients, transposed
  int *lut;              // [B] dynamic-contour LUT rows
  float *joints;         // [B][K][3] joints when the caller asks for none
  __half *x_hi, *x_lo;   // pose-blend GEMM activations [B][Kpad], split fp16
  __half *y_hi, *y_lo;   // pose-blend GEMM result [B][V3g], split fp16
  size_t bytes;
};

// base == nullptr: only `bytes` is meaningful
static SmplxWorkspace smplx_workspace(const SmplxDev &d, int B, void *base) {
  SmplxWorkspace w;
  w.bytes = 0;
  auto take = [&](size_t n) { void *p = base ? (char *)base + w.bytes : nullptr; w.bytes += align_up(n, 256); return p; };
  const size_t x = (size_t)B * pose_kpad((d.J - 1) * 9) * sizeof(__half), y = (size_t)B * pose_v3g(d) * sizeof(__half);
  w.A = (float *)take((size_t)B * d.J * 12 * sizeof(float));
  w.pfT = (float *)take((size_t)d.NC * bpad(B) * sizeof(float));
  w.lut = (int *)take((size_t)B * sizeof(int));
  w.joints = (float *)take((size_t)B * d.K * 3 * sizeof(float));
  w.x_hi = (__half *)take(x); w.x_lo = (__half *)take(x);
  w.y_hi = (__half *)take(y); w.y_lo = (__half *)take(y);
  return w;
}

// Pose blend (R[1:] - I) . P of all B bodies as one split-fp16 tensor-core GEMM on the wgmma engine, expressed as a
// 1x1 convolution: "pixels" = bodies, cin = pose features, cout = the 3V vertex coordinates.  Its input is what
// smplx_pose_kernel wrote to ws.x_*.  Fills va.pb_*.
static int pose_blend_gemm(const shapy_smplx *m, int B, int Kp, const SmplxWorkspace &ws, cudaStream_t st,
                           VertexArgs &va) {
  const SmplxDev &d = m->d;
  const int Kpad = pose_kpad(Kp), V3g = pose_v3g(d);
  shapy_smplx::PoseW pw;
  {
    std::lock_guard<std::mutex> lk(m->pw_mu);
    auto it = m->pw.find(Kpad);
    if (it == m->pw.end()) {
      const size_t n = (size_t)V3g * Kpad;
      SHAPY_CUDA_TRY(cudaMalloc((void **)&pw.hi, n * sizeof(__half)));
      SHAPY_CUDA_TRY(cudaMalloc((void **)&pw.lo, n * sizeof(__half)));
      pack_pose_weights_kernel<<<1024, 256, 0, st>>>(d.posedirs, d.V * 3, (d.J - 1) * 9, Kpad, V3g, pw.hi, pw.lo);
      SHAPY_LAUNCH_CHECK();
      m->pw[Kpad] = pw;
    } else {
      pw = it->second;
    }
  }
  ConvW w;
  w.w_hi = pw.hi; w.w_lo = pw.lo; w.bias = m->zero_bias;
  w.cin = Kpad; w.cout = V3g; w.ksize = 1; w.stride = 1;
  ActView in, out;
  in.hi = ws.x_hi; in.lo = ws.x_lo; in.N = B; in.H = 1; in.W = 1; in.C = Kpad; in.Ctot = Kpad; in.coff = 0;
  out.hi = ws.y_hi; out.lo = ws.y_lo; out.N = B; out.H = 1; out.W = 1; out.C = V3g; out.Ctot = V3g; out.coff = 0;
  WgmmaPlan *plan = wgmma_plan_create(w, in, out, nullptr, false);
  if (!plan) return SHAPY_ERR_UNSUPPORTED;
  const int rc = wgmma_plan_launch(plan, st, false);
  wgmma_plan_destroy(plan);
  if (rc != SHAPY_OK) return rc;
  va.pb_hi = ws.y_hi; va.pb_lo = ws.y_lo; va.pb_ld = V3g;
  return SHAPY_OK;
}

extern "C" size_t shapy_smplx_workspace_bytes(const shapy_smplx_t *m, int B) {
  if (!m || B <= 0) return 0;
  return smplx_workspace(m->d, B, nullptr).bytes;
}

extern "C" int shapy_decode_rot6d(const float *raw, int n, float *rot, void *stream) {
  SHAPY_REQUIRE(raw && rot && n >= 0, "shapy_decode_rot6d: bad argument");
  if (n == 0) return SHAPY_OK;
  decode_rot6d_kernel<<<ceil_div(n, 128), 128, 0, (cudaStream_t)stream>>>(raw, n, rot);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

// smplx_joints_kernel as a programmatic dependent of the vertex kernel before it
static int launch_joints(const SmplxDev &d, const float *vertices, const float *camera, const int *lut, int B,
                         float *joints, float *proj_joints, cudaStream_t st) {
  JointsArgs ja{d, vertices, camera, lut, B, joints, proj_joints};
  size_t smem = ((size_t)d.K * 3 + (size_t)std::max(d.n_extra, 1) * 3) * sizeof(float);
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(B);
  cfg.blockDim = dim3(512);     // 16 warps: the 14 sparse J14 rows and the 68 landmarks are each one pass of dependent loads
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  SHAPY_CUDA_TRY(cudaLaunchKernelEx(&cfg, smplx_joints_kernel, ja));
  count_launch();
  return SHAPY_OK;
}

extern "C" int shapy_smplx_forward(const shapy_smplx_t *m, const float *betas, const float *rot, int n_rot,
                                   const float *expr, const float *camera, int B, float *vertices, float *v_shaped,
                                   float *joints, float *proj_joints, void *workspace, size_t workspace_bytes,
                                   void *stream) {
  SHAPY_REQUIRE(m && betas && rot, "shapy_smplx_forward: null argument");
  SHAPY_REQUIRE(B > 0, "shapy_smplx_forward: batch %d", B);
  SHAPY_REQUIRE(n_rot >= 1 && n_rot <= m->d.J, "shapy_smplx_forward: n_rot %d out of range", n_rot);
  SHAPY_REQUIRE(workspace && workspace_bytes >= shapy_smplx_workspace_bytes(m, B), "shapy_smplx_forward: workspace too small");
  SHAPY_REQUIRE(!(proj_joints && !joints) , "proj_joints requires joints");
  SHAPY_REQUIRE(!(joints && !vertices && (m->d.L + m->d.D + m->d.n_extra) > 0), "joints require vertices");
  cudaStream_t st = (cudaStream_t)stream;
  const SmplxDev &d = m->d;
  const SmplxWorkspace ws = smplx_workspace(d, B, workspace);
  const int Kp = (n_rot - 1) * 9;
  const bool gemm = vertices && Kp > 0;
  {
    PoseArgs pa{d, betas, d.NE ? expr : nullptr, rot, n_rot, B, bpad(B), Kp, pose_kpad(Kp), ws.A, ws.pfT,
                joints ? joints : ws.joints, ws.lut, gemm ? ws.x_hi : nullptr, gemm ? ws.x_lo : nullptr};
    smplx_pose_kernel<<<B, 128, 0, st>>>(pa);
    SHAPY_LAUNCH_CHECK();
    if (vertices || v_shaped) {
      VertexArgs va{d, betas, d.NE ? expr : nullptr, ws.A, ws.pfT, B, bpad(B), vertices, v_shaped, nullptr, nullptr, 0};
      if (gemm) {
        const int rc = pose_blend_gemm(m, B, Kp, ws, st, va);
        if (rc != SHAPY_OK) return rc;
      }
      dim3 grid(ceil_div(d.V, TV), ceil_div(B, TB));
      smplx_vertex_kernel<<<grid, 128, 0, st>>>(va);
      SHAPY_LAUNCH_CHECK();
    }
  }
  if (joints && (d.L + d.D + d.n_extra > 0 || proj_joints))
    return launch_joints(d, vertices, camera, ws.lut, B, joints, proj_joints, st);
  return SHAPY_OK;
}

extern "C" int shapy_smplx_forward_shape(const shapy_smplx_t *m, const float *betas, int B, float *v_shaped,
                                         void *stream) {
  SHAPY_REQUIRE(m && betas && v_shaped && B > 0, "shapy_smplx_forward_shape: bad argument");
  const SmplxDev &d = m->d;
  cudaStream_t st = (cudaStream_t)stream;
  const int V3 = d.V * 3;
  if (d.NB == 10) {
    dim3 grid(ceil_div(V3, 512), ceil_div(B, SB));
    smplx_shape_kernel<10><<<grid, 256, 0, st>>>(d.v_template, d.basis, d.V3p, betas, V3, B, v_shaped);
  } else {
    dim3 grid(ceil_div(V3, 256), B);
    smplx_shape_kernel_generic<<<grid, 256, 0, st>>>(d.v_template, d.basis, d.V3p, betas, d.NB, V3, B, v_shaped);
  }
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

extern "C" size_t shapy_smplx_backward_shape_workspace_bytes(const shapy_smplx_t *m, int batch) {
  return m && batch > 0 ? (size_t)batch * kShapeSplit * m->d.NB * sizeof(float) : 0;
}

extern "C" int shapy_smplx_backward_shape(const shapy_smplx_t *m, const float *grad_v_shaped, int B, float *grad_betas,
                                          void *workspace, size_t workspace_bytes, void *stream) {
  SHAPY_REQUIRE(m && grad_v_shaped && grad_betas && B > 0, "shapy_smplx_backward_shape: bad argument");
  SHAPY_REQUIRE(workspace && workspace_bytes >= shapy_smplx_backward_shape_workspace_bytes(m, B),
                "shapy_smplx_backward_shape: workspace too small");
  const SmplxDev &d = m->d;
  cudaStream_t st = (cudaStream_t)stream;
  const int V3 = d.V * 3;
  float *part = static_cast<float *>(workspace);
  if (d.NB == 10) {
    smplx_shape_bwd_kernel<10, 0, kShapeTile><<<dim3(ceil_div(B, kShapeTile), kShapeSplit), 256, 0, st>>>(
        d.basis, d.V3p, grad_v_shaped, nullptr, V3, B, part);
  } else {
    smplx_shape_bwd_kernel_generic<<<dim3(B, kShapeSplit, d.NB), 256, 0, st>>>(d.basis, d.V3p, grad_v_shaped, nullptr,
                                                                               d.NB, d.NB, V3, part);
  }
  SHAPY_LAUNCH_CHECK();
  smplx_shape_bwd_sum_kernel<<<ceil_div(B * d.NB, 256), 256, 0, st>>>(part, d.NB, B, grad_betas);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

extern "C" int shapy_decode_rot6d_backward(const float *raw, int n, const float *grad_rot, float *grad_raw,
                                           void *stream) {
  SHAPY_REQUIRE(raw && grad_rot && grad_raw && n >= 0, "shapy_decode_rot6d_backward: bad argument");
  if (n == 0) return SHAPY_OK;
  decode_rot6d_bwd_kernel<<<ceil_div(n, 128), 128, 0, (cudaStream_t)stream>>>(raw, n, grad_rot, grad_raw);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

// Workspace of shapy_smplx_backward: the forward's, then the backward's buffers, 256-byte aligned pieces.
struct SmplxBwdWorkspace {
  SmplxWorkspace f;
  float *vp, *gv, *gvp;      // [B][V][3] v_posed, vertex cotangent (first the recomputed vertices), its pull-back
  float *gP, *gkp, *gA;      // [B][J][3] posed-joint, [B][nkp][3] landmark / J14, [B][J][12] transform cotangents
  float *pf_part;            // [B][kPfSplit][Kp] pose-feature adjoint partial sums
  float *shape_part, *gcoef; // [B][kShapeSplit][NC] shape adjoint partial sums, [B][NC] their sums
  size_t bytes;
};

static SmplxBwdWorkspace smplx_bwd_workspace(const SmplxDev &d, int B, int n_rot, void *base) {
  SmplxBwdWorkspace w;
  w.f = smplx_workspace(d, B, base);
  w.bytes = w.f.bytes;
  auto take = [&](size_t n) {
    float *p = base ? (float *)((char *)base + w.bytes) : nullptr;
    w.bytes += align_up(std::max<size_t>(n, 1) * sizeof(float), 256);
    return p;
  };
  const size_t Bs = (size_t)B, V3 = (size_t)d.V * 3;
  const int nkp = d.L + d.D + d.n_extra, Kp = (n_rot - 1) * 9;
  w.vp = take(Bs * V3); w.gv = take(Bs * V3); w.gvp = take(Bs * V3);
  w.gP = take(Bs * d.J * 3); w.gkp = take(Bs * nkp * 3); w.gA = take(Bs * d.J * 12);
  w.pf_part = take(Bs * kPfSplit * Kp);
  w.shape_part = take(Bs * kShapeSplit * d.NC); w.gcoef = take(Bs * d.NC);
  return w;
}

extern "C" size_t shapy_smplx_backward_workspace_bytes(const shapy_smplx_t *m, int B, int n_rot) {
  if (!m || B <= 0 || n_rot < 1 || n_rot > m->d.J) return 0;
  return smplx_bwd_workspace(m->d, B, n_rot, nullptr).bytes;
}

extern "C" int shapy_smplx_backward(const shapy_smplx_t *m, const float *betas, const float *rot, int n_rot,
                                    const float *expr, const float *camera, int B, const float *grad_vertices,
                                    const float *grad_v_shaped, const float *grad_joints,
                                    const float *grad_proj_joints, float *grad_betas, float *grad_rot,
                                    float *grad_expr, float *grad_camera, void *workspace, size_t workspace_bytes,
                                    void *stream) {
  SHAPY_REQUIRE(m && betas && rot, "shapy_smplx_backward: null argument");
  SHAPY_REQUIRE(B >= 0, "shapy_smplx_backward: batch %d", B);
  SHAPY_REQUIRE(n_rot >= 1 && n_rot <= m->d.J, "shapy_smplx_backward: n_rot %d out of range", n_rot);
  SHAPY_REQUIRE(!((grad_proj_joints || grad_camera) && !camera),
                "shapy_smplx_backward: grad_proj_joints and grad_camera require camera");
  SHAPY_REQUIRE(!(grad_expr && m->d.NE == 0), "shapy_smplx_backward: grad_expr of a model without expression basis");
  if (B == 0) return SHAPY_OK;
  SHAPY_REQUIRE(workspace && workspace_bytes >= shapy_smplx_backward_workspace_bytes(m, B, n_rot),
                "shapy_smplx_backward: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const SmplxDev &d = m->d;
  const SmplxBwdWorkspace ws = smplx_bwd_workspace(d, B, n_rot, workspace);
  const int Kp = (n_rot - 1) * 9, V3 = d.V * 3;
  const float *ex = d.NE ? expr : nullptr;
  const bool chain = grad_betas || grad_rot || grad_expr;   // anything behind the vertices and the chain
  const bool kp = grad_joints || grad_proj_joints;          // keypoint cotangents
  const bool cam = grad_camera && grad_proj_joints;         // the camera gradient reads the forward joints
  if (!chain && !grad_camera) return SHAPY_OK;
  // ---- recompute: A, LUT rows, posed joints, pose offsets (the forward's launches, bit for bit)
  const bool gemm = (chain || cam) && Kp > 0;
  PoseArgs pa{d, betas, ex, rot, n_rot, B, bpad(B), Kp, pose_kpad(Kp), ws.f.A, ws.f.pfT, ws.f.joints, ws.f.lut,
              gemm ? ws.f.x_hi : nullptr, gemm ? ws.f.x_lo : nullptr};
  smplx_pose_kernel<<<B, 128, 0, st>>>(pa);
  SHAPY_LAUNCH_CHECK();
  VertexArgs va{d, betas, ex, ws.f.A, ws.f.pfT, B, bpad(B), nullptr, nullptr, nullptr, nullptr, 0};
  if (gemm) {
    const int rc = pose_blend_gemm(m, B, Kp, ws.f, st, va);
    if (rc != SHAPY_OK) return rc;
  }
  const dim3 vgrid(ceil_div(d.V, TV), ceil_div(B, TB));
  if (cam) {   // the forward's vertices (into gv, free until the vertex backward) and joints
    VertexArgs vf = va;
    vf.vertices = ws.gv;
    smplx_vertex_kernel<<<vgrid, 128, 0, st>>>(vf);
    SHAPY_LAUNCH_CHECK();
    if (d.L + d.D + d.n_extra > 0) {
      const int rc = launch_joints(d, ws.gv, nullptr, ws.f.lut, B, ws.f.joints, nullptr, st);
      if (rc != SHAPY_OK) return rc;
    }
  }
  // ---- adjoints
  if (kp || grad_camera) {
    JointsBwdArgs ja{d, ws.f.joints, camera, grad_joints, grad_proj_joints, chain ? ws.gP : nullptr, ws.gkp,
                     grad_camera};
    const size_t smem = ((size_t)d.K * 3 + (size_t)std::max(d.n_extra, 1) * 3) * sizeof(float);
    smplx_joints_bwd_kernel<<<B, 128, smem, st>>>(ja);
    SHAPY_LAUNCH_CHECK();
  }
  if (!chain) return SHAPY_OK;
  VertexBwdArgs vb{va, grad_vertices, kp ? ws.gkp : nullptr, ws.f.lut, ws.vp, ws.gv, ws.gvp};
  smplx_vertex_bwd_kernel<<<vgrid, 128, 0, st>>>(vb);
  SHAPY_LAUNCH_CHECK();
  smplx_skin_bwd_kernel<<<B, 256, 0, st>>>(d, ws.gv, ws.vp, ws.gA);
  SHAPY_LAUNCH_CHECK();
  const bool pf = grad_rot && Kp > 0;
  if (pf) {
    smplx_posefeat_bwd_kernel<<<dim3(ceil_div(Kp, kPfTK), ceil_div(B, kPfTB), kPfSplit), 256, 0, st>>>(
        d.posedirs, ws.gvp, V3, Kp, B, ws.pf_part);
    SHAPY_LAUNCH_CHECK();
  }
  int NR = 0;   // basis rows of the shape adjoint: the shape rows, and the expression rows when their gradient is wanted
  if (grad_betas || grad_expr) {
    NR = grad_expr ? d.NC : d.NB;
    if (d.NB == 10 && NR == 10) {
      smplx_shape_bwd_kernel<10, 0, kShapeTile><<<dim3(ceil_div(B, kShapeTile), kShapeSplit), 256, 0, st>>>(
          d.basis, d.V3p, ws.gvp, grad_v_shaped, V3, B, ws.shape_part);
    } else if (d.NB == 10 && NR == 20) {
      smplx_shape_bwd_kernel<10, 10, 4><<<dim3(ceil_div(B, 4), kShapeSplit), 256, 0, st>>>(
          d.basis, d.V3p, ws.gvp, grad_v_shaped, V3, B, ws.shape_part);
    } else {
      smplx_shape_bwd_kernel_generic<<<dim3(B, kShapeSplit, NR), 256, 0, st>>>(d.basis, d.V3p, ws.gvp, grad_v_shaped,
                                                                               d.NB, NR, V3, ws.shape_part);
    }
    SHAPY_LAUNCH_CHECK();
    smplx_shape_bwd_sum_kernel<<<ceil_div(B * NR, 256), 256, 0, st>>>(ws.shape_part, NR, B, ws.gcoef);
    SHAPY_LAUNCH_CHECK();
  }
  ChainBwdArgs ca{d, betas, ex, rot, n_rot, Kp, ws.gA, kp ? ws.gP : nullptr, pf ? ws.pf_part : nullptr,
                  NR ? ws.gcoef : nullptr, NR, grad_rot, grad_betas, grad_expr};
  smplx_chain_bwd_kernel<<<B, 128, 0, st>>>(ca);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

extern "C" int shapy_smplx_keypoint_jacobian(const shapy_smplx_t *m, const float *betas, const float *rot, int n_rot,
                                             const float *transl, int B, float *keypoints, float *jac, void *stream) {
  SHAPY_REQUIRE(m && betas && rot && keypoints && jac, "shapy_smplx_keypoint_jacobian: null argument");
  SHAPY_REQUIRE(B >= 0, "shapy_smplx_keypoint_jacobian: batch %d", B);
  SHAPY_REQUIRE(n_rot >= 1 && n_rot <= m->d.J, "shapy_smplx_keypoint_jacobian: n_rot %d out of range", n_rot);
  if (B == 0) return SHAPY_OK;
  const SmplxDev &d = m->d;
  const int n_entries = 3 * (d.L + d.D) + m->extra_nnz;
  const int cached = n_entries <= kKpCacheEntries;
  const size_t smem = cached ? (size_t)n_entries * kKpState * sizeof(float) : 0;
  // the static shared memory (33.6 KB) plus the entry cache passes the 48 KB a launch gets without opting in
  if (smem > 0)
    SHAPY_CUDA_TRY(cudaFuncSetAttribute(smplx_kp_jac_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  KpJacArgs a{d, betas, rot, transl, n_rot, (n_rot - 1) * 9, 3 * n_rot + d.NB + 3, n_entries, cached, keypoints, jac};
  smplx_kp_jac_kernel<<<B, kKpJacThreads, smem, (cudaStream_t)stream>>>(a);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

extern "C" int shapy_smplx_keypoint_jacobian_expr(const shapy_smplx_t *m, const float *betas, const float *expr,
                                                  const float *rot, int n_rot, const float *transl, int B,
                                                  float *keypoints, float *jac, void *stream) {
  SHAPY_REQUIRE(m && betas && expr && rot && keypoints && jac, "shapy_smplx_keypoint_jacobian_expr: null argument");
  SHAPY_REQUIRE(B >= 0, "shapy_smplx_keypoint_jacobian_expr: batch %d", B);
  SHAPY_REQUIRE(n_rot >= 1 && n_rot <= m->d.J, "shapy_smplx_keypoint_jacobian_expr: n_rot %d out of range", n_rot);
  SHAPY_REQUIRE(m->d.NE >= 1, "shapy_smplx_keypoint_jacobian_expr: the model has no expression basis");
  if (B == 0) return SHAPY_OK;
  const SmplxDev &d = m->d;
  const int n_entries = 3 * (d.L + d.D) + m->extra_nnz;
  const int cached = n_entries <= kKpCacheEntries;
  const size_t smem = cached ? (size_t)n_entries * kKpState * sizeof(float) : 0;
  if (smem > 0)
    SHAPY_CUDA_TRY(
        cudaFuncSetAttribute(smplx_kp_jac_expr_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  KpJacExprArgs a;
  static_cast<KpJacArgs &>(a) =
      KpJacArgs{d, betas, rot, transl, n_rot, (n_rot - 1) * 9, 3 * n_rot + d.NC + 3, n_entries, cached, keypoints, jac};
  a.expr = expr;
  smplx_kp_jac_expr_kernel<<<B, kKpJacThreads, smem, (cudaStream_t)stream>>>(a);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

extern "C" int shapy_smplx_vertex_jacobian(const shapy_smplx_t *m, const float *betas, const float *rot, int n_rot,
                                           const float *transl, int B, float *vertices, float *jac, void *stream) {
  SHAPY_REQUIRE(m && betas && rot && vertices && jac, "shapy_smplx_vertex_jacobian: null argument");
  SHAPY_REQUIRE(B >= 0 && B <= 65535, "shapy_smplx_vertex_jacobian: batch %d", B);
  SHAPY_REQUIRE(n_rot >= 1 && n_rot <= m->d.J, "shapy_smplx_vertex_jacobian: n_rot %d out of range", n_rot);
  if (B == 0) return SHAPY_OK;
  const SmplxDev &d = m->d;
  const int P = 3 * n_rot + d.NB + 3;
  const size_t smem = (size_t)kVjTile * 3 * P * sizeof(float);
  SHAPY_CUDA_TRY(cudaFuncSetAttribute(smplx_vertex_jac_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  VertJacArgs a{d, betas, rot, transl, n_rot, (n_rot - 1) * 9, P, vertices, jac};
  smplx_vertex_jac_kernel<<<dim3(ceil_div(d.V, kVjTile), B), kKpJacThreads, smem, (cudaStream_t)stream>>>(a);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}
