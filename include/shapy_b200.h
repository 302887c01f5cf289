/* shapy_b200 -- C ABI of the H100-native (sm_90a) SHAPY inference hot path.
 *
 * Every entry point is `extern "C"`, takes plain pointers / sizes / a CUDA stream
 * (passed as void* so the header needs no CUDA include) and returns 0 on success or
 * a negative shapy_b200 error / positive cudaError_t code; shapy_last_error() gives
 * the message.  No torch types.  All device work is stream-ordered on `stream`; no
 * call synchronises the device.  Outputs are caller-owned device buffers.
 *
 * What each entry point replaces in the reference (paths relative to the reference
 * repo, see SURVEY.md section 8):
 *
 *   shapy_smplx_*        lbs()                      regressor/human_shape/models/body_models/lbs.py:99-196
 *                        SMPLX.forward              regressor/human_shape/models/body_models/body_models.py:628-767
 *                        SMPL.forward_shape         body_models.py:292-302
 *                        ContinuousRotReprDecoder   regressor/human_shape/models/common/pose_utils.py:138-153
 *                        WeakPerspectiveCamera      regressor/human_shape/models/camera/camera_projection.py:181-213
 *   shapy_measure_*      BodyMeasurements.forward   mesh-mesh-intersection/body_measurements/body_measurements.py:217-246
 *   shapy_mmi_forward    mesh_to_mesh_forward       mesh-mesh-intersection/src/mesh_mesh_intersect.cpp:36-64
 *   shapy_mmi_forward_f64  (float / float64)        + src/mesh_mesh_intersect_cuda_op.cu:969-1079
 *   shapy_closest_points, shapy_nearest_points, shapy_closest_points_backward   (no reference counterpart: the scan
 *                        terms of shapy_b200.fit.fit_body_to_scan, on the LBVH of shapy_mmi_forward)
 *   shapy_head_*         IterativeRegression.forward regressor/human_shape/models/common/networks.py:536-592
 *   shapy_hrnet_*        HighResolutionNet.forward  regressor/human_shape/models/backbone/hrnet.py:426-498
 *   shapy_p2p_error      v2vhdError.__call__        regressor/human_shape/utils/metrics.py:368-456
 *   shapy_v2v_error      PointError, translation / no alignment   metrics.py:85-98, 232-277, 335-366
 *   shapy_point_error_aligned   PointError, scale / root alignment   metrics.py:173-229, 279-303, 335-366
 *   shapy_regress_points        J14 joint regression of mpjpe14    regressor/human_shape/evaluation.py:161-190
 */
#ifndef SHAPY_B200_H_
#define SHAPY_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SHAPY_OK 0
#define SHAPY_ERR_ARG (-1)      /* bad argument (null pointer, unsupported size) */
#define SHAPY_ERR_STATE (-2)    /* object not bound / wrong device */
#define SHAPY_ERR_UNSUPPORTED (-3)
#define SHAPY_ERR_OVERFLOW (-4) /* a fixed-capacity device buffer overflowed */

const char *shapy_last_error(void);
int shapy_version(void);
/* number of kernels this library launched since process start (all entry points) */
long long shapy_launch_count(void);

/* ------------------------------------------------------------------ SMPL-X */
typedef struct shapy_smplx shapy_smplx_t;

/* Dense model tensors exactly as the reference registers them as buffers
 * (body_models.py:112-166, 563-597).  HOST pointers, fp32 / int64, row-major. */
typedef struct {
  int num_verts;               /* V  (10475) */
  int num_joints;              /* J  (55)    */
  int num_betas;               /* NB (10)  shapedirs is (V,3,NB) */
  int num_expr;                /* NE (10)  expr_dirs is (V,3,NE); may be 0 */
  int num_faces;               /* F  (20908) */
  const float *v_template;     /* (V,3) */
  const float *shapedirs;      /* (V,3,NB) */
  const float *expr_dirs;      /* (V,3,NE) or NULL */
  const float *posedirs;       /* ((J-1)*9, V*3) */
  const float *J_regressor;    /* (J,V) */
  const float *lbs_weights;    /* (V,J) */
  const int64_t *parents;      /* (J), parents[0] = -1 */
  const int64_t *faces;        /* (F,3) */
  int num_static_lmk;          /* 51 */
  const int64_t *lmk_faces_idx;        /* (L) */
  const float *lmk_bary_coords;        /* (L,3) */
  int num_dyn_lmk;             /* 17, 0 disables use_face_contour */
  int num_dyn_rows;            /* 79 */
  const int64_t *dynamic_lmk_faces_idx;   /* (rows, D) */
  const float *dynamic_lmk_bary_coords;   /* (rows, D, 3) */
  int neck_chain_len;          /* 6 */
  const int64_t *neck_kin_chain;       /* e.g. [15,12,9,6,3,0] */
  int num_extra;               /* 14 rows of the J14 regressor, 0 disables */
  const float *extra_joint_regressor;  /* (num_extra, V) */
  int num_overwrite;           /* len(source_idxs) */
  const int64_t *source_idxs;  /* joints[:, source] = reg[:, target] */
  const int64_t *target_idxs;
} shapy_smplx_desc_t;

int shapy_smplx_create(shapy_smplx_t **out, const shapy_smplx_desc_t *desc);
void shapy_smplx_destroy(shapy_smplx_t *m);
int shapy_smplx_num_keypoints(const shapy_smplx_t *m);          /* J + L + D (123) */
const int32_t *shapy_smplx_faces_i32(const shapy_smplx_t *m);   /* device (F,3) int32 */
size_t shapy_smplx_workspace_bytes(const shapy_smplx_t *m, int batch);

/* 6D -> rotation matrices: raw (n, 6) row-major 3x2 -> rot (n, 3, 3). */
int shapy_decode_rot6d(const float *raw, int n, float *rot, void *stream);

/* Full SMPL-X evaluation for `batch` bodies.
 *   betas   (B, NB)                 device fp32
 *   rot     (B, n_rot, 3, 3)        rotations of the first n_rot joints of the full pose
 *                                   [global, body(21), jaw, leye, reye, lhand(15), rhand(15)];
 *                                   the remaining joints are identity (SHAPY_A: n_rot = 22)
 *   expr    (B, NE) or NULL (zeros)
 *   camera  (B, 3) or NULL; when given, proj_joints = softplus(c0) * (joints_xy + c[1:3])
 * outputs (any may be NULL): vertices (B,V,3), v_shaped (B,V,3), joints (B,K,3), proj_joints (B,K,2)
 */
int shapy_smplx_forward(const shapy_smplx_t *m, const float *betas, const float *rot, int n_rot,
                        const float *expr, const float *camera, int batch, float *vertices, float *v_shaped,
                        float *joints, float *proj_joints, void *workspace, size_t workspace_bytes,
                        void *stream);

/* v_shaped = v_template + shapedirs . betas  (T-pose path, BASELINE configs 1 and 4) */
int shapy_smplx_forward_shape(const shapy_smplx_t *m, const float *betas, int batch, float *v_shaped,
                              void *stream);

/* Adjoint of shapy_smplx_forward_shape (the betas term of lbs.blend_shapes, lbs.py:207-225, under autograd):
 * grad_betas (B,NB) = shapedirs^T . grad_v_shaped (B,V,3), device fp32.  Deterministic; a body's result does not
 * depend on the rest of the batch.  workspace: device, >= shapy_smplx_backward_shape_workspace_bytes(m, batch). */
size_t shapy_smplx_backward_shape_workspace_bytes(const shapy_smplx_t *m, int batch);
int shapy_smplx_backward_shape(const shapy_smplx_t *m, const float *grad_v_shaped, int batch, float *grad_betas,
                               void *workspace, size_t workspace_bytes, void *stream);

/* Adjoint of shapy_smplx_forward (the reference's lbs() and SMPLX.forward under autograd, pose2rot=False), first
 * order.  Inputs as in shapy_smplx_forward; it recomputes the forward from them, nothing is kept between the calls.
 *   cotangents (any may be NULL = zero): grad_vertices (B,V,3), grad_v_shaped (B,V,3), grad_joints (B,K,3),
 *                                        grad_proj_joints (B,K,2)
 *   gradients  (any may be NULL = not wanted): grad_betas (B,NB), grad_rot (B,n_rot,3,3), grad_expr (B,NE),
 *                                        grad_camera (B,3)
 * Semantics: a rotation's gradient is the raw dL/dR (9 entries, no tangent projection); v_shaped carries no
 * expression, so its cotangent reaches betas only; the dynamic-contour LUT row is a constant (the barycentric mix of
 * its vertices is differentiated); an overwritten J14 keypoint's cotangent goes to the J14 regression of the
 * vertices, not to the joint or landmark it replaced; proj = softplus(c0) (xy + c[1:3]) with softplus' threshold 20.
 * grad_expr is the gradient at expr (zeros when expr is NULL).  grad_proj_joints and grad_camera require camera.
 * Deterministic, no atomics; a body's gradient does not depend on the rest of the batch.  batch 0: no launch.
 * workspace: device, >= shapy_smplx_backward_workspace_bytes(m, batch, n_rot) (about 3 x 12 V bytes per body). */
size_t shapy_smplx_backward_workspace_bytes(const shapy_smplx_t *m, int batch, int n_rot);
int shapy_smplx_backward(const shapy_smplx_t *m, const float *betas, const float *rot, int n_rot, const float *expr,
                         const float *camera, int batch, const float *grad_vertices, const float *grad_v_shaped,
                         const float *grad_joints, const float *grad_proj_joints, float *grad_betas, float *grad_rot,
                         float *grad_expr, float *grad_camera, void *workspace, size_t workspace_bytes, void *stream);

/* The keypoints of shapy_smplx_forward (its `joints`, expression zero) plus transl, and their Jacobian, in one launch.
 *   betas (B,NB), rot (B,n_rot,3,3) as in shapy_smplx_forward (joints >= n_rot are the identity), transl (B,3) or
 *   NULL (zero); outputs keypoints (B,K,3) and jac (B,3K,P) fp32, rows keypoint-major in xyz order, device.
 * Columns, P = 3 n_rot + NB + 3: delta_j (3 per joint j < n_rot, the right-multiplied tangent R_j Exp(delta_j) at
 * delta = 0), then betas, then transl.  Semantics of shapy_smplx_backward: the dynamic-contour LUT row is a constant,
 * an overwritten J14 keypoint takes the J14 row's derivative, the model buffers are constants.  Only the vertices the
 * landmarks and J14 rows reference are evaluated (v_posed from the fp32 posedirs rows below 9 (n_rot - 1)); the cost
 * grows with the J14 regressor's non-zeros.  The keypoints agree with shapy_smplx_forward to fp32 rounding (its pose
 * blend is the split-fp16 GEMM).  No atomics: a body's result is bit-identical from run to run and independent of the
 * rest of the batch.  1 <= n_rot <= J; batch 0: no launch. */
int shapy_smplx_keypoint_jacobian(const shapy_smplx_t *m, const float *betas, const float *rot, int n_rot,
                                  const float *transl, int batch, float *keypoints, float *jac, void *stream);

/* shapy_smplx_keypoint_jacobian at a non-zero facial expression, with its columns: expr (B,NE) as in
 * shapy_smplx_forward, P = 3 n_rot + NB + NE + 3, the columns [delta_j | betas | expression | transl].  The expression
 * rows are rows NB .. NC-1 of the shape basis, so their columns have the betas columns' form.  At expr = 0 the keypoints
 * and every column but the expression's are shapy_smplx_keypoint_jacobian's bit for bit.  SHAPY_ERR_ARG for a model
 * without an expression basis; otherwise the same rules. */
int shapy_smplx_keypoint_jacobian_expr(const shapy_smplx_t *m, const float *betas, const float *expr, const float *rot,
                                       int n_rot, const float *transl, int batch, float *keypoints, float *jac,
                                       void *stream);

/* Every posed vertex and its Jacobian, for the dense fits: betas (B,NB), rot (B,n_rot,3,3), transl (B,3) or NULL
 * (zero); outputs vertices (B,V,3) and jac (B,V,3,P) fp32, row 3 v + c the c coordinate of vertex v, with the columns
 * of shapy_smplx_keypoint_jacobian (P = 3 n_rot + NB + 3: delta_j, betas, transl) and its semantics (v_posed from the
 * fp32 posedirs rows, the model buffers constants); a barycentric mix of three vertices' rows is the keypoint
 * Jacobian's row of a landmark on that face up to fp32 rounding, and the vertices agree with shapy_smplx_forward to
 * fp32 rounding.  The output is large: 4 V 3 P bytes per body, 9.9 MB at V = 10475 and P = 79 (635 MB at B = 64).
 * One CTA per (tile of 32 vertices, body), each recomputing its body's kinematic chain.  No atomics: a body's result is
 * bit-identical from run to run and independent of the rest of the batch.  1 <= n_rot <= J, B <= 65535 (SHAPY_ERR_ARG
 * otherwise); batch 0: no launch. */
int shapy_smplx_vertex_jacobian(const shapy_smplx_t *m, const float *betas, const float *rot, int n_rot,
                                const float *transl, int batch, float *vertices, float *jac, void *stream);

/* Adjoint of shapy_decode_rot6d: grad_raw (n, 6) from raw (n, 6) and grad_rot (n, 3, 3), elementwise.  The 1e-12
 * clamp of each norm passes gradient to the norm only where the norm is >= 1e-12 (torch's clamp_min). */
int shapy_decode_rot6d_backward(const float *raw, int n, const float *grad_rot, float *grad_raw, void *stream);

/* ------------------------------------------------------- virtual measurements */
typedef struct {
  int face_idx[5];      /* head_top, left_heel, chest, waist, hips landmark faces */
  float bc[5][3];       /* barycentrics */
} shapy_measure_landmarks_t;

/* v_shaped (B,V,3), faces int32 (F,3) device.  out (B,5) = mass, height, chest, waist, hips.
 * plane_points (optional, (B,3,max_points,3)) / plane_counts (optional, (B,3) int32) receive the
 * reference-selected intersection points of each slicing plane.  status (device int32[1], may be
 * NULL) is set non-zero if any plane exceeded max_points (SHAPY_ERR_OVERFLOW semantics). */
int shapy_measure_forward(const float *v_shaped, const int32_t *faces, int batch, int num_verts, int num_faces,
                          const shapy_measure_landmarks_t *lm, float *out, float *plane_points,
                          int32_t *plane_counts, int max_points, int32_t *status, void *stream);

/* Same on explicit triangles (B,F,3,3) -- the tensor BodyMeasurements.forward receives. */
int shapy_measure_forward_tris(const float *triangles, int batch, int num_faces,
                               const shapy_measure_landmarks_t *lm, float *out, float *plane_points,
                               int32_t *plane_counts, int max_points, int32_t *status, void *stream);

/* Backward of shapy_measure_forward with the reference's autograd semantics (body_measurements.py:137-173 for the
 * circumferences, 182-199 height, 201-215 mass): grad_out (B,5) device -> grad_v (B,V,3) device, overwritten.
 * The intersection points' barycentrics are constants (the reference selects them under no_grad, 137-139) and the
 * plane height gets no gradient, so for the circumferences this is not what a finite difference of the mesh gives.
 * inc_ptr (V+1) / inc (3F) int32 device: the vertex -> (face, corner) incidence of `faces` in CSR form, entries
 * 3 f + k in ascending order per vertex.  The hull is recomputed from v_shaped (no forward state); the result is
 * bit-identical from run to run and independent of the rest of the batch.  Where a circumference is NaN and its
 * upstream gradient is non-zero, the body's whole gradient is NaN. */
int shapy_measure_backward(const float *v_shaped, const int32_t *faces, const int32_t *inc_ptr, const int32_t *inc,
                           int batch, int num_verts, int num_faces, const shapy_measure_landmarks_t *lm,
                           const float *grad_out, float *grad_v, void *stream);

/* Same on explicit triangles (B,F,3,3) -> grad_triangles (B,F,3,3) (BodyMeasurements.forward's input). */
int shapy_measure_backward_tris(const float *triangles, int batch, int num_faces,
                                const shapy_measure_landmarks_t *lm, const float *grad_out,
                                float *grad_triangles, void *stream);

/* The measurements of shapy_measure_forward and their Jacobian with respect to betas, in one launch:
 * out (B,5) bit-identical to shapy_measure_forward on the same v_shaped (NaNs included), jac (B,5,NB) device fp32,
 * row k = shapedirs^T . (the gradient shapy_measure_backward gives for the cotangent e_k), with its semantics (constant
 * barycentrics, no gradient through the plane heights, sign(0) = 0).  Faces, V and NB come from the model; v_shaped
 * (B,V,3), 16-byte aligned, need not come from shapy_smplx_forward_shape.  inc_ptr / inc: the incidence table of the model's faces, as
 * for shapy_measure_backward.  A NaN circumference makes its row NaN, the other rows stay finite; an inconsistent
 * hull walk makes the body's five rows NaN.  status as in shapy_measure_forward.  No atomics touch out or jac: a
 * body's result is bit-identical from run to run and independent of the rest of the batch.  1 <= NB <= 16, else
 * SHAPY_ERR_UNSUPPORTED. */
int shapy_measure_jacobian_betas(const shapy_smplx_t *m, const float *v_shaped, const int32_t *inc_ptr,
                                 const int32_t *inc, int batch, const shapy_measure_landmarks_t *lm,
                                 float *out, float *jac, int32_t *status, void *stream);

/* The _exact entries: shapy_measure_backward, shapy_measure_backward_tris and shapy_measure_jacobian_betas with the
 * exact derivative of the chest, waist and hip circumferences instead of the reference's autograd semantics.  With
 * the hull's combinatorics held fixed (which points, in what order, from which face and ray), each hull point moves
 * with its triangle's corners and with the plane height h = bc . y of its landmark face: a point on a triangle edge
 * a -> b is a + s (b - a) with s = (h - a_y) / (b_y - a_y), a point where a query-quad edge pierces the triangle is
 * the line-plane intersection, and a point without a ray hit is a constant.  The height's adjoint reaches the y
 * components of the landmark face's corners, weighted by its barycentrics.  This is the derivative of the measured
 * circumference wherever the hull's combinatorics do not change.  Mass and height terms and rows, the measurements,
 * the NaN rules, determinism and batch independence are those of the non-exact entries, bit for bit. */
int shapy_measure_backward_exact(const float *v_shaped, const int32_t *faces, const int32_t *inc_ptr,
                                 const int32_t *inc, int batch, int num_verts, int num_faces,
                                 const shapy_measure_landmarks_t *lm, const float *grad_out, float *grad_v,
                                 void *stream);
int shapy_measure_backward_tris_exact(const float *triangles, int batch, int num_faces,
                                      const shapy_measure_landmarks_t *lm, const float *grad_out,
                                      float *grad_triangles, void *stream);
int shapy_measure_jacobian_betas_exact(const shapy_smplx_t *m, const float *v_shaped, const int32_t *inc_ptr,
                                       const int32_t *inc, int batch, const shapy_measure_landmarks_t *lm,
                                       float *out, float *jac, int32_t *status, void *stream);

/* One Levenberg-Marquardt step per body of the fit of betas to the five measurements, one warp per body.  Loss
 * L = sum_{w_k > 0} w_k (t_k - m_k)^2 + betas_weight |beta|^2; a term with weight 0 is skipped (its measurement and
 * Jacobian row may be NaN).  targets, weights (B,5); the state betas (B,NB), meas (B,5), jac (B,5,NB), loss (B),
 * lambda (B), accepted (B, a count); trial (B,NB) is the point whose trial_meas (B,5) / trial_jac (B,5,NB) were
 * evaluated, and receives the next trial.  With `first` the trial becomes the state and lambda = 1e-3 max(diag
 * (J^T W J), 1e-6); otherwise a finite trial loss below the state's is accepted (state := trial, lambda /= lambda_down,
 * accepted += 1) and any other rejected (lambda *= lambda_up).  lambda is clamped to [1e-9, 1e9].  The next trial is
 * beta + delta, (J^T W J + (betas_weight + lambda) I) delta = -(J^T W (m - t) + betas_weight beta), by Cholesky in
 * fp64; a body whose loss is not finite, or whose factorisation fails, gets its state as the trial.  A non-finite
 * starting loss is reported as NaN.  Deterministic, no atomics, per-body independent.  1 <= NB <= 16. */
int shapy_fit_lm_step(int batch, int nb, const float *targets, const float *weights, float betas_weight,
                      float lambda_up, float lambda_down, int first, float *betas, float *meas, float *jac,
                      float *loss, float *lambda, int32_t *accepted, float *trial, const float *trial_meas,
                      const float *trial_jac, void *stream);

/* One Levenberg-Marquardt step per body of the fit of pose and shape to K 3D keypoints, one CTA per body, with
 * shapy_fit_lm_step's policy and lambda constants.  Parameters as the columns of shapy_smplx_keypoint_jacobian,
 * P = 3 n_rot + nb + 3.  Loss L = sum_{w_k > 0} w_k |kp_k - target_k|^2 in fp64, k order; a keypoint with weight
 * <= 0 is dropped (its rows are never read).  targets (B,K,3), weights (B,K); the state rot (B,n_rot,3,3), betas
 * (B,nb), transl (B,3), keypoints (B,K,3), jac (B,3K,P), loss (B), lambda (B), accepted (B, a count); trial_rot /
 * trial_betas / trial_transl is the point whose trial_keypoints / trial_jac were evaluated, and receives the next
 * trial.  With `first` the trial becomes the state and lambda = 1e-3 max(diag(J^T W J), 1e-6); otherwise a finite
 * trial loss below the state's is accepted (state := trial, lambda /= lambda_down, accepted += 1) and any other
 * rejected (lambda *= lambda_up); lambda is clamped to [1e-9, 1e9].  (J^T W J + lambda I) delta = -J^T W (kp - target)
 * by Cholesky in fp64; the next trial is R_j Exp(delta_j) (Rodrigues in fp64, re-orthonormalised by the 6D decoder's
 * Gram-Schmidt of the first two columns), beta + delta_beta, t + delta_t, rounded to fp32.  A body whose loss is not
 * finite, or whose factorisation fails, gets its state as the trial; a non-finite starting loss is reported as NaN.
 * Deterministic, no atomics, per-body independent.  P > 96: SHAPY_ERR_UNSUPPORTED.  batch 0: no launch. */
int shapy_fit_lm_keypoints_step(int batch, int num_keypoints, int n_rot, int nb, const float *targets,
                                const float *weights, float lambda_up, float lambda_down, int first, float *rot,
                                float *betas, float *transl, float *keypoints, float *jac, float *loss, float *lambda,
                                int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_transl,
                                const float *trial_keypoints, const float *trial_jac, void *stream);

/* shapy_fit_lm_keypoints_step with the five virtual measurements and a betas regulariser stacked under the keypoint
 * rows: one Gauss-Newton step on L = L_kp + sum_{w_k > 0} w_k (t_k - m_k)^2 + betas_weight |beta|^2, summed left to
 * right, L_kp as in shapy_fit_lm_keypoints_step, the measurement terms in k order (mass, height, chest, waist, hips),
 * |beta|^2 in l order.  meas_targets, meas_weights (B,5); the state adds meas (B,5) and meas_jac (B,5,nb), the trial
 * trial_meas / trial_meas_jac (shapy_measure_jacobian_betas at the trial betas); on accept they are copied into the
 * state too.  A measurement with weight <= 0 is dropped (its value and Jacobian row are never read and may be NaN); a
 * weighted NaN trial measurement makes the trial loss NaN, so the trial is rejected.  Normal equations: A = J_kp^T W
 * J_kp, then + J_m^T W_m J_m in the betas block (k order); g = J_kp^T W (kp - target), then + J_m^T W_m (m - t), then
 * + betas_weight beta.  The first lambda is 1e-3 max(diag A, 1e-6), without betas_weight; the diagonal then gets
 * betas_weight + lambda on the betas columns and lambda elsewhere.  The policy, the solve and the next trial are those
 * of shapy_fit_lm_keypoints_step.  With every measurement weight <= 0 and betas_weight = 0 the outputs equal
 * shapy_fit_lm_keypoints_step's bit for bit.  A null pointer, betas_weight < 0 or a lambda factor < 1:
 * SHAPY_ERR_ARG; P > 96: SHAPY_ERR_UNSUPPORTED.  batch 0: no launch. */
int shapy_fit_lm_keypoints_measurements_step(
    int batch, int num_keypoints, int n_rot, int nb, const float *targets, const float *weights,
    const float *meas_targets, const float *meas_weights, float betas_weight, float lambda_up, float lambda_down,
    int first, float *rot, float *betas, float *transl, float *keypoints, float *jac, float *meas, float *meas_jac,
    float *loss, float *lambda, int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_transl,
    const float *trial_keypoints, const float *trial_jac, const float *trial_meas, const float *trial_meas_jac,
    void *stream);

/* One Levenberg-Marquardt step per body of the fit of pose, shape and weak-perspective camera to K 2D keypoints, one
 * CTA per body, with shapy_fit_lm_keypoints_step's policy, lambda constants, solve and rotation update.  Parameters
 * [delta_j (3 n_rot) | beta (nb) | c0, c1, c2], P = 3 n_rot + nb + 3: the camera (B,3) of shapy_smplx_forward takes
 * the place of transl, p_k = softplus(c0) (kp_k,xy + (c1, c2)) with the forward's softplus threshold of 20.  Loss, fp64,
 * left to right: sum_{w_k > 0} w_k rho(|p_k - x_k|^2) (k order) + pose_prior_weight / 2 sum_{j = 1}^{n_rot - 1}
 * |R_j - R0_j|_F^2 + betas_weight |beta|^2; rho(e) = e when robust_sigma = +inf, else sigma^2 e / (sigma^2 + e)
 * (Geman-McClure).  A keypoint with weight <= 0 is dropped (its target, keypoint and rows are never read).
 * targets (B,K,2) in the frame of proj_joints, weights (B,K), pose_anchor (B,n_rot,3,3) the rotations R0 (read only
 * when pose_prior_weight > 0, may be null otherwise).  The state rot (B,n_rot,3,3), betas (B,nb), camera (B,3),
 * keypoints (B,K,3) and jac (B,3K,P) are those of shapy_smplx_keypoint_jacobian without transl (its transl columns
 * are not read), loss (B), lambda (B), accepted (B, a count); trial_rot / trial_betas / trial_camera is the point
 * whose trial_keypoints / trial_jac were evaluated, and receives the next trial.  Gauss-Newton rows: the x and y rows
 * of the keypoints, projected (s J on the rotation and betas columns, ds/dc0 (kp_xy + c_xy) on c0, s on c1 / c2),
 * weighted by w_k rho'(e_k) = w_k sigma^4 / (sigma^2 + e_k)^2 at the state (IRLS); then per prior joint the nine
 * rows (R_j - R0_j) / sqrt(2) with Jacobian R_j [e_a]x / sqrt(2) in its three columns; then betas_weight beta in the
 * gradient.  The first lambda is 1e-3 max(diag, 1e-6) of the keypoint rows alone; the diagonal gets betas_weight +
 * lambda on the betas columns and lambda elsewhere.  Accept / reject compares the true robust losses, so a body's loss
 * never increases.  The next trial is R_j Exp(delta_j), beta + delta_beta, c + delta_c.  A null pointer,
 * robust_sigma <= 0 or NaN, a negative prior weight or a lambda factor < 1: SHAPY_ERR_ARG; P > 96:
 * SHAPY_ERR_UNSUPPORTED.  batch 0: no launch.  Deterministic, no atomics, per-body independent. */
int shapy_fit_lm_keypoints_2d_step(int batch, int num_keypoints, int n_rot, int nb, const float *targets,
                                   const float *weights, const float *pose_anchor, float robust_sigma,
                                   float pose_prior_weight, float betas_weight, float lambda_up, float lambda_down,
                                   int first, float *rot, float *betas, float *camera, float *keypoints, float *jac,
                                   float *loss, float *lambda, int32_t *accepted, float *trial_rot, float *trial_betas,
                                   float *trial_camera, const float *trial_keypoints, const float *trial_jac,
                                   void *stream);

/* shapy_fit_lm_keypoints_2d_step with the five virtual measurements stacked under its rows, as
 * shapy_fit_lm_keypoints_measurements_step is to shapy_fit_lm_keypoints_step: one Gauss-Newton step on, in fp64, left
 * to right, L = sum_{w_k > 0} w_k rho(|p_k - x_k|^2) + pose_prior_weight / 2 sum_j |R_j - R0_j|_F^2 +
 * sum_{u_m > 0} u_m (t_m - meas_m)^2 (m order: mass, height, chest, waist, hips; summed on its own, then added) +
 * betas_weight |beta|^2 (the 2D step's betas prior: one regulariser).  2D keypoints fix the proportions of a body and
 * not its metric size (a larger body under a smaller softplus(c0) projects to the same points); a known height or mass
 * removes that freedom.  meas_targets, meas_weights (B,5); the state adds meas (B,5) and meas_jac (B,5,nb), the trial
 * trial_meas / trial_meas_jac (shapy_measure_jacobian_betas or _exact at the trial betas); on accept they are copied
 * into the state too.  A measurement with weight <= 0 is dropped (its value and Jacobian row are never read and may be
 * NaN); a weighted NaN trial measurement makes the trial loss NaN, so the trial is rejected.  Normal equations: the 2D
 * step's keypoint rows (IRLS weights at the state), then its pose-prior rows, then J_m^T U J_m into the betas block and
 * J_m^T U (meas - t) into g in m order (plain least squares: rho applies to keypoints only), then betas_weight beta.
 * The first lambda is 1e-3 max(diag, 1e-6) of the keypoint rows alone, as in the 2D step; policy, damping, solve and
 * next trial are the 2D step's.  With every measurement weight <= 0 every output equals
 * shapy_fit_lm_keypoints_2d_step's bit for bit, for any robust_sigma, pose prior and betas_weight.  Errors as
 * shapy_fit_lm_keypoints_2d_step, the measurement pointers included.  batch 0: no launch.  Deterministic, no atomics,
 * per-body independent. */
int shapy_fit_lm_keypoints_2d_measurements_step(
    int batch, int num_keypoints, int n_rot, int nb, const float *targets, const float *weights,
    const float *pose_anchor, float robust_sigma, float pose_prior_weight, float betas_weight,
    const float *meas_targets, const float *meas_weights, float lambda_up, float lambda_down, int first, float *rot,
    float *betas, float *camera, float *keypoints, float *jac, float *meas, float *meas_jac, float *loss, float *lambda,
    int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_camera, const float *trial_keypoints,
    const float *trial_jac, const float *trial_meas, const float *trial_meas_jac, void *stream);

/* shapy_fit_lm_keypoints_2d_step under a perspective camera with known intrinsics: one Levenberg-Marquardt step per
 * body of the fit of pose, shape and translation to K 2D keypoints.  Camera frame x right, y down, z forward;
 * intrinsics (B,3) = (f, px, py) per body, f > 0, in the units of the targets (pixels, or any other: the kernel does
 * not care).  Parameters [delta_j (3 n_rot) | beta (nb) | t], P = 3 n_rot + nb + 3, the translation t (B,3) in the
 * place of the camera.  With Y_k = kp_k + t (fp64, kp_k the keypoint of shapy_smplx_keypoint_jacobian without transl):
 *   p_k = f (Y_k,x / Y_k,z, Y_k,y / Y_k,z) + (px, py);
 * the loss is the 2D step's term for term with this p_k: sum_{w_k > 0} w_k rho(|p_k - x_k|^2) (k order) +
 * pose_prior_weight / 2 sum_{j >= 1} |R_j - R0_j|_F^2 + betas_weight |beta|^2.  Keypoint rows 2k + c (IRLS weights at
 * the state): (f / Y_z) (J_{3k+c} - (Y_c / Y_z) J_{3k+2}) on the rotation and betas columns, and on the t columns with
 * J_t = I (the transl columns of jac are not read).  Depth rule: a trial with a weighted keypoint at Y_z <= 0 or
 * non-finite has loss +inf and is rejected (a point behind the camera would project mirrored); a start that breaks the
 * rule, or a body whose f is not finite and > 0, has a non-finite loss, reports NaN and does not move.  Pose-prior
 * rows, first lambda, damping, solve and next trial (t + delta_t rounded to fp32) are the 2D step's.  A null
 * intrinsics, like any null pointer, is SHAPY_ERR_ARG; other errors as shapy_fit_lm_keypoints_2d_step.  batch 0: no
 * launch.  Deterministic, no atomics, per-body independent. */
int shapy_fit_lm_keypoints_2d_perspective_step(
    int batch, int num_keypoints, int n_rot, int nb, const float *targets, const float *weights,
    const float *intrinsics, const float *pose_anchor, float robust_sigma, float pose_prior_weight, float betas_weight,
    float lambda_up, float lambda_down, int first, float *rot, float *betas, float *transl, float *keypoints,
    float *jac, float *loss, float *lambda, int32_t *accepted, float *trial_rot, float *trial_betas,
    float *trial_transl, const float *trial_keypoints, const float *trial_jac, void *stream);

/* shapy_fit_lm_keypoints_2d_perspective_step with the five virtual measurements stacked under its rows, as
 * shapy_fit_lm_keypoints_2d_measurements_step is to shapy_fit_lm_keypoints_2d_step (same loss order, rows, first
 * lambda and arguments).  A known height fixes the body's metric size; with a known focal length the projected size
 * then fixes its distance.  With every measurement weight <= 0 every output equals
 * shapy_fit_lm_keypoints_2d_perspective_step's bit for bit. */
int shapy_fit_lm_keypoints_2d_perspective_measurements_step(
    int batch, int num_keypoints, int n_rot, int nb, const float *targets, const float *weights,
    const float *intrinsics, const float *pose_anchor, float robust_sigma, float pose_prior_weight, float betas_weight,
    const float *meas_targets, const float *meas_weights, float lambda_up, float lambda_down, int first, float *rot,
    float *betas, float *transl, float *keypoints, float *jac, float *meas, float *meas_jac, float *loss, float *lambda,
    int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_transl, const float *trial_keypoints,
    const float *trial_jac, const float *trial_meas, const float *trial_meas_jac, void *stream);

/* shapy_fit_lm_keypoints_2d_step for the whole SMPL-X body: any n_rot (the hands, jaw and eyes past joint 21) and ne
 * expression coefficients, P = 3 n_rot + nb + ne + 3 <= 200 (SHAPY_ERR_UNSUPPORTED past that).  Parameters [delta_j
 * (3 n_rot) | beta (nb) | psi (ne) | c], the columns of shapy_smplx_keypoint_jacobian_expr (of
 * shapy_smplx_keypoint_jacobian when ne = 0) without transl.  Loss per body, fp64, left to right: the 2D step's
 * keypoint term and pose prior, + betas_weight |beta|^2, + expression_weight |psi|^2.  joint_weights: null (every
 * joint j >= 1 weighted pose_prior_weight, the 2D step's prior) or (n_rot) device floats w_j, the prior then
 * sum_{j >= 1, w_j > 0} (w_j / 2) |R_j - R0_j|_F^2 (j order; joint 0 is not read and has no prior), which lets the
 * hands, jaw and eyes be held apart from the body.  The expression columns are damped by expression_weight + lambda,
 * the betas columns by betas_weight + lambda, the rest by lambda; g gains expression_weight psi.  expression /
 * trial_expression (B,ne) may be null when ne = 0.  With ne = 0 and joint_weights null every output equals
 * shapy_fit_lm_keypoints_2d_step's bit for bit (at n_rot, nb where that step runs).  Other rules and errors as
 * shapy_fit_lm_keypoints_2d_step. */
int shapy_fit_lm_keypoints_2d_expressive_step(
    int batch, int num_keypoints, int n_rot, int nb, int ne, const float *targets, const float *weights,
    const float *pose_anchor, const float *joint_weights, float robust_sigma, float pose_prior_weight,
    float betas_weight, float expression_weight, float lambda_up, float lambda_down, int first, float *rot,
    float *betas, float *expression, float *camera, float *keypoints, float *jac, float *loss, float *lambda,
    int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_expression, float *trial_camera,
    const float *trial_keypoints, const float *trial_jac, void *stream);

/* shapy_fit_lm_keypoints_2d_expressive_step under the perspective camera of
 * shapy_fit_lm_keypoints_2d_perspective_step (intrinsics (B,3), translation t in the place of the camera, its depth
 * rule).  With ne = 0 and joint_weights null every output equals that step's bit for bit. */
int shapy_fit_lm_keypoints_2d_expressive_perspective_step(
    int batch, int num_keypoints, int n_rot, int nb, int ne, const float *targets, const float *weights,
    const float *intrinsics, const float *pose_anchor, const float *joint_weights, float robust_sigma,
    float pose_prior_weight, float betas_weight, float expression_weight, float lambda_up, float lambda_down, int first,
    float *rot, float *betas, float *expression, float *transl, float *keypoints, float *jac, float *loss,
    float *lambda, int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_expression,
    float *trial_transl, const float *trial_keypoints, const float *trial_jac, void *stream);

/* shapy_fit_lm_keypoints_2d_step over groups of images of one person: the images [group_offsets[g],
 * group_offsets[g+1]) of group g share one beta_g, each keeps its own rotations and camera.  Loss per group, fp64, left
 * to right: the sum over its images (image order) of the 2D step's keypoint term and pose prior, + betas_weight
 * |beta_g|^2.  group_offsets: num_groups + 1 int32 in host memory, non-decreasing from 0 to batch, every group
 * non-empty; copied into the workspace on the stream at every call.  Per image (batch rows): targets, weights,
 * pose_anchor, rot, camera, keypoints, jac, trial_rot, trial_camera, trial_keypoints, trial_jac and trial_betas_images
 * (batch,nb), the trial betas of each image's group (what shapy_smplx_keypoint_jacobian evaluated).  Per group
 * (num_groups rows): betas (G,nb), loss, lambda, accepted and trial_betas (G,nb).  Policy, lambda constants, damping
 * and rotation update are the 2D step's, per group: one decision, lambda, loss and accept count; the first lambda is
 * 1e-3 max(1e-6, the largest diagonal entry of the group's keypoint rows), per image on the pose and camera columns
 * and summed over the images on the betas columns.  The step is the exact LM step of the group's block-arrow normal
 * matrix by its Schur complement: each image's [pose | camera] block (damped by lambda) is eliminated, the nb x nb
 * system (damped by betas_weight + lambda) solved for dbeta, each image's delta back-substituted.  Three launches, no
 * synchronisation, no atomics: a group's results do not depend on the rest of the batch.  If the group's loss is not
 * finite or one of its factorisations fails, the group keeps its state.  The next trial goes to trial_betas and to
 * each image's row of trial_betas_images.  workspace: shapy_fit_lm_groups_workspace_bytes(batch, num_groups, n_rot, nb)
 * bytes of device memory.  Errors as shapy_fit_lm_keypoints_2d_step, and SHAPY_ERR_ARG for bad offsets or an empty
 * group.  batch 0 (with num_groups 0): no launch. */
size_t shapy_fit_lm_groups_workspace_bytes(int batch, int num_groups, int n_rot, int nb);
int shapy_fit_lm_keypoints_2d_groups_step(
    int batch, int num_groups, const int32_t *group_offsets, int num_keypoints, int n_rot, int nb,
    const float *targets, const float *weights, const float *pose_anchor, float robust_sigma, float pose_prior_weight,
    float betas_weight, float lambda_up, float lambda_down, int first, float *rot, float *betas, float *camera,
    float *keypoints, float *jac, float *loss, float *lambda, int32_t *accepted, float *trial_rot, float *trial_betas,
    float *trial_betas_images, float *trial_camera, const float *trial_keypoints, const float *trial_jac,
    void *workspace, void *stream);

/* shapy_fit_lm_keypoints_2d_groups_step with the five virtual measurements of each group (on the T-pose of beta_g):
 * the group loss gains sum_{u_m > 0} u_m (t_gm - meas_gm)^2 (m order, summed on its own) before the betas prior, and
 * J_m^T U J_m, J_m^T U (meas - t) (m order) join the betas system before betas_weight beta.  meas_targets,
 * meas_weights, meas, trial_meas (G,5), meas_jac, trial_meas_jac (G,5,nb): shapy_measure_jacobian_betas of the G
 * trial betas.  With every measurement weight <= 0 every output equals shapy_fit_lm_keypoints_2d_groups_step's bit for
 * bit.  Errors as that entry, the measurement pointers included. */
int shapy_fit_lm_keypoints_2d_groups_measurements_step(
    int batch, int num_groups, const int32_t *group_offsets, int num_keypoints, int n_rot, int nb,
    const float *targets, const float *weights, const float *pose_anchor, float robust_sigma, float pose_prior_weight,
    float betas_weight, const float *meas_targets, const float *meas_weights, float lambda_up, float lambda_down,
    int first, float *rot, float *betas, float *camera, float *keypoints, float *jac, float *meas, float *meas_jac,
    float *loss, float *lambda, int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_betas_images,
    float *trial_camera, const float *trial_keypoints, const float *trial_jac, const float *trial_meas,
    const float *trial_meas_jac, void *workspace, void *stream);

/* shapy_fit_lm_keypoints_2d_groups_step for views of one posed body at one moment: the images of group g share beta_g
 * and the body rotations R_g,j, j = 1 .. n_rot-1; each keeps its global rotation R_0,i and camera.  Loss per group,
 * fp64, left to right: the sum over its images (image order) of the 2D step's keypoint term, + pose_prior_weight / 2
 * sum_{j >= 1} |R_g,j - R0_g,j|_F^2 once per group, + betas_weight |beta_g|^2.  Arguments as
 * shapy_fit_lm_keypoints_2d_groups_step, except pose_anchor, which is per group, (G,n_rot,3,3), joint 0 unread.  rot
 * and trial_rot stay per image (batch,n_rot,3,3): the kernels read each group's body rotations from its first image's
 * rows and write the same values to all of its images' rows, so on the first step the caller fills every image's
 * rows of joints 1.. with the group's rotations.  The step is the exact LM step of the group's normal matrix by its
 * Schur complement: each image's [delta_0 | camera] block (damped by lambda) is eliminated, the (3 (n_rot-1) + nb)
 * square shared system (lambda on the rotation diagonal, betas_weight + lambda on the betas diagonal) solved, each
 * image's delta back-substituted.  The first lambda is 1e-3 max(1e-6, the largest diagonal entry of the group's
 * keypoint rows), per image on the [delta_0 | camera] columns and summed over the images on the shared columns.
 * A group of one has shapy_fit_lm_keypoints_2d_step's loss, lambda and decision bit for bit; with n_rot 1 every
 * output is shapy_fit_lm_keypoints_2d_groups_step's.  workspace: shapy_fit_lm_shared_pose_workspace_bytes(batch,
 * num_groups, n_rot, nb) bytes of device memory.  Three launches; errors as shapy_fit_lm_keypoints_2d_groups_step. */
size_t shapy_fit_lm_shared_pose_workspace_bytes(int batch, int num_groups, int n_rot, int nb);
int shapy_fit_lm_keypoints_2d_shared_pose_step(
    int batch, int num_groups, const int32_t *group_offsets, int num_keypoints, int n_rot, int nb,
    const float *targets, const float *weights, const float *pose_anchor, float robust_sigma, float pose_prior_weight,
    float betas_weight, float lambda_up, float lambda_down, int first, float *rot, float *betas, float *camera,
    float *keypoints, float *jac, float *loss, float *lambda, int32_t *accepted, float *trial_rot, float *trial_betas,
    float *trial_betas_images, float *trial_camera, const float *trial_keypoints, const float *trial_jac,
    void *workspace, void *stream);

/* shapy_fit_lm_keypoints_2d_shared_pose_step with the five virtual measurements of each group, as
 * shapy_fit_lm_keypoints_2d_groups_measurements_step adds them; their rows join the betas block of the shared system.
 * With every measurement weight <= 0 every output equals shapy_fit_lm_keypoints_2d_shared_pose_step's bit for bit. */
int shapy_fit_lm_keypoints_2d_shared_pose_measurements_step(
    int batch, int num_groups, const int32_t *group_offsets, int num_keypoints, int n_rot, int nb,
    const float *targets, const float *weights, const float *pose_anchor, float robust_sigma, float pose_prior_weight,
    float betas_weight, const float *meas_targets, const float *meas_weights, float lambda_up, float lambda_down,
    int first, float *rot, float *betas, float *camera, float *keypoints, float *jac, float *meas, float *meas_jac,
    float *loss, float *lambda, int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_betas_images,
    float *trial_camera, const float *trial_keypoints, const float *trial_jac, const float *trial_meas,
    const float *trial_meas_jac, void *workspace, void *stream);

/* One Levenberg-Marquardt step per body of the fit of bodies seen by a calibrated rig: num_bodies (G) bodies in one
 * world frame, body g seen by the views [view_offsets[g], view_offsets[g+1]) (num_bodies + 1 int32 in host memory,
 * rising strictly from 0 to num_views, copied into the workspace on the stream at every call).  Per view (num_views
 * rows): targets (B,K,2), weights (B,K), intrinsics (B,3) = (f, px, py) and extrinsics (B,12) = world-to-camera R
 * (row-major) then T, camera frame x right, y down, z forward.  Per body (G rows): pose_anchor, rot, betas, transl (the
 * world translation t), keypoints, jac (of shapy_smplx_keypoint_jacobian without transl), loss, lambda, accepted and
 * the trial.  Parameters [delta_j (3 n_rot) | beta (nb) | t], P = 3 n_rot + nb + 3.  With X_k = kp_k + t and Y_vk =
 * R_v X_k + T_v (fp64), p_vk = f_v (Y_x / Y_z, Y_y / Y_z) + (px_v, py_v); loss per body, fp64, left to right: the sum
 * over its views (view order) of sum_{w_vk > 0} w_vk rho(|p_vk - x_vk|^2) (k order), + pose_prior_weight / 2
 * sum_{j >= 1} |R_j - R0_j|_F^2 + betas_weight |beta|^2.  Keypoint rows 2k + c of each view in view order (IRLS
 * weights at the state): (f_v / Y_z) (R_v[c,:] - (Y_c / Y_z) R_v[2,:]) J3_k, J3_k the 3 x P block of keypoint k with
 * J_t = I.  Depth rule per view: a trial with a weighted keypoint at Y_z <= 0 or non-finite in any view, or a view
 * whose f is not finite and > 0, has loss +inf and is rejected; a start that breaks it reports NaN and does not move.
 * Pose-prior rows, first lambda (from the keypoint rows alone), damping and solve are the 2D step's, the next trial
 * R Exp(delta), beta + delta_beta, t + delta_t.  One launch, one CTA per body; no synchronisation, no atomics: a
 * body's results do not depend on the rest of the batch.  workspace: shapy_fit_lm_calibrated_workspace_bytes(
 * num_views, num_bodies) bytes of device memory.  Errors as shapy_fit_lm_keypoints_2d_perspective_step (over the G
 * bodies), and SHAPY_ERR_ARG for a null extrinsics or workspace, bad offsets or a body without a view.  num_bodies 0
 * (with num_views 0): no launch. */
size_t shapy_fit_lm_calibrated_workspace_bytes(int num_views, int num_bodies);
int shapy_fit_lm_keypoints_2d_calibrated_step(
    int num_views, int num_bodies, const int32_t *view_offsets, int num_keypoints, int n_rot, int nb,
    const float *targets, const float *weights, const float *intrinsics, const float *extrinsics,
    const float *pose_anchor, float robust_sigma, float pose_prior_weight, float betas_weight, float lambda_up,
    float lambda_down, int first, float *rot, float *betas, float *transl, float *keypoints, float *jac, float *loss,
    float *lambda, int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_transl,
    const float *trial_keypoints, const float *trial_jac, void *workspace, void *stream);

/* One Levenberg-Marquardt step of the perspective 2D fit over video sequences of one person filmed by one camera: the
 * frames [sequence_offsets[s], sequence_offsets[s+1]) of sequence s (num_sequences + 1 int32 in host memory, rising
 * strictly from 0 to batch, copied into the workspace on the stream at every call), in time order, share one beta_s;
 * each frame keeps its rotations and camera-frame translation tau_t and projects as
 * shapy_fit_lm_keypoints_2d_perspective_step does with its own intrinsics (batch,3).  Loss per sequence, fp64, left to
 * right: the sum over its frames (frame order) of [the perspective step's keypoint term and pose prior, +
 * smooth_rot_weight / 2 sum_{j >= 0} |R_{t+1},j - R_t,j|_F^2 + smooth_transl_weight |tau_{t+1} - tau_t|^2 when frame
 * t + 1 is in the sequence], + betas_weight |beta_s|^2.  Per frame (batch rows): targets, weights, intrinsics,
 * pose_anchor, rot, transl, keypoints, jac, trial_rot, trial_transl, trial_keypoints, trial_jac and trial_betas_images
 * (batch,nb), the trial betas of each frame's sequence.  Per sequence (num_sequences rows): betas, loss, lambda,
 * accepted and trial_betas.  Policy, lambda constants and rotation update are the grouped step's, per sequence; the
 * first lambda is 1e-3 max(1e-6, the largest diagonal entry of the sequence's keypoint rows), per frame on the
 * [rotation | translation] columns and summed over the frames on the betas columns.  The normal matrix of a sequence is
 * block tridiagonal in its frames with an arrow of betas columns; the step solves it exactly by a block LDL^T sweep along
 * the frames (each frame's block damped by lambda, the betas block by betas_weight + lambda).  Depth rule per frame, as
 * the perspective step's: a weighted keypoint at Y_z <= 0 or a bad focal length in any frame gives the trial a loss of
 * +inf.  If a sequence's loss is not finite or one of its pivots fails, it keeps its state.  Three launches, no
 * synchronisation, no atomics: a sequence's results do not depend on the rest of the batch.  A sequence of one frame has
 * the perspective step's loss, lambda and decision bit for bit.  workspace: shapy_fit_lm_sequence_workspace_bytes(batch,
 * num_sequences, n_rot, nb) bytes of device memory.  Errors as shapy_fit_lm_keypoints_2d_groups_step, with a null
 * intrinsics and smoothness weights < 0 or not finite refused.  batch 0 (with num_sequences 0): no launch. */
size_t shapy_fit_lm_sequence_workspace_bytes(int batch, int num_sequences, int n_rot, int nb);
int shapy_fit_lm_keypoints_2d_sequence_step(
    int batch, int num_sequences, const int32_t *sequence_offsets, int num_keypoints, int n_rot, int nb,
    const float *targets, const float *weights, const float *intrinsics, const float *pose_anchor, float robust_sigma,
    float pose_prior_weight, float betas_weight, float smooth_rot_weight, float smooth_transl_weight, float lambda_up,
    float lambda_down, int first, float *rot, float *betas, float *transl, float *keypoints, float *jac, float *loss,
    float *lambda, int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_betas_images,
    float *trial_transl, const float *trial_keypoints, const float *trial_jac, void *workspace, void *stream);

/* shapy_fit_lm_keypoints_2d_calibrated_step with the five virtual measurements of each body stacked under its rows, as
 * shapy_fit_lm_keypoints_2d_measurements_step adds them (meas_targets, meas_weights, meas, trial_meas (G,5), meas_jac,
 * trial_meas_jac (G,5,nb)).  With every measurement weight <= 0 every output equals
 * shapy_fit_lm_keypoints_2d_calibrated_step's bit for bit. */
int shapy_fit_lm_keypoints_2d_calibrated_measurements_step(
    int num_views, int num_bodies, const int32_t *view_offsets, int num_keypoints, int n_rot, int nb,
    const float *targets, const float *weights, const float *intrinsics, const float *extrinsics,
    const float *pose_anchor, float robust_sigma, float pose_prior_weight, float betas_weight,
    const float *meas_targets, const float *meas_weights, float lambda_up, float lambda_down, int first, float *rot,
    float *betas, float *transl, float *keypoints, float *jac, float *meas, float *meas_jac, float *loss, float *lambda,
    int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_transl, const float *trial_keypoints,
    const float *trial_jac, const float *trial_meas, const float *trial_meas_jac, void *workspace, void *stream);

/* Drop-in for mesh_mesh_intersect_cuda.mesh_to_mesh_forward: query (B,Q,3,3), target (B,F,3,3) fp32;
 * collision_faces (B,Q*M) int64 pre-filled by the callee with -1; collision_bcs (B,Q*M,2,3) with 0.
 * num_target > 32768 returns SHAPY_ERR_UNSUPPORTED. */
size_t shapy_mmi_workspace_bytes(int batch, int num_query, int num_target);
int shapy_mmi_forward(const float *query, const float *target, int batch, int num_query, int num_target,
                      int max_collisions, int64_t *collision_faces, float *collision_bcs, void *workspace,
                      size_t workspace_bytes, void *stream);

/* The same on float64 triangles, with the reference operator's double instantiation semantics: the SAT's CMP
 * tolerance and its projected intervals are rounded to float as op.cu does, everything else (AABBs, the inclusive
 * leaf test, the ray test, barycentrics) is computed in double.  collision_bcs is float64. */
size_t shapy_mmi_workspace_bytes_f64(int batch, int num_query, int num_target);
int shapy_mmi_forward_f64(const double *query, const double *target, int batch, int num_query, int num_target,
                          int max_collisions, int64_t *collision_faces, double *collision_bcs, void *workspace,
                          size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------ scans */
/* Exact closest point of every scan point on its own body's mesh: vertices (B,V,3), faces (F,3) int32 (indices < V,
 * shared by the batch), points (B,N,3), weights (B,N) or NULL (all kept).  For each kept point: face_idx (B,N) the
 * face of the closest point, bary (B,N,3) its barycentrics on that face, sq_dist (B,N) the squared distance, all
 * fp32.  The closest point on a face is the Voronoi-region test over its vertices, edges and interior; a zero-area face
 * is the nearest of its edges.  A point with weight <= 0 is never read (it may be NaN): face -1, zero barycentrics
 * and distance.
 * Deterministic and a function of the mesh and the points alone: the winner is the face with the smallest float
 * squared distance, the smallest face index on a tie, whatever the tree's shape, so a body's result does not depend
 * on the rest of the batch, and a tree refit from another pose gives the same bits as one built fresh.
 * The LBVH of shapy_mmi_forward is built over the posed triangles in the workspace (>=
 * shapy_closest_points_workspace_bytes(B, F)); refit != 0 keeps the tree a previous call built in the same workspace
 * for the same B and faces and only recomputes its boxes from the new vertices.
 * F > 32768 or N > 32768 returns SHAPY_ERR_UNSUPPORTED before any launch; B = 0 or N = 0 launches nothing. */
size_t shapy_closest_points_workspace_bytes(int batch, int num_faces);
int shapy_closest_points(const float *vertices, const int32_t *faces, int batch, int num_verts, int num_faces,
                         const float *points, int num_points, const float *weights, int refit, int32_t *face_idx,
                         float *bary, float *sq_dist, void *workspace, size_t workspace_bytes, void *stream);

/* Nearest kept scan point of every query (a model vertex): queries (B,Q,3), points (B,N,3), weights (B,N) or NULL;
 * idx (B,Q) int32, sq_dist (B,Q).  Points with weight <= 0 are excluded (never read); the winner is the smallest
 * float squared distance, the smallest point index on a tie; idx -1 and distance 0 when a body keeps no point.  The
 * tree is the same LBVH over the points as degenerate triangles, workspace >= shapy_nearest_points_workspace_bytes.
 * N must be >= 1; N > 32768 returns SHAPY_ERR_UNSUPPORTED; B = 0 or Q = 0 launches nothing. */
size_t shapy_nearest_points_workspace_bytes(int batch, int num_points);
int shapy_nearest_points(const float *queries, int batch, int num_queries, const float *points, int num_points,
                         const float *weights, int32_t *idx, float *sq_dist, void *workspace, size_t workspace_bytes,
                         void *stream);

/* One Levenberg-Marquardt step per body of the fit of pose, shape and translation to 3D scans, with the policy,
 * lambda constants, Cholesky and rotation update of shapy_fit_lm_keypoints_step.  Parameters [delta_j (3 n_rot) | beta
 * (nb) | t], the columns of shapy_smplx_vertex_jacobian, P = 3 n_rot + nb + 3 <= 96 (SHAPY_ERR_UNSUPPORTED past that).
 * Inputs: points (B,N,3) and weights (B,N) (a point with weight <= 0 is dropped and never read: it may be NaN), faces
 * (F,3); the trial's vertices (B,V,3) and jac (B,V,3,P) of shapy_smplx_vertex_jacobian (with transl), its closest
 * points trial_face_idx / trial_bary (B,N) / (B,N,3) of shapy_closest_points, and trial_nearest (B,V) of
 * shapy_nearest_points (NULL when model_to_scan_weight is 0).  Loss per body, fp64, left to right:
 *   s2m / W sum_{w_i > 0} w_i rho(d_i^2) + m2s / V sum_v rho(e_v^2) + pose_w / 2 sum_{j >= 1} |R_j - anchor_j|_F^2
 *   + the measurement terms of shapy_fit_lm_keypoints_2d_measurements_step + betas_w |beta|^2,
 * W = sum_{w_i > 0} w_i (1 when 0), d_i = |c_i - p_i|, c_i = sum_k bary_ik x_{f_i,k} the trial's closest point, e_v =
 * |x_v - p_{nearest_v}| (a vertex without a nearest point adds nothing), rho the Geman-McClure e s^2 / (s^2 + e) at
 * robust_sigma s, the identity at s = inf.  Rows at the held correspondences, each with the IRLS weight rho'(.) (times
 * w_i s2m / W or m2s / V): a point whose barycentrics are all > 0 on a face of non-zero area gives one point-to-plane
 * row n^T (c_i - p_i), n the face's unit normal held constant; any other kept point three point-to-point rows
 * c_i - p_i; a vertex three rows x_v - p_{nearest_v}; then the chordal pose-prior rows, the measurement rows and
 * betas_w.  Two launches: the rows in fp64 by chunks of 1024 points or vertices per CTA into workspace (>=
 * shapy_fit_lm_scan_workspace_bytes(B, N, V, P)), then one CTA per body sums the chunks in chunk order.  The state:
 * rot (B,n_rot,3,3), betas (B,nb), transl (B,3), normal_matrix (B,P,P) and gradient (B,P) fp64, the undamped data
 * rows J^T W J and J^T W r at the state, loss, lambda, accepted; with measurements (meas_targets, meas_weights, meas,
 * meas_jac, trial_meas, trial_meas_jac all non-NULL, as in shapy_fit_lm_keypoints_2d_measurements_step; all NULL
 * without) meas (B,5) and meas_jac (B,5,nb).  On accept the trial's parameters, data rows and measurements become the
 * state.  The first lambda reads the data rows' diagonal.  A body whose loss is not finite, or whose factorisation
 * fails, gets its state as the trial.  With every measurement weight <= 0 the outputs equal the step without
 * measurements bit for bit.  Deterministic, no atomics, a body's result independent of the rest of the batch.  A null
 * pointer, a bad size, robust_sigma <= 0 or NaN, a negative or non-finite term weight, a negative prior weight, a
 * lambda factor < 1 or a small workspace: SHAPY_ERR_ARG.  batch 0: no launch. */
size_t shapy_fit_lm_scan_workspace_bytes(int batch, int num_points, int num_verts, int num_params);
int shapy_fit_lm_scan_step(int batch, int num_points, int num_verts, int n_rot, int nb, const float *points,
                           const float *weights, const int32_t *faces, const float *pose_anchor, float robust_sigma,
                           float scan_to_model_weight, float model_to_scan_weight, float pose_prior_weight,
                           float betas_weight, const float *meas_targets, const float *meas_weights, float lambda_up,
                           float lambda_down, int first, float *rot, float *betas, float *transl,
                           double *normal_matrix, double *gradient, float *meas, float *meas_jac, float *loss,
                           float *lambda, int32_t *accepted, float *trial_rot, float *trial_betas, float *trial_transl,
                           const float *trial_vertices, const float *trial_jac, const int32_t *trial_face_idx,
                           const float *trial_bary, const int32_t *trial_nearest, const float *trial_meas,
                           const float *trial_meas_jac, void *workspace, size_t workspace_bytes, void *stream);

/* Backward of sq_dist of shapy_closest_points with respect to the vertices, face_idx and bary held at the forward's
 * values: grad_vertices (B,V,3) = sum over the points of 2 g_i (q_i - p_i) bary_{i,c} at corner c of face_idx_i, q_i =
 * sum_c bary_{i,c} x_c recomputed from `vertices`.  inc_ptr (V+1) / inc (3F) is the vertex -> (3 face + corner)
 * incidence CSR of `faces` (shapy_b200.ops.face_incidence).  A point whose face is outside [0, F) adds nothing.  One
 * CTA per body sorts its (face, point) pairs in shared memory; each vertex sums over its incident faces in CSR order
 * and each face's points in index order: no atomics, bit-identical run to run and alone or in a batch.  No gradient
 * with respect to the points.  F > 32768 or N > 32768 returns SHAPY_ERR_UNSUPPORTED; N = 0 zeroes grad_vertices. */
int shapy_closest_points_backward(const float *vertices, const int32_t *faces, const int32_t *inc_ptr,
                                  const int32_t *inc, int batch, int num_verts, int num_faces, const float *points,
                                  int num_points, const int32_t *face_idx, const float *bary,
                                  const float *grad_sq_dist, float *grad_vertices, void *stream);

/* ------------------------------------------------------------ regression head */
/* params_out (num_stages, B, P).  W0 (H0, F+P), W1 (H1, H0), W2 (P, H1) row-major as nn.Linear stores
 * them; mean (P).  workspace >= shapy_head_workspace_bytes. */
size_t shapy_head_workspace_bytes(int batch, int feat_dim, int param_dim, int h0, int h1);
int shapy_head_forward(const float *feats, int batch, int feat_dim, int param_dim, int h0, int h1,
                       const float *W0, const float *b0, const float *W1, const float *b1, const float *W2,
                       const float *b2, const float *mean, int num_stages, float *params_out, void *workspace,
                       size_t workspace_bytes, void *stream);

/* The MLP has no activation, so a stage collapses exactly (in real arithmetic) to p' = p + Mf f + Mp p + c.
 * MfT (F, P) = (W2 W1 W0[:, :F])^T, MpT (P, P) = (W2 W1 W0[:, F:])^T, c (P) = W2 (W1 b0 + b1) + b2, contracted by
 * the caller in fp64.  workspace >= B * P * 4 bytes. */
int shapy_head_forward_collapsed(const float *feats, int batch, int feat_dim, int param_dim, const float *MfT,
                                 const float *MpT, const float *c, const float *mean, int num_stages,
                                 float *params_out, void *workspace, size_t workspace_bytes, void *stream);

/* -------------------------------------------------------------------- HRNet */
typedef struct shapy_hrnet shapy_hrnet_t;

/* One convolution of the backbone, BN already folded by the caller's choice: the library folds
 * scale into the weights itself when `bn_*` are given.  HOST pointers. */
typedef struct {
  int cin, cout, ksize, stride; /* ksize 1 or 3, stride 1 or 2, padding ksize/2 */
  const float *weight;          /* (cout, cin, k, k) */
  const float *bias;            /* (cout) or NULL */
  const float *bn_weight, *bn_bias, *bn_mean, *bn_var; /* (cout) each or all NULL */
  float bn_eps;
} shapy_conv_desc_t;

enum { SHAPY_OP_STEM = 0, SHAPY_OP_CONV = 1, SHAPY_OP_FUSE = 2, SHAPY_OP_POOL = 3 };

/* Program of the network: a flat list of ops over numbered activation slots.  A slot is a
 * (B, H/div, W/div, C) NHWC tensor; outputs may write a channel slice of a wider slot
 * (out_coff / slot channels) which is how the 4x384 concat is formed without a copy. */
typedef struct {
  int kind;          /* SHAPY_OP_* */
  int conv;          /* index into the conv table (STEM / CONV) */
  int in_slot;       /* -1 = network input (STEM) */
  int out_slot, out_coff;
  int res_slot;      /* residual added before ReLU, -1 none */
  int relu;
  /* FUSE: out = relu(sum_i up(in_i)); in_i at scale 2^shift_i coarser than out (nearest) */
  int n_in;
  int fuse_in[4];
  int fuse_shift[4];
  /* Execution lane (0..SHAPY_MAX_LANES-1).  Ops of one lane run in program order on one CUDA stream; ops of
   * different lanes may run concurrently (the independent branches of a HighResolutionModule, reference
   * hrnet.py:175-193).  The executor derives every cross-lane ordering itself from the slots an op reads and
   * writes (RAW, WAR and WAW), so the lane is a scheduling hint only: any assignment gives the serial result. */
  int lane;
} shapy_op_t;
enum { SHAPY_MAX_LANES = 4 };

typedef struct {
  int channels;      /* total channels of the slot */
  int div;           /* spatial divisor w.r.t. the network input (4, 8, 16, 32, 2) */
} shapy_slot_t;

/* mode: 0 = fp16 operands, single pass (BASELINE config 2);
 *       1 = split-fp16 (hi + lo planes, 3 MMAs per tile, ~fp32 accuracy; parity mode);
 * engine: 0 = wgmma implicit GEMM where the shape allows, 1 = SIMT fp32 everywhere (debug). */
int shapy_hrnet_create(shapy_hrnet_t **out, const shapy_conv_desc_t *convs, int n_convs, const shapy_op_t *ops,
                       int n_ops, const shapy_slot_t *slots, int n_slots, int feat_slot, int mode, int engine);
void shapy_hrnet_destroy(shapy_hrnet_t *p);
size_t shapy_hrnet_workspace_bytes(const shapy_hrnet_t *p, int batch, int height, int width);
/* images (B,3,H,W) fp32 NCHW device; feats (B, C_feat) fp32 device. */
int shapy_hrnet_forward(shapy_hrnet_t *p, const float *images, int batch, int height, int width, float *feats,
                        void *workspace, size_t workspace_bytes, void *stream);
/* copies slot `slot` (after a forward) to dst as fp32 NCHW (B,C,H/div,W/div); for tests. */
int shapy_hrnet_read_slot(shapy_hrnet_t *p, int slot, float *dst, void *stream);
double shapy_hrnet_flops(const shapy_hrnet_t *p, int batch, int height, int width);

/* Standalone conv for unit tests of the implicit-GEMM kernel: x (B,H,W,Cin) fp32 NHWC device,
 * y (B,Ho,Wo,Cout) fp32 NHWC device, res optional (same shape as y).  engine: 0 = wgmma with the path the network
 * would take, 1 = SIMT, 2 = wgmma per-tap path, 3 = wgmma halo-resident path (error where it does not apply).
 * Views (0 = dense): in_ctot > 0 gives x in_ctot channels per pixel, of which the conv reads in_coff .. in_coff + cin;
 * out_ctot > 0 writes the conv into channels out_coff .. out_coff + cout of (batch + 1, Ho, Wo, out_ctot) planes
 * filled with NaN beforehand, and y returns all of them (batch + 1, Ho, Wo, out_ctot).  plan (optional, int[3]):
 * the plan built, as the engine digits that force it: path (2, 3 or 4), schedule (1 cooperative, 2 ping-pong), cout
 * tile; -1 each for the SIMT engine. */
int shapy_conv_test(const shapy_conv_desc_t *conv, const float *x, const float *res, int batch, int height,
                    int width, int relu, int mode, int engine, int in_ctot, int in_coff, int out_ctot, int out_coff,
                    int *plan, float *y, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Input stage (SURVEY.md 8f rank 1): uint8 full images + crop windows -> normalised fp32 NCHW crops.
 * Replaces, per detected person, the reference's CPU chain
 *   read_img        regressor/human_shape/utils/img_utils.py:57-61         (uint8 -> float32 / 255, clip)
 *   crop            regressor/human_shape/utils/transf_utils.py:51-96      (window [ul, br), zero padding,
 *                                                                           cv2.resize INTER_LINEAR to size x size)
 *   ToTensor + Normalize  regressor/human_shape/data/transforms/transforms.py:710-733  (clamp [0,1], (x - mean) / std)
 * The window corners are computed by the host exactly as transf_utils.py:41-56 does (float32 matrix inverse and
 * integer truncation; shapy_b200/preprocess.py mirrors it) and passed in the descriptor.
 *   images : device, all uint8 HxWx3 (RGB, row-major) images of the batch back to back
 *   descs  : device, one per output crop (several crops may name the same image)
 *   mean, stdv : host, 3 floats each
 *   out    : device (B, 3, size, size) fp32 */
typedef struct shapy_image_desc_t {
  long long offset;        /* byte offset of the image inside `images` */
  int height, width;       /* image extent */
  int ul_x, ul_y;          /* window upper-left corner (inclusive), may be negative */
  int br_x, br_y;          /* window bottom-right corner (exclusive), may exceed the image */
} shapy_image_desc_t;
int shapy_preprocess_forward(const unsigned char *images, const shapy_image_desc_t *descs, int batch, int size,
                             const float *mean, const float *stdv, float *out, void *stream);

/* ------------------------------------------------------------------------------------------------
 * B2A attribute head (SURVEY.md 8f rank 2): betas -> attribute ratings with the male / female regressors.
 * Replaces regressor/human_shape/models/common/iterative_regressor.py:761-776 and
 * attributes/attributes/attributes_betas/polynomial.py:61-69,137-140 (degree-2 polynomial features + Linear).
 *   betas  : device (B, num_betas) fp32        gender : device (B) int32, 0 = male, 1 = female, other = row of zeros
 *   w_*    : device (num_outputs, num_betas + num_betas (num_betas + 1) / 2) fp32 row-major (Linear.weight)
 *   b_*    : device (num_outputs) fp32         out    : device (B, num_outputs) fp32 */
int shapy_b2a_forward(const float *betas, const int *gender, const float *w_male, const float *b_male,
                      const float *w_female, const float *b_female, int batch, int num_betas, int num_outputs, float *out,
                      void *stream);

/* A2B head (SURVEY.md 8f rank 2): attribute ratings (+ height / weight) -> betas, per gender.  Replaces
 * regressor/human_shape/models/common/iterative_regressor.py:837-850 around A2B.forward
 * (attributes/attributes/attributes_betas/a2b.py:278-279) for the `polynomial` (degree 2) and `linear` networks.
 *   feat_male / feat_female : device (B, num_features) fp32 -- the reference builds one feature vector per gender
 *                             (its default height / weight differ, iterative_regressor.py:793-836)
 *   gender : device (B) int32, 0 = male, 1 = female, other = row of zeros
 *   w_*    : device (num_betas, F) fp32 row-major, F = num_features (linear != 0) or num_features + num_features
 *            (num_features + 1) / 2 (degree-2 polynomial);  b_* : device (num_betas);  out : device (B, num_betas) */
int shapy_a2b_forward(const float *feat_male, const float *feat_female, const int *gender, const float *w_male,
                      const float *b_male, const float *w_female, const float *b_female, int batch, int num_features,
                      int num_betas, int linear, float *out, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Evaluation metric (SURVEY.md 8f rank 3): translation-aligned point-to-point error through sparse point regressors
 * ("P2P-20k", also plain v2v with identity regressors).  Replaces regressor/human_shape/utils/metrics.py:368-456
 * (v2vhdError.__call__) and regressor/hbw_evaluation/evaluate_hbw.py:44-58,147-151.
 *   in_* / tg_* : device CSR (row_ptr int32 [P+1], col int32 [nnz], val fp32 [nnz]) of the P x V1 / P x V2 regressors
 *   input_vertices (B, V1, 3), target_vertices (B, V2, 3) : device fp32
 *   align : 1 = translate by mean(target points) - mean(input points) (metrics.py:431-439)
 *   error (B, P), mean_error (B) : device fp32      workspace : >= shapy_p2p_workspace_bytes(B, P) */
size_t shapy_p2p_workspace_bytes(int batch, int num_points);
int shapy_p2p_error(const int *in_row_ptr, const int *in_col, const float *in_val, const int *tg_row_ptr, const int *tg_col,
                    const float *tg_val, const float *input_vertices, const float *target_vertices, int batch, int num_points,
                    int num_input_vertices, int num_target_vertices, int align, float *error, float *mean_error, void *workspace,
                    size_t workspace_bytes, void *stream);

/* Vertex-to-vertex error between meshes of the SAME topology, translation aligned or not: PointError with
 * TranslationAlignment / NoAlignment, regressor/human_shape/utils/metrics.py:232-277, 335-366 (evaluation.py:192-224
 * `v2v_t` / `v2v`): est' = est + (mean(gt) - mean(est)); error[b][v] = |est'[b][v] - gt[b][v]|.
 * input / target: device (B, V, 3) fp32; error (B, V), mean_error (B); workspace >= shapy_p2p_workspace_bytes(B, V). */
int shapy_v2v_error(const float *input_vertices, const float *target_vertices, int batch, int num_verts, int align,
                    float *error, float *mean_error, void *workspace, size_t workspace_bytes, void *stream);

/* Point error between point sets of the same topology after a scale or root alignment: PointError with ScaleAlignment /
 * RootAlignment, regressor/human_shape/utils/metrics.py:173-229, 279-303, 335-366 (evaluation.py:595-620: the
 * scale-corrected `v2v_t` and the root-aligned `mpjpe` / `mpjpe14`).  Per body b:
 *   SHAPY_ALIGN_SCALE  s = sqrt(var2 / var1) from the centred sums of squares of est / gt about their means mu1 / mu2;
 *                      error[b][p] = |s est + (mu2 - s mu1) - gt|.  var1 == 0 is not guarded (inf / NaN, as in fp32).
 *   SHAPY_ALIGN_ROOT   r_est, r_gt = means of the points listed in `roots` (numpy indexing: -P <= index < P);
 *                      error[b][p] = |(est - r_est) - (gt - r_gt)|.  An empty list gives NaN, numpy's mean of an empty axis.
 * input_points / target_points : device (B, P, 3) fp32, points first;  roots : HOST int array of num_roots <=
 * SHAPY_MAX_ROOTS entries, checked in the call and passed to the kernel by value (ignored in scale mode);
 * error (B, P), mean_error (B) : device fp32;  workspace >= shapy_point_error_workspace_bytes(B) (per-body statistics).
 * Every reduction has a fixed order: the result of a body is bit-identical run to run and whatever else is in the batch. */
enum { SHAPY_ALIGN_SCALE = 1, SHAPY_ALIGN_ROOT = 2 };
#define SHAPY_MAX_ROOTS 16
size_t shapy_point_error_workspace_bytes(int batch);
int shapy_point_error_aligned(const float *input_points, const float *target_points, int batch, int num_points, int mode,
                              const int *roots, int num_roots, float *error, float *mean_error, void *workspace,
                              size_t workspace_bytes, void *stream);

/* Sparse point regression: points (B, P, 3) = (P x V regressor) times vertices (B, V, 3), per body; the J14 joints of
 * `mpjpe14` (evaluation.py:161-190, np.einsum('jv,bvn->bjn', J14_regressor, vertices)).  row_ptr int32 [P+1], col
 * int32 [nnz] (< V), val fp32 [nnz]: device CSR;  vertices, points : device fp32. */
int shapy_regress_points(const int *row_ptr, const int *col, const float *val, const float *vertices, int batch,
                         int num_points, int num_verts, float *points, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* SHAPY_B200_H_ */
