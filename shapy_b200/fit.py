"""Batched fitting of SMPL-X bodies on the device: betas to virtual measurements, and pose and shape to 3D keypoints.

    from shapy_b200.fit import fit_betas_to_measurements, fit_body_to_keypoints
    res = fit_betas_to_measurements(body_model, body_measurements, {'height': h, 'mass': m, ...})   # (B,) targets
    res = fit_body_to_keypoints(body_model, keypoints)                                             # (B, K, 3)

    python -m shapy_b200.fit --synthetic --height 1.80 --mass 80 --output fit.npz
    python -m shapy_b200.fit --model-folder models/smplx --targets targets.npz --output fit.npz

The loss is the one of the reference's mesh-mesh-intersection/examples/fit_measurements.py:111-133, per body:
sum_k w_k (target_k - measured_k)^2 + betas_weight |betas|^2, default weights height 100, mass 1, chest 2000,
waist 1000, hips 1000; a target <= 0 or a weight <= 1e-3 drops that term (per body for the targets).  The bodies go
through SMPLX.forward_shape -> BodyMeasurements.forward_vertices, both differentiable (shapy_b200.autograd), and the
whole batch is optimised at once with Adam: Adam is elementwise, so every body's trajectory is independent of the
rest of the batch (the reference's L-BFGS / TrustRegion would couple them through the line search and needs a double
backward, which is not supported).

method='lm' fits the same loss with a batched Levenberg-Marquardt loop instead: per iteration, forward_shape of the
trial betas, then the measurements and their (5, NB) Jacobian with respect to betas in one launch
(ops.measure_jacobian_betas), then one damped Gauss-Newton step per body (ops.fit_lm_step: accept the trial if its
loss is lower, adapt the damping, solve the NB x NB normal equations in fp64).  Three launches per iteration, no host
synchronisation, and every body's loss is non-increasing.  measurement_jacobian(body_model, body_measurements, betas)
exposes the Jacobian itself.

fit_body_to_keypoints optimises the raw 6D global and body pose (through the 6D decoder), betas and transl of every
body against its K 3D keypoints (the model's joints output: posed joints, landmarks, J14 overwrite), loss per body
sum_k w_k |joint_k - keypoint_k|^2, with the same batched Adam: SMPLX.forward and the decoder are differentiable
(shapy_b200.autograd), and a body's gradient does not depend on the rest of the batch.

fit_body_to_keypoints(..., method='lm') fits the same loss (a keypoint with weight <= 0 dropped) with a batched
Levenberg-Marquardt loop: the raw 6D start is decoded once, and each iteration evaluates the trial's keypoints and
their (3K, P) Jacobian with respect to right-multiplied rotation tangents, betas and transl in one launch
(ops.smplx_keypoint_jacobian), then takes one damped Gauss-Newton step per body (ops.fit_lm_keypoints_step: the
measurement LM's policy, the P x P normal equations in fp64, the next rotations R Exp(delta) re-orthonormalised).  Two
launches per iteration, no host synchronisation, and one SMPLX.forward at the end gives the returned keypoints and
loss.  keypoint_jacobian(body_model, rot, betas, transl) exposes the Jacobian itself.  The step takes at most 96
parameters, so a model with more than 27 betas raises ValueError before any launch.

fit_body_to_keypoints(..., body_measurements=bm, measurements={'height': h, 'mass': m, ...}) fits the keypoints and
known measurements of the same bodies together, loss per body: the keypoint loss + the measurement loss of
fit_betas_to_measurements on the T-pose of the fitted betas (same targets, weights and dropping rule) +
betas_weight |betas|^2.  Keypoints pin down the bone lengths, the measurements the soft tissue behind the
circumferences and the mass; fitting one after the other lets the second fit undo the first.  With Adam the
measurement term goes through forward_shape and BodyMeasurements.forward_vertices; with method='lm' each iteration
stacks the five measurement rows under the keypoint rows of one damped Gauss-Newton step (four launches: the keypoint
Jacobian, forward_shape and the measurement Jacobian of the trial, then ops.fit_lm_keypoints_measurements_step), no
host synchronisation, and every body's total loss is non-increasing.

circumference_derivative (every measurement fit, Adam and LM, and measurement_jacobian; python -m shapy_b200.fit
--circumference-derivative): how the chest, waist and hip circumferences are differentiated.  'reference' (the
default) keeps the reference's autograd semantics: the hull points' barycentrics are constants and the slicing planes'
heights get no gradient, so those rows are not the derivative of the measured circumference, and with the
circumferences at their default weights LM stalls.  'exact' uses the exact derivative (the hull points move with their
faces and with the planes, which follow their landmarks; include/shapy_b200.h, shapy_measure_backward_exact).  The
launches are the same in number, and LM still never synchronises with the host.

fit_body_to_keypoints_2d refines a prediction against 2D keypoints (B, K, 2) in the crop frame of the regressor's
proj_joints = softplus(c0) (joints_xy + c[1:3]): pose, betas and the weak-perspective camera, with an optional
Geman-McClure robust loss (robust_sigma), a chordal prior keeping the body pose near its start (pose_prior_weight) and
a betas prior.  With method='lm' each iteration is the keypoint Jacobian of the trial and one
ops.fit_lm_keypoints_2d_step (the 3D step's policy, the projected rows with IRLS weights, the prior rows), two
launches, no host synchronisation, every body's loss non-increasing; keypoint_jacobian_2d exposes the projected
Jacobian.

fit_body_to_keypoints_2d(..., body_measurements=bm, measurements={'height': h, 'mass': m, ...}) adds the measurement
loss of fit_body_to_keypoints (same targets, weights and dropping rule, T-pose of the fitted betas) to the 2D loss.
Under the weak-perspective camera a larger body seen by a smaller scale projects to the same points, so 2D keypoints
fix a body's proportions and not its metric size: a known height removes that freedom, a known mass pins the soft
tissue no joint sees.  With method='lm' each iteration is four launches (the keypoint Jacobian, forward_shape and the
measurement Jacobian of the trial, then ops.fit_lm_keypoints_2d_measurements_step), none synchronising.

fit_body_to_keypoints_2d(..., groups=labels) fits several images of one person with one shape: images with the same
label 0 .. G-1 share their betas, each keeps its pose and camera, and the loss of a group is the sum of its images'
2D losses + its measurement terms + betas_weight |betas|^2.  A bone foreshortened in one view is seen at full length in
another, and every view must agree on the same proportions.  With method='lm' each iteration is the keypoint Jacobian
of every image and ops.fit_lm_keypoints_2d_groups_step, whose three launches eliminate each image's pose and camera
block (a Schur complement) and solve for the group's betas (six launches with measurements), no host synchronisation,
every group's loss non-increasing.

fit_body_to_keypoints_2d(..., groups=labels, share_pose=True) fits simultaneous views of one posed body: the images of a
group share the betas and the body pose (joints 1 .., each relative to its parent, so the same in every view), each
keeps its global rotation and camera.  A weak-perspective view cannot see depth; a limb that one view sees
foreshortened another sees side-on.  With method='lm' each iteration is the keypoint Jacobian of every image and
ops.fit_lm_keypoints_2d_shared_pose_step, the grouped step with [global rotation | camera] eliminated per image and
[body pose | betas] solved per group.

fit_body_to_keypoints_2d(..., focal_length=f, principal_point=pp) fits under a perspective camera with known
intrinsics instead: the keypoints in the intrinsics' units (usually pixels), the last three parameters the body's
translation t in the camera frame (x right, y down, z forward), p_k = f (Y_x / Y_z, Y_y / Y_z) + pp with Y_k =
joint_k + t (PerspectiveCamera).  A weak-perspective camera cannot see depth; a pinhole camera sees a limb nearer the
camera larger, and with a known height a known focal length fixes the body's distance.  With method='lm' each
iteration is the keypoint Jacobian and ops.fit_lm_keypoints_2d_perspective_step (four launches with measurements), no
host synchronisation.  A trial with a weighted keypoint at Y_z <= 0 is rejected, and a body whose start has one
reports an infinite loss.  perspective_start converts the regressor's crop camera into a starting translation.

fit_body_to_calibrated_views fits bodies seen by a synchronised rig of calibrated cameras: each view has known
intrinsics and world-to-camera extrinsics (R_v, T_v), each body one pose, shape and world translation t, and every view
is a fixed projection of the same 3D keypoints, p_vk = f_v (Y_x / Y_z, Y_y / Y_z) + pp_v with Y_vk = R_v (joint_k + t) +
T_v.  The metric baseline between the cameras fixes the body's size and position, which no single view does.  With
method='lm' each iteration is the keypoint Jacobian of the bodies (one per body, whatever the number of views) and
ops.fit_lm_keypoints_2d_calibrated_step, two launches (four with measurements), no host synchronisation.
calibrated_start maps a camera-frame start of one view (a perspective fit, or perspective_start) into the world frame.

fit_body_to_sequence fits videos of one person filmed by one camera with known intrinsics: per frame the pose and the
camera-frame translation, per sequence one betas, and smoothness terms tying each frame to the next, so the pose and
translation do not jitter from frame to frame.  With method='lm' each iteration is the keypoint Jacobian of every frame
and ops.fit_lm_keypoints_2d_sequence_step, whose three launches solve each sequence's block-tridiagonal normal matrix
exactly by a block LDL^T sweep along its frames, no host synchronisation.

    python -m shapy_b200.fit --synthetic --keypoints-2d kp.npz --init pred.npz --method lm --robust-sigma 0.05
    python -m shapy_b200.fit --synthetic --keypoints-2d kp.npz --init pred.npz --method lm --targets known.npz

With --keypoints-2d, known measurements are read from --targets only (per-body arrays height / mass / ...); --height
and the other single-target flags are not used there, so a command line without --targets fits the keypoints alone.
With a `focal_length` (scalar or (B,)) in kp.npz, and `principal_point` ((2,) or (B, 2), by default the centre of
`image_size` (W, H)), the fit is perspective: raw `openpose` detections are mapped onto the model's keypoints in
pixels (no crop frame), an --init `camera` is converted by perspective_start with kp.npz's `center` / `scale`, and the
output holds `transl`.  An optional `groups` array (B,) in kp.npz fits the images of one label with one shape; the --targets arrays are then
per group, and the output carries `groups`.  With --share-pose the images of one label are simultaneous views of one
posed body: they share the body pose too, and body_pose is then per group in the output.

shapy_b200.keypoints2d reads OpenPose detections and maps them into that frame; with raw detections and their crop
descriptors in kp.npz, --keypoint-map openpose_smplx_map.json does the same on the command line.
"""
import argparse
import json

import numpy as np
import torch

from .body_measurements import CIRCUMFERENCE_DERIVATIVES, exact_circumferences

NAMES = ('mass', 'height', 'chest', 'waist', 'hips')
DEFAULT_WEIGHTS = {'height': 100.0, 'mass': 1.0, 'chest': 2000.0, 'waist': 1000.0, 'hips': 1000.0}


def _targets(targets, B, device):
    out = {}
    for k in NAMES:
        v = targets.get(k, -1.0)
        if isinstance(v, (int, float)):            # filled on the device: no host-to-device copy
            t = torch.full((B,), float(v), dtype=torch.float32, device=device)
        else:
            t = torch.as_tensor(v, dtype=torch.float32, device=device).reshape(-1)
        out[k] = t.expand(B).contiguous() if t.numel() == 1 else t
        if out[k].numel() != B:
            raise ValueError(f'target `{k}` has {out[k].numel()} values for {B} bodies')
    return out


def _measurement_terms(targets, weights, B, device):
    """(targets (B, 5), weights (B, 5)) in NAMES order: the weight is 0 where the target is <= 0 or the weight is
    <= 1e-3 (fit_measurements.py:111-133), and such a target is clamped to 0."""
    tg = _targets(targets, B, device)
    w = dict(DEFAULT_WEIGHTS, **(weights or {}))
    wt = torch.stack([torch.where(tg[k] > 0, torch.full_like(tg[k], w[k]), torch.zeros_like(tg[k]))
                      if w[k] > 1e-3 else torch.zeros_like(tg[k]) for k in NAMES], 1)
    tgt = torch.stack([tg[k].clamp(min=0) for k in NAMES], 1)
    return tgt, wt


def _measurement_loss(tgt, wt, meas, betas, betas_weight):
    """sum_k w_k (t_k - m_k)^2 + betas_weight |betas|^2 per body; a dropped term passes no (NaN) value or gradient."""
    diff = torch.where(wt > 0, tgt - meas, torch.zeros_like(meas))
    return (wt * diff.pow(2)).sum(1) + betas_weight * betas.pow(2).sum(1)


class _MeasurementTerm:
    """The measurement term of a fit over n bodies or groups: targets and weights (n, 5) (_measurement_terms), measured
    by body_measurements on the T-pose of the fitted betas, the circumferences differentiated as
    circumference_derivative says."""

    def __init__(self, tgt, wt, body_measurements, circumference_derivative):
        self.tgt, self.wt = tgt.contiguous(), wt.contiguous()
        self.bm, self.cd = body_measurements, circumference_derivative
        self.exact = exact_circumferences(circumference_derivative)

    def measure(self, body_model, betas):
        """The measurements (n, 5) of betas through forward_shape and BodyMeasurements.forward_vertices (Adam)."""
        v = body_model.forward_shape(betas=betas)['v_shaped']
        m = self.bm.forward_vertices(v, body_model.faces_i32, self.cd)['measurements']
        return torch.stack([m[k]['tensor'] for k in NAMES], 1)

    def loss(self, meas, betas, rho):
        return _measurement_loss(self.tgt, self.wt, meas, betas, rho)

    def prime(self, body_model):
        """Builds the faces' incidence table (one copy to the host) and the landmarks before an LM loop, which never
        synchronises."""
        from . import ops
        ops.face_incidence(body_model.faces_i32)
        self.bm.landmarks()

    def trial(self, packed, body_model, betas):
        """(trial_meas (n, 5), trial_meas_jac (n, 5, NB)) of the trial betas of an LM step: forward_shape and the
        measurement Jacobian, two launches."""
        from . import ops
        v = ops.smplx_forward_shape(packed, betas)
        meas, jac, _ = ops.measure_jacobian_betas(packed, self.bm.landmarks(), v, body_model.faces_i32,
                                                  exact=self.exact)
        return meas, jac

    def state(self, nb, device):
        """The entries an LM step's state gains with measurements: 'meas' (n, 5) and 'meas_jac' (n, 5, NB)."""
        n = self.tgt.shape[0]
        return {'meas': torch.empty(n, 5, dtype=torch.float32, device=device),
                'meas_jac': torch.empty(n, 5, nb, dtype=torch.float32, device=device)}


def _measurement_term(measurements, measurement_weights, n, device, body_measurements, circumference_derivative):
    """The _MeasurementTerm of n bodies or groups, or None without measurements."""
    if measurements is None:
        return None
    tgt, wt = _measurement_terms(measurements, measurement_weights, n, device)
    return _MeasurementTerm(tgt, wt, body_measurements, circumference_derivative)


def _adam(params, lr, iterations, loss_fn):
    """Adam on the tensors `params` over the batch sum of loss_fn()[0], the per-body loss; returns loss_fn() at the
    result, without a graph."""
    opt = torch.optim.Adam(params, lr=lr)
    # the step size decays geometrically to lr / 100 over the run, so the last iterations refine instead of orbiting
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda i: 0.01 ** (i / max(1, int(iterations))))
    for _ in range(int(iterations)):
        opt.zero_grad(set_to_none=True)
        loss_fn()[0].sum().backward()
        opt.step()
        sched.step()
    with torch.no_grad():
        return loss_fn()


def fit_betas_to_measurements(body_model, body_measurements, targets, weights=None, betas_weight=0.0, iterations=None,
                              lr=0.05, betas_init=None, batch_size=None, method='adam',
                              circumference_derivative='reference'):
    """Fits betas (B, NB) so that the model's T-pose measurements match `targets`.

    body_model: shapy_b200 SMPLX (its forward_shape and faces are used); body_measurements: shapy_b200
    BodyMeasurements on the same device.  targets: {name: float or (B,) values} for mass [kg], height, chest, waist,
    hips [m]; a missing name or a value <= 0 drops that term.  batch_size: B when every target is a scalar (default 1).
    method: 'adam' (the default) or 'lm' (Levenberg-Marquardt, see the top; `lr` is ignored).  iterations: None means
    500 for Adam and 50 for LM.  circumference_derivative: 'reference' or 'exact' (see the top).
    Returns {'betas': (B, NB), 'measurements': (B, 5) of the final betas (mass, height, chest, waist, hips),
    'loss': (B,) final per-body loss}."""
    if method not in ('adam', 'lm'):
        raise ValueError(f"method must be 'adam' or 'lm', got {method!r}")
    exact_circumferences(circumference_derivative)
    if iterations is None:
        iterations = 500 if method == 'adam' else 50
    device = body_model.shapedirs.device
    B = batch_size or max([torch.as_tensor(v).numel() for v in targets.values()] + [1])
    if betas_init is not None:
        B = betas_init.shape[0]
    mt = _measurement_term(targets, weights, B, device, body_measurements, circumference_derivative)
    if method == 'lm':
        return _fit_lm(body_model, mt, betas_weight, iterations, betas_init, B, device)
    nb = body_model.shapedirs.shape[-1]
    betas = (torch.zeros(B, nb, device=device) if betas_init is None else betas_init.detach().clone().float())
    betas.requires_grad_(True)

    def loss_fn():
        meas = mt.measure(body_model, betas)
        return mt.loss(meas, betas, betas_weight), meas

    per_body, meas = _adam([betas], lr, iterations, loss_fn)
    return {'betas': betas.detach(), 'measurements': meas, 'loss': per_body}


# Levenberg-Marquardt damping: divided by LM_DOWN after an accepted step, multiplied by LM_UP after a rejected one
LM_UP, LM_DOWN = 10.0, 3.0
# parameters of one body the keypoint LM step takes (kLmKpMaxP of fit.cu): 22 rotations, the betas and the translation
LM_KP_MAX_PARAMS = 96


def _check_kp_fit(fn, body_model, method, iterations, circumference_derivative='reference', body_measurements=None,
                  measurements=None, robust_sigma=None, pose_prior_weight=0.0, betas_weight=0.0):
    """The argument checks every keypoint fit makes, `fn` naming it in the messages.  Returns the iterations (None
    means 600 for Adam and 50 for LM) and robust_sigma as the fits take it (None for least squares)."""
    if method not in ('adam', 'lm'):
        raise ValueError(f"method must be 'adam' or 'lm', got {method!r}")
    exact_circumferences(circumference_derivative)
    if measurements is not None and body_measurements is None:
        raise ValueError(f'{fn}: measurements need body_measurements')
    if robust_sigma is not None and not robust_sigma > 0:
        raise ValueError(f'{fn}: robust_sigma must be > 0 or None, got {robust_sigma}')
    if not (pose_prior_weight >= 0 and betas_weight >= 0):
        raise ValueError(f'{fn}: pose_prior_weight and betas_weight must be >= 0')
    if method == 'lm' and 3 * 22 + body_model.num_betas + 3 > LM_KP_MAX_PARAMS:
        raise ValueError(f"{fn}(method='lm'): 22 rotations, {body_model.num_betas} betas and the translation or camera "
                         f'are {3 * 22 + body_model.num_betas + 3} parameters, at most {LM_KP_MAX_PARAMS} are '
                         f'supported (at most {LM_KP_MAX_PARAMS - 3 * 22 - 3} betas)')
    if iterations is None:
        iterations = 600 if method == 'adam' else 50
    return iterations, None if robust_sigma is None or robust_sigma == float('inf') else float(robust_sigma)


def measurement_jacobian(body_model, body_measurements, betas, circumference_derivative='reference'):
    """The measurements of forward_shape(betas) and their Jacobian with respect to betas, without autograd:
    {'measurements': (B, 5) (mass, height, chest, waist, hips, bit-identical to BodyMeasurements.forward_vertices),
    'jacobian': (B, 5, NB)}.  The Jacobian has the semantics of the measurements' backward for the same
    circumference_derivative ('reference': constant barycentrics, no gradient through the plane heights; 'exact': the
    circumferences' exact derivative); a NaN circumference gives a NaN row."""
    from . import ops
    exact = exact_circumferences(circumference_derivative)
    betas = torch.as_tensor(betas, dtype=torch.float32, device=body_model.shapedirs.device).detach().contiguous()
    packed = body_model.packed(betas.device)
    v = ops.smplx_forward_shape(packed, betas)
    out, jac, status = ops.measure_jacobian_betas(packed, body_measurements.landmarks(), v, body_model.faces_i32,
                                                  exact=exact)
    body_measurements.last_status = status
    return {'measurements': out, 'jacobian': jac}


def _fit_lm(body_model, mt, betas_weight, iterations, betas_init, B, device):
    from . import ops
    packed = body_model.packed(device)
    nb = packed.NB
    trial = (torch.zeros(B, nb, device=device) if betas_init is None
             else betas_init.detach().to(device=device, dtype=torch.float32).clone().contiguous())
    mk = lambda *s: torch.empty(*s, dtype=torch.float32, device=device)  # noqa: E731
    state = {'betas': mk(B, nb), 'meas': mk(B, 5), 'jac': mk(B, 5, nb), 'loss': mk(B), 'lambda': mk(B),
             'accepted': torch.zeros(B, dtype=torch.int32, device=device)}
    if B == 0:
        return {'betas': state['betas'], 'measurements': state['meas'], 'loss': state['loss']}
    mt.prime(body_model)
    for it in range(int(iterations) + 1):
        meas, jac = mt.trial(packed, body_model, trial)
        ops.fit_lm_step(state, mt.tgt, mt.wt, betas_weight, LM_UP, LM_DOWN, it == 0, trial, meas, jac)
    return {'betas': state['betas'], 'measurements': state['meas'], 'loss': state['loss']}


IDENT6 = (1.0, 0.0, 0.0, 1.0, 0.0, 0.0)      # the 6D code of the identity rotation (row-major 3x2)


def _start_params(init, B, nb, device, method, last, last0=0.0):
    """The raw 6D global and body pose, betas and last three parameters (named `last`: 'transl' or 'camera') a keypoint
    fit starts from: init's entries, and for a missing one the identity pose, zero betas and (last0, 0, 0)."""
    ident = torch.zeros(6, device=device)      # IDENT6, filled on the device: no host-to-device copy
    ident[0::3].fill_(1.0)
    last3 = torch.zeros(B, 3, device=device)
    if last0:
        last3[:, 0].fill_(last0)
    start = {'global_rot': ident.repeat(B, 1), 'body_pose': ident.repeat(B, 21),
             'betas': torch.zeros(B, nb, device=device), last: last3}
    params = {}
    for k, v in start.items():
        t = init.get(k)
        t = v if t is None else torch.as_tensor(t, dtype=torch.float32, device=device).reshape(v.shape)
        params[k] = t.detach().clone().contiguous().requires_grad_(method == 'adam')
    return params


def keypoint_jacobian(body_model, rot, betas, transl=None):
    """The model's keypoints (its joints output, expression zero, plus transl) and their Jacobian without autograd:
    rot (B, n_rot, 3, 3) of the first n_rot joints, betas (B, NB), transl (B, 3) or None.  Returns {'keypoints'
    (B, K, 3), 'jacobian' (B, 3K, 3 n_rot + NB + 3)}, columns [delta_j (R_j Exp(delta_j) at delta = 0) | betas |
    transl], with the semantics of the SMPL-X backward (constant LUT row, J14 overwrite)."""
    from . import ops
    device = body_model.shapedirs.device
    f = lambda t: None if t is None else torch.as_tensor(t, dtype=torch.float32, device=device).detach().contiguous()  # noqa: E731
    kp, jac = ops.smplx_keypoint_jacobian(body_model.packed(device), f(betas), f(rot), f(transl))
    return {'keypoints': kp, 'jacobian': jac}


def fit_body_to_keypoints(body_model, keypoints, weights=None, iterations=None, lr=0.05, init=None, method='adam',
                          body_measurements=None, measurements=None, measurement_weights=None, betas_weight=0.0,
                          circumference_derivative='reference'):
    """Fits pose and shape so that the model's keypoints match `keypoints` (B, K, 3), K = body_model's keypoint count.

    weights: None (all 1), (K,) or (B, K) per-keypoint weights.  init: optional {'global_rot': (B, 6),
    'body_pose': (B, 126) raw 6D, 'betas': (B, NB), 'transl': (B, 3)}; a missing entry starts at the identity pose,
    zero betas or zero transl.  method: 'adam' (the default: the step size decays geometrically from lr to lr / 100)
    or 'lm' (batched Levenberg-Marquardt on the keypoint Jacobian, see the top; `lr` is ignored, a keypoint with
    weight <= 0 is dropped).  iterations: None means 600 for Adam and 50 for LM.
    measurements: optional known measurements of the bodies, fitted together with the keypoints: the targets dict of
    fit_betas_to_measurements ({name: float or (B,) values}, mass [kg], height, chest, waist, hips [m]), with
    measurement_weights over DEFAULT_WEIGHTS and the same dropping rule (a target <= 0 or a weight <= 1e-3 drops
    that term), measured by body_measurements (required with them) on the T-pose of the fitted betas; betas_weight
    adds betas_weight |betas|^2 and needs measurements.  circumference_derivative: 'reference' or 'exact', how the
    circumferences of the measurement term are differentiated (see the top).
    Returns {'global_rot', 'body_pose' (raw 6D), 'betas', 'transl', 'global_rot_mat' (B, 1, 3, 3),
    'body_pose_mat' (B, 21, 3, 3), 'keypoints' (B, K, 3) of the final parameters, 'loss' (B,) final per-body loss},
    with measurements also 'measurements' (B, 5) of the final betas (mass, height, chest, waist, hips), and 'loss'
    the total: keypoints + measurements + betas_weight |betas|^2."""
    iterations, _ = _check_kp_fit('fit_body_to_keypoints', body_model, method, iterations, circumference_derivative,
                                  body_measurements, measurements)
    if measurements is None and betas_weight != 0:
        raise ValueError('fit_body_to_keypoints: betas_weight needs measurements (the keypoint fit has no betas prior)')
    if not betas_weight >= 0:
        raise ValueError(f'fit_body_to_keypoints: betas_weight must be >= 0, got {betas_weight}')
    from .autograd import Rot6dFunction
    device = body_model.shapedirs.device
    kp = torch.as_tensor(keypoints, dtype=torch.float32, device=device)
    B, K = kp.shape[0], kp.shape[1]
    w = torch.ones(K, device=device) if weights is None else torch.as_tensor(weights, dtype=torch.float32,
                                                                             device=device)
    w = w.expand(B, K).contiguous()
    mt = _measurement_term(measurements, measurement_weights, B, device, body_measurements, circumference_derivative)
    rho = float(betas_weight)
    params = _start_params(init or {}, B, body_model.num_betas, device, method, 'transl')
    if method == 'lm':
        return _fit_keypoints_lm(body_model, kp, w, params, int(iterations), mt, rho)

    def loss_fn():
        grot = Rot6dFunction.apply(params['global_rot'])
        bpose = Rot6dFunction.apply(params['body_pose'])
        out = body_model(global_rot=grot, body_pose=bpose, betas=params['betas'], transl=params['transl'],
                         return_shaped=False)
        joints = out['joints'][:]                  # the KeypointTensor's tensor, still in the graph
        per_body = ((joints - kp).pow(2).sum(-1) * w).sum(1)
        meas = None
        if mt is not None:
            meas = mt.measure(body_model, params['betas'])
            per_body = per_body + mt.loss(meas, params['betas'], rho)
        return per_body, joints, grot, bpose, meas

    per_body, joints, grot, bpose, meas = _adam(list(params.values()), lr, iterations, loss_fn)
    return _adam_result(params, grot, bpose, meas, keypoints=joints, loss=per_body)


def _adam_result(params, grot, bpose, meas, **outputs):
    """What an Adam keypoint fit returns: the fitted raw parameters, the rotations, `outputs` and, with measurements
    (meas not None), 'measurements'."""
    res = {k: v.detach() for k, v in params.items()}
    res.update(global_rot_mat=grot, body_pose_mat=bpose, **outputs)
    if meas is not None:
        res['measurements'] = meas
    return res


def _kp_lm_state(B, K, n_rot, nb, last, device, G=None, ne=None):
    """The state tensors of a keypoint LM step (ops.fit_lm_keypoints_step), `last` naming the last three parameters;
    with G, the grouped steps' state: 'betas', 'loss', 'lambda' and 'accepted' per group; with ne, the wide 2D step's
    state (ops.fit_lm_keypoints_2d_expressive_step): 'expression' (B, ne) and ne more Jacobian columns."""
    G = B if G is None else G
    mk = lambda *s: torch.empty(*s, dtype=torch.float32, device=device)  # noqa: E731
    state = {'rot': mk(B, n_rot, 3, 3), 'betas': mk(G, nb), last: mk(B, 3), 'keypoints': mk(B, K, 3),
             'jac': mk(B, 3 * K, 3 * n_rot + nb + (ne or 0) + 3), 'loss': mk(G), 'lambda': mk(G),
             'accepted': torch.zeros(G, dtype=torch.int32, device=device)}
    if ne is not None:
        state['expression'] = mk(B, ne)
    return state


def _kp_lm_result(state, last, **outputs):
    """The fitted parameters of a keypoint LM state as the fits return them, the rotations also as raw 6D, then
    `outputs` and, with measurements, 'measurements'."""
    rot = state['rot']
    raw = rot[..., :2].reshape(rot.shape[0], 6 * rot.shape[1])   # the first two columns, the decoder's row-major 3x2
    res = {'global_rot': raw[:, :6].contiguous(), 'body_pose': raw[:, 6:].contiguous(), 'betas': state['betas'],
           last: state[last], 'global_rot_mat': rot[:, :1], 'body_pose_mat': rot[:, 1:], **outputs}
    if 'meas' in state:
        res['measurements'] = state['meas']
    return res


def _fit_keypoints_lm(body_model, kp, w, params, iterations, mt, rho):
    from . import ops
    device = kp.device
    packed = body_model.packed(device)
    B, K = kp.shape[0], kp.shape[1]
    n_rot, nb = 22, params['betas'].shape[1]
    trial = {'rot': ops.decode_rot6d(torch.cat([params['global_rot'], params['body_pose']], 1)).contiguous(),
             'betas': params['betas'].contiguous(), 'transl': params['transl'].contiguous()}
    state = _kp_lm_state(B, K, n_rot, nb, 'transl', device)
    tg = kp.contiguous()
    if mt is not None:
        state.update(mt.state(nb, device))
    if B > 0:
        if mt is not None:
            mt.prime(body_model)
        for it in range(iterations + 1):
            tkp, tjac = ops.smplx_keypoint_jacobian(packed, trial['betas'], trial['rot'], trial['transl'])
            if mt is None:
                ops.fit_lm_keypoints_step(state, trial, tg, w, LM_UP, LM_DOWN, it == 0, tkp, tjac)
            else:
                tm, tmj = mt.trial(packed, body_model, trial['betas'])
                ops.fit_lm_keypoints_measurements_step(state, trial, tg, w, mt.tgt, mt.wt, rho, LM_UP, LM_DOWN,
                                                       it == 0, tkp, tjac, tm, tmj)
    rot = state['rot']
    with torch.no_grad():
        out = body_model(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=state['betas'], transl=state['transl'],
                         return_shaped=False)
        joints = out['joints'][:]
        per_body = ((joints - kp).pow(2).sum(-1) * w).sum(1)
        if mt is not None:
            per_body = per_body + mt.loss(state['meas'], state['betas'], rho)
    return _kp_lm_result(state, 'transl', keypoints=joints, loss=per_body)


def keypoint_jacobian_2d(body_model, rot, betas, camera):
    """The projected keypoints p_k = softplus(c0) (kp_k,xy + c[1:3]) and their Jacobian, composed from
    keypoint_jacobian (no transl): rot (B, n_rot, 3, 3), betas (B, NB), camera (B, 3).  Returns {'proj_joints'
    (B, K, 2), 'jacobian' (B, 2K, 3 n_rot + NB + 3)}, rows 2k + c (x, y), columns [delta_j | betas | c0, c1, c2]: the x
    and y rows of the 3D Jacobian times s on the rotation and betas columns, sigmoid(c0) (kp_xy + c[1:3]) on c0 (1 past
    softplus' threshold of 20), s on c1 and c2 (the step kernel stages the same rows in fp64)."""
    device = body_model.shapedirs.device
    camera = torch.as_tensor(camera, dtype=torch.float32, device=device)
    res = keypoint_jacobian(body_model, rot, betas)
    kp, jac = res['keypoints'], res['jacobian']
    B, K = kp.shape[:2]
    P = jac.shape[2]
    c0 = camera[:, 0]
    s = torch.nn.functional.softplus(c0)                                      # threshold 20, as the forward
    ds = torch.where(c0 > 20, torch.ones_like(c0), torch.sigmoid(c0))
    xy = kp[..., :2] + camera[:, None, 1:3]                                   # (B, K, 2)
    j2 = torch.zeros(B, K, 2, P, dtype=torch.float32, device=device)
    j2[..., :P - 3] = s[:, None, None, None] * jac.view(B, K, 3, P)[:, :, :2, :P - 3]
    j2[..., P - 3] = ds[:, None, None] * xy
    j2[:, :, 0, P - 2] = s[:, None]
    j2[:, :, 1, P - 1] = s[:, None]
    return {'proj_joints': s[:, None, None] * xy, 'jacobian': j2.view(B, 2 * K, P)}


def _kp2d_loss(proj, target, w, sigma, pose_w, rot, anchor, betas_w, betas, joint_w=None, expr_w=0.0, expr=None):
    """The 2D fit's per-body loss: sum_{w_k > 0} w_k rho(|proj_k - target_k|^2) + pose_w / 2 sum_{j >= 1}
    |R_j - R0_j|_F^2 + betas_w |betas|^2, rho(e) = e (sigma None) or sigma^2 e / (sigma^2 + e), over all n_rot
    rotations of rot.  joint_w (n_rot,) (joint 0 unread; with pose_w 0): the pose prior per joint,
    sum_{j >= 1} joint_w_j / 2 |R_j - R0_j|_F^2; expr (B, NE): expr_w |psi|^2 as well."""
    keep = w > 0
    diff = torch.where(keep[..., None], proj - torch.where(keep[..., None], target, torch.zeros_like(target)),
                       torch.zeros_like(proj))
    e = diff.pow(2).sum(-1)
    if sigma is not None:
        e = sigma * sigma * e / (sigma * sigma + e)
    per_body = (torch.where(keep, w, torch.zeros_like(w)) * e).sum(1)
    if pose_w > 0:
        per_body = per_body + 0.5 * pose_w * (rot[:, 1:] - anchor[:, 1:]).pow(2).sum((1, 2, 3))
    if betas_w > 0:
        per_body = per_body + betas_w * betas.pow(2).sum(1)
    if joint_w is not None:
        d = (rot[:, 1:] - anchor[:, 1:]).pow(2).sum((2, 3))                  # (B, n_rot - 1)
        per_body = per_body + (0.5 * joint_w[1:] * d).sum(1)
    if expr is not None and expr_w > 0:
        per_body = per_body + expr_w * expr.pow(2).sum(1)
    return per_body


def _raw_init(init):
    """A copy of init with the regressor's raw_global_rot / raw_body_pose, when given, as global_rot / body_pose."""
    init = dict(init or {})
    for k in ('global_rot', 'body_pose'):
        if init.get('raw_' + k) is not None:
            init[k] = init['raw_' + k]
    return init


def _keypoints_2d(fn, keypoints2d, weights, device):
    """The 2D targets as a contiguous float32 (B, K, 2) tensor and their weights (None: all 1, (K,) or (B, K)) as
    (B, K)."""
    x = torch.as_tensor(keypoints2d, dtype=torch.float32, device=device).contiguous()
    if x.dim() != 3 or x.shape[2] != 2:
        raise ValueError(f'{fn}: keypoints2d must be (B, K, 2), got {tuple(x.shape)}')
    B, K = x.shape[0], x.shape[1]
    w = torch.ones(K, device=device) if weights is None else torch.as_tensor(weights, dtype=torch.float32,
                                                                             device=device)
    return x, w.expand(B, K).contiguous()


def _start_rotations(params, pose_anchor, n, parts=()):
    """The decoded starting rotations (n, n_rot, 3, 3) of a fit's raw 6D params, the global rotation, the body and the
    pose parts `parts` of _parts_in (n_rot = 22 without), and the pose prior's anchor: pose_anchor as
    (n, n_rot, 3, 3), by default the start."""
    from . import ops
    raw = torch.cat([params['global_rot'], params['body_pose']] + [params[name] for name, _, _ in parts], 1)
    rot0 = ops.decode_rot6d(raw.detach()).contiguous()
    if pose_anchor is None:
        return rot0, rot0
    return rot0, torch.as_tensor(pose_anchor, dtype=torch.float32, device=rot0.device).reshape(
        n, rot0.shape[1], 3, 3).contiguous()


def _forward_2d(body_model, grot, bpose, betas, last, intr, parts=None, expression=None):
    """SMPLX.forward of a 2D fit with its proj_joints: `last` the weak-perspective camera (intr None) or the
    translation seen by the perspective camera with intrinsics intr (B, 3); parts: the rotations of the pose parts
    past the body by SMPLX.forward's names, expression (B, NE) or None."""
    kw = dict(parts or {}, expression=expression)
    if intr is None:
        return body_model(global_rot=grot, body_pose=bpose, betas=betas, camera=last, return_shaped=False, **kw)
    out = body_model(global_rot=grot, body_pose=bpose, betas=betas, transl=last, return_shaped=False, **kw)
    out['proj_joints'] = _project(out['joints'][:], intr)
    return out


def _init_2d(init, B, nb, device, method, x=None, w=None, intr=None):
    """The raw 6D global and body pose, betas and camera to start from: fit_body_to_keypoints' init with 'camera' in
    place of 'transl'; the regressor's stage output (raw_global_rot, raw_body_pose, betas, camera) works as-is.  With
    intrinsics intr (B, 3) the last three are 'transl', by default START_DEPTH in front of the camera on the ray
    through the centroid of the keypoints x with weight w > 0 (the principal point without one)."""
    init = _raw_init(init)
    if intr is None:
        return _start_params(init, B, nb, device, method, 'camera', 0.9)   # softplus(0.9) ~ 1.24, the mean scale
    if init.get('transl') is None:
        keep = (w > 0)[..., None]
        n = keep.sum(1).clamp(min=1)
        c = torch.where(keep, x, torch.zeros_like(x)).sum(1) / n
        c = torch.where(keep.any(1), c, intr[:, 1:])
        init['transl'] = torch.cat([(c - intr[:, 1:]) * START_DEPTH / intr[:, :1],
                                    torch.full((B, 1), START_DEPTH, device=device)], 1)
    return _start_params(init, B, nb, device, method, 'transl')


# the distance [m] a perspective fit starts at without a translation: a person photographed whole with a phone
START_DEPTH = 3.0


def _intrinsics(focal_length, principal_point, B, device):
    """(B, 3) float32 (f, px, py) from a scalar or (B,) focal length and a (2,) or (B, 2) principal point; numbers are
    filled on the device (no host-to-device copy)."""
    num = lambda v: isinstance(v, (int, float, np.floating))  # noqa: E731
    if num(focal_length):
        f = torch.full((B,), float(focal_length), device=device)
    else:
        f = torch.as_tensor(focal_length, dtype=torch.float32, device=device).reshape(-1)
    if isinstance(principal_point, (tuple, list)) and len(principal_point) == 2 and all(map(num, principal_point)):
        pp = torch.stack([torch.full((B,), float(v), device=device) for v in principal_point], 1)
    else:
        pp = torch.as_tensor(principal_point, dtype=torch.float32, device=device).reshape(-1, 2)
    if f.numel() not in (1, B) or pp.shape[0] not in (1, B):
        raise ValueError(f'fit_body_to_keypoints_2d: focal_length must be a scalar or ({B},) and principal_point (2,) '
                         f'or ({B}, 2), got {tuple(f.shape)} and {tuple(pp.shape)}')
    return torch.cat([f.expand(B)[:, None], pp.expand(B, 2)], 1).contiguous()


def _project(joints, intr):
    """The perspective projection of the fit, through the camera module's PerspectiveCamera: joints (B, K, 3) in the
    camera frame (transl included), intr (B, 3)."""
    from .human_shape.models.camera.camera_projection import PerspectiveCamera
    return PerspectiveCamera()(joints, focal_length=intr[:, 0], camera_center=intr[:, 1:])


def _depth_rule(per_body, joints, w):
    """+inf for a body with a weighted keypoint at Y_z <= 0 or not finite (the perspective step's rule)."""
    z = joints[..., 2]
    bad = ((w > 0) & ~(z > 0)).any(1) | ((w > 0) & ~torch.isfinite(z)).any(1)
    return torch.where(bad, torch.full_like(per_body, float('inf')), per_body)


def perspective_start(camera, center, scale, focal_length, principal_point):
    """The starting translation (B, 3) of a perspective fit from the regressor's weak-perspective crop camera (B, 3)
    and the crop descriptors: center (B, 2) in pixels and scale (B,) = box / 200 (as keypoints2d.to_crop), focal_length
    a scalar or (B,) and principal_point (2,) or (B, 2) in pixels.  With s = softplus(c0) and h = 200 scale:
    t_z = 2 f / (s h), t_xy = c[1:3] + (center - pp) t_z / f.  Points at Y_z = t_z then project exactly where the crop
    projection puts them, mapped back to pixels (up to to_crop's +1 and pixel rounding); nearer or farther points
    differ by O(depth / t_z).  Unlike the reference demo's conversion, the real principal point is kept."""
    camera = torch.as_tensor(camera, dtype=torch.float32)
    dev = camera.device
    center = torch.as_tensor(center, dtype=torch.float32, device=dev).reshape(-1, 2)
    h = 200.0 * torch.as_tensor(scale, dtype=torch.float32, device=dev).reshape(-1)
    f = torch.as_tensor(focal_length, dtype=torch.float32, device=dev).reshape(-1)
    pp = torch.as_tensor(principal_point, dtype=torch.float32, device=dev).reshape(-1, 2)
    s = torch.nn.functional.softplus(camera[:, 0])
    tz = 2.0 * f / (s * h)
    txy = camera[:, 1:3] + (center - pp) * (tz / f)[:, None]
    return torch.cat([txy, tz[:, None]], 1)


def group_plan(groups, B):
    """The images of each group, from labels (B,) of integers 0 .. G-1, each used at least once: (order (B,) int64, the
    stable sort of the labels, so that the caller's order within a group is kept; offsets (G + 1,) int32, group g the
    sorted images [offsets[g], offsets[g + 1])), both on the CPU.  Labels on the device are read once on the host
    (one synchronisation, before any fit loop); labels on the CPU cost none."""
    g = torch.as_tensor(groups).detach().cpu()
    if g.dtype.is_floating_point or g.dtype == torch.bool or g.dtype.is_complex or g.shape != (B,):
        raise ValueError(f'groups must be a ({B},) integer tensor, got {g.dtype} {tuple(g.shape)}')
    g = g.long()
    if B and int(g.min()) < 0:
        raise ValueError('groups: labels must be >= 0')
    counts = torch.bincount(g) if B else torch.zeros(0, dtype=torch.long)
    if bool((counts == 0).any()):
        raise ValueError(f'groups: labels must be 0 .. G-1, each used at least once; label {int((counts == 0).nonzero()[0])} '
                         f'is not used')
    order = torch.sort(g, stable=True).indices
    offsets = torch.cat([torch.zeros(1, dtype=torch.long), counts.cumsum(0)]).to(torch.int32)
    return order, offsets


def _to_device(t, device):
    """A host tensor on `device` without synchronising (a non-blocking copy from pinned memory)."""
    if torch.device(device).type != 'cuda':
        return t.to(device)
    return t.pin_memory().to(device, non_blocking=True)


def _group_sum(x, offsets):
    """Per group, the sum of the rows of x (sorted by group) in image order, left to right: (G, ...)."""
    off = offsets.long()
    cnt = off[1:] - off[:-1]
    start, cnt_d = _to_device(off[:-1], x.device), _to_device(cnt, x.device)
    acc = x[start]
    for j in range(1, int(cnt.max()) if cnt.numel() else 0):
        more = (cnt_d > j).view(-1, *([1] * (x.dim() - 1)))
        acc = torch.where(more, acc + x[(start + j).clamp(max=x.shape[0] - 1)], acc)
    return acc


def fit_body_to_keypoints_2d(body_model, keypoints2d, weights=None, init=None, method='adam', iterations=None,
                             robust_sigma=None, pose_prior_weight=0.0, betas_weight=0.0, pose_anchor=None, lr=0.05,
                             body_measurements=None, measurements=None, measurement_weights=None,
                             circumference_derivative='reference', groups=None, share_pose=False, focal_length=None,
                             principal_point=None, pose_width=22, fit_expression=False, expression_weight=0.0):
    """Fits pose, shape and the weak-perspective camera so that the projected keypoints proj_joints = softplus(c0)
    (joints_xy + c[1:3]) match `keypoints2d` (B, K, 2), K = body_model's keypoint count, in the normalised crop frame of
    the regressor's proj_joints (shapy_b200.keypoints2d.to_crop maps pixel detections there).

    Loss per body: sum_{w_k > 0} w_k rho(|p_k - x_k|^2) + pose_prior_weight / 2 sum_{j=1}^{21} |R_j - R0_j|_F^2 +
    betas_weight |betas|^2, rho(e) = e when robust_sigma is None, else the Geman-McClure sigma^2 e / (sigma^2 + e).
    R0 = pose_anchor (B, 22, 3, 3), by default the starting rotations: the prior keeps the body pose near the
    regressor's prediction (the global rotation has no prior).  weights: None (all 1), (K,) or (B, K); a keypoint with
    weight <= 0 is dropped and its target may be NaN.  init: fit_body_to_keypoints' init with 'camera' (B, 3) in place
    of 'transl' (the regressor's stage output, with raw_global_rot / raw_body_pose, works as-is); without a camera the
    fit starts at c = (0.9, 0, 0).  method: 'adam' (the step size decays geometrically from lr to lr / 100, through
    SMPLX.forward(camera=...) and the 6D decoder) or 'lm' (batched Levenberg-Marquardt: the raw 6D start is decoded
    once, then per iteration the keypoint Jacobian of the trial and one ops.fit_lm_keypoints_2d_step, two launches,
    no host synchronisation; every body's loss is non-increasing).  iterations: None means 600 for Adam and 50 for LM.
    measurements: optional known measurements of the bodies, fitted together with the keypoints, with the vocabulary
    of fit_body_to_keypoints: the targets dict of fit_betas_to_measurements, measurement_weights over DEFAULT_WEIGHTS,
    the same dropping rule, measured by body_measurements (required with them) on the T-pose of the fitted betas, and
    circumference_derivative 'reference' or 'exact'.  The loss gains sum_m u_m (t_m - meas_m)^2; betas_weight stays the
    one betas regulariser.  With 'lm' an iteration then takes four launches (see the top).
    Returns {'global_rot', 'body_pose' (raw 6D), 'betas', 'camera', 'global_rot_mat' (B, 1, 3, 3), 'body_pose_mat'
    (B, 21, 3, 3), 'keypoints' (B, K, 3) and 'proj_joints' (B, K, 2) of the final parameters, 'loss' (B,)}, with
    measurements also 'measurements' (B, 5) of the final betas (mass, height, chest, waist, hips), and 'loss' the
    total.
    groups: None, or (B,) integer labels 0 .. G-1, each used at least once: images with the same label are one person
    and share their betas.  init, weights and pose_anchor stay per image; a group starts from the mean of its images'
    init betas (image order).  measurements and measurement_weights are then per group ((G,) values or scalars).
    'betas' (G, NB), 'measurements' (G, 5) and 'loss' (G,) are per group, the rest per image in the caller's order.
    With 'lm' the returned loss is the step's fp64 loss of the final state; the images of a group are summed in the
    caller's order.
    share_pose: with groups, the images of a group are simultaneous views of one posed body (a synchronised rig, or
    front and side photos of one held pose) and also share the body pose: each keeps its global rotation (which absorbs
    the camera's rotation) and camera.  A limb one view sees foreshortened another sees side-on, which a single
    weak-perspective view cannot.  A group starts from the image-order mean of its images' decoded starting body
    rotations, made rotations again by the 6D decoder's Gram-Schmidt; pose_anchor is then per group, (G, 22, 3, 3)
    with the global rows unread, by default that start, and the pose prior counts once per group.  'body_pose' and
    'body_pose_mat' are then per group as well.  With 'lm' an iteration is the keypoint Jacobian of every image and
    ops.fit_lm_keypoints_2d_shared_pose_step (six launches with measurements).
    focal_length: None (the weak-perspective fit above), or a scalar or (B,) focal length f > 0 with principal_point
    (2,) or (B, 2) (required with it): the fit is then perspective, p_k = f (Y_x / Y_z, Y_y / Y_z) + principal_point,
    Y_k = joint_k + transl, camera frame x right, y down, z forward.  keypoints2d are then in the intrinsics' units,
    init may carry 'transl' (B, 3) in the place of 'camera' (without one the fit starts 3 m in front of the camera, on
    the ray through the centroid of the weighted keypoints; perspective_start converts a regressor's crop camera), and
    the result has 'transl' instead of 'camera' and perspective 'proj_joints'.  'lm' loops over the keypoint Jacobian
    and ops.fit_lm_keypoints_2d_perspective_step (with measurements, forward_shape and the measurement Jacobian as
    well); 'adam' fits raw 6D pose, betas and transl through SMPLX.forward(transl=...) and PerspectiveCamera.  A trial
    with a weighted keypoint at Y_z <= 0 is rejected by 'lm'; the returned loss is +inf for a body that has one.
    The measurement weights are the crop frame's; with targets in pixels a known height needs a larger weight to
    count (measurement_weights={'height': 1e6}: 1 mm of height costs what 1 px of one keypoint does).  groups and
    share_pose are not supported with a focal length.
    pose_width: 22 (the global rotation and the body), or 23, 24, 25, 40 or 55 to fit the jaw, the eyes and the hands
    as well (SMPL-X's joint order: jaw, left eye, right eye, 15 left-hand and 15 right-hand joints); fit_expression
    also fits the NE expression coefficients psi, with the regulariser expression_weight |psi|^2.  Either one takes
    the wide path: init may carry raw 6D 'jaw_pose' (B, 6), 'leye_pose', 'reye_pose', 'left_hand_pose' (B, 90) and
    'right_hand_pose' for the parts inside the width and 'expression' (B, NE); a part without one starts at the
    identity and the expression at 0.  pose_prior_weight may then be a scalar or (pose_width,) per-joint weights with
    joint 0 zero, so that the hands, jaw and eyes can be held differently from the body; pose_anchor is (B,
    pose_width, 3, 3).  'lm' runs ops.smplx_keypoint_jacobian(expr=...) and ops.fit_lm_keypoints_2d_expressive_step per
    iteration (two launches, no host synchronisation; at most 200 parameters); 'adam' fits the same loss through
    SMPLX.forward.  The result also holds the raw 6D parts in the width, 'full_pose_mat' (B, pose_width, 3, 3) and,
    when fitted, 'expression'.  A part is only as determined as its keypoints make it: one without a weighted keypoint
    (the eyes: the OpenPose pupils are dropped on load) is held by its prior alone, and without a prior it stays where
    it starts.  groups, share_pose and measurements are not supported on the wide path."""
    fn = 'fit_body_to_keypoints_2d'
    wide = pose_width != 22 or fit_expression
    ne, jw = 0, None
    if wide:
        if pose_width not in POSE_WIDTHS:
            raise ValueError(f'{fn}: pose_width must be one of {POSE_WIDTHS}, got {pose_width}')
        if groups is not None or share_pose or measurements is not None:
            raise ValueError(f'{fn}: groups, share_pose and measurements are not supported with a pose_width past 22 '
                             f'or fit_expression')
        if focal_length is not None and principal_point is None:
            raise ValueError(f'{fn}: focal_length needs principal_point')
        if not expression_weight >= 0:
            raise ValueError(f'{fn}: expression_weight must be >= 0')
        if np.ndim(pose_prior_weight) > 0:
            jw = torch.as_tensor(pose_prior_weight, dtype=torch.float32).detach().cpu().reshape(-1)
            if jw.shape != (pose_width,) or float(jw[0]) != 0 or not bool((jw >= 0).all()):
                raise ValueError(f'{fn}: per-joint pose_prior_weight must be ({pose_width},), >= 0, with joint 0 zero')
            pose_prior_weight = 0.0
        ne, nb = body_model.num_expression_coeffs if fit_expression else 0, body_model.num_betas
        if method == 'lm' and 3 * pose_width + nb + ne + 3 > LM_WIDE_MAX_PARAMS:
            raise ValueError(f"{fn}(method='lm'): {pose_width} rotations, {nb} betas, {ne} expression coefficients "
                             f'and the translation or camera are {3 * pose_width + nb + ne + 3} parameters, at most '
                             f'{LM_WIDE_MAX_PARAMS} are supported')
        # _check_kp_fit's checks; its parameter bound is the 22-joint step's, so it sees the Adam method
        iterations, sigma = _check_kp_fit(fn, body_model, 'adam' if method == 'lm' else method,
                                          50 if method == 'lm' and iterations is None else iterations,
                                          robust_sigma=robust_sigma, pose_prior_weight=pose_prior_weight,
                                          betas_weight=betas_weight)
    else:
        iterations, sigma = _check_kp_fit(fn, body_model, method, iterations, circumference_derivative,
                                          body_measurements, measurements, robust_sigma, pose_prior_weight,
                                          betas_weight)
        if share_pose and groups is None:
            raise ValueError(f'{fn}: share_pose needs groups')
        if focal_length is not None and (groups is not None or share_pose):
            raise ValueError(f'{fn}: groups and share_pose are not supported with a focal_length')
        if focal_length is not None and principal_point is None:
            raise ValueError(f'{fn}: focal_length needs principal_point')
    from .autograd import Rot6dFunction
    device, nb = body_model.shapedirs.device, body_model.num_betas
    x, w = _keypoints_2d(fn, keypoints2d, weights, device)
    B = x.shape[0]
    intr = None if focal_length is None else _intrinsics(focal_length, principal_point, B, device)
    params = _init_2d(init, B, nb, device, method, x, w, intr)
    parts = _parts_in(pose_width)
    raw_init = _raw_init(init)
    ident = torch.zeros(6, device=device) if parts else None     # IDENT6, filled on the device
    if parts:
        ident[0::3].fill_(1.0)
    for name, _, n in parts:        # the pose parts past the body, by default at the identity
        t = raw_init.get(name)
        t = ident.repeat(B, n) if t is None else \
            torch.as_tensor(t, dtype=torch.float32, device=device).reshape(B, 6 * n)
        params[name] = t.detach().clone().contiguous().requires_grad_(method == 'adam')
    if fit_expression:
        t = raw_init.get('expression')
        t = torch.zeros(B, ne, device=device) if t is None else \
            torch.as_tensor(t, dtype=torch.float32, device=device).reshape(B, ne)
        params['expression'] = t.detach().clone().contiguous().requires_grad_(method == 'adam')
    rot0, anchor = _start_rotations(params, None if share_pose else pose_anchor, B, parts)
    if share_pose:          # per group: its shape is checked once the groups are known
        anchor = None if pose_anchor is None else torch.as_tensor(pose_anchor, dtype=torch.float32, device=device)
    pw, bw, ew = float(pose_prior_weight), float(betas_weight), float(expression_weight)
    if groups is not None:
        return _fit_keypoints_2d_groups(body_model, x, w, params, rot0, anchor, method, int(iterations), sigma, pw, bw,
                                        lr, groups, body_measurements, measurements, measurement_weights,
                                        circumference_derivative, bool(share_pose))
    jw = None if jw is None else jw.to(device)
    mt = _measurement_term(measurements, measurement_weights, B, device, body_measurements, circumference_derivative)
    last = 'camera' if intr is None else 'transl'
    if method == 'lm':
        return _fit_keypoints_2d_lm(body_model, x, w, params, parts, rot0, anchor, int(iterations), sigma, pw, jw, bw,
                                    ew, ne, mt, intr, wide)

    def loss_fn():
        grot = Rot6dFunction.apply(params['global_rot'])
        bpose = Rot6dFunction.apply(params['body_pose'])
        pr = {name: Rot6dFunction.apply(params[name]) for name, _, _ in parts}
        expr = params.get('expression')
        out = _forward_2d(body_model, grot, bpose, params['betas'], params[last], intr, pr, expr)
        rot = torch.cat([grot, bpose] + list(pr.values()), 1)
        per_body = _kp2d_loss(out['proj_joints'], x, w, sigma, pw, rot, anchor, bw, params['betas'], jw, ew, expr)
        meas = None
        if mt is not None:      # _kp2d_loss already counted betas_weight |betas|^2
            meas = mt.measure(body_model, params['betas'])
            per_body = per_body + mt.loss(meas, params['betas'], 0.0)
        return per_body, out, rot, meas

    per_body, out, rot, meas = _adam(list(params.values()), lr, iterations, loss_fn)
    if intr is not None:
        per_body = _depth_rule(per_body, out['joints'][:], w)
    wide_out = {'full_pose_mat': rot} if wide else {}
    return _adam_result(params, rot[:, :1], rot[:, 1:22], meas, **wide_out, keypoints=out['joints'][:],
                        proj_joints=out['proj_joints'], loss=per_body)


def _fit_keypoints_2d_lm(body_model, x, w, params, parts, rot0, anchor, iterations, sigma, pw, jw, bw, ew, ne, mt, intr,
                         wide):
    """The LM loop of fit_body_to_keypoints_2d: per iteration the keypoint Jacobian of the trial, with measurements
    their trial values and Jacobian, and one single-image 2D step; `wide` runs the expressive step."""
    from . import ops
    device = x.device
    packed = body_model.packed(device)
    B, K = x.shape[0], x.shape[1]
    nb, n_rot = params['betas'].shape[1], rot0.shape[1]
    last = 'camera' if intr is None else 'transl'
    trial = {'rot': rot0.clone(), 'betas': params['betas'].contiguous(), last: params[last].contiguous()}
    state = _kp_lm_state(B, K, n_rot, nb, last, device, ne=ne if wide else None)
    kw = {'pose_anchor': anchor if pw > 0 or jw is not None else None}
    if intr is not None:
        kw['intrinsics'] = intr
    if wide:
        step = ops.fit_lm_keypoints_2d_expressive_step
        trial['expression'] = (params['expression'] if ne else torch.zeros(B, 0, device=device)).clone().contiguous()
        kw.update(expression_weight=ew, joint_weights=jw)
    elif mt is None:
        step = ops.fit_lm_keypoints_2d_step if intr is None else ops.fit_lm_keypoints_2d_perspective_step
    else:
        step = ops.fit_lm_keypoints_2d_measurements_step if intr is None else \
            ops.fit_lm_keypoints_2d_perspective_measurements_step
        state.update(mt.state(nb, device))
    if B > 0:
        if mt is not None:
            mt.prime(body_model)
        for it in range(iterations + 1):
            tkp, tjac = ops.smplx_keypoint_jacobian(packed, trial['betas'], trial['rot'],
                                                    expr=trial['expression'] if ne else None)
            if mt is not None:
                tm, tmj = mt.trial(packed, body_model, trial['betas'])
                kw.update(meas_targets=mt.tgt, meas_weights=mt.wt, trial_meas=tm, trial_meas_jac=tmj)
            step(state, trial, x, w, robust_sigma=sigma, pose_prior_weight=pw, betas_weight=bw, lambda_up=LM_UP,
                 lambda_down=LM_DOWN, first=it == 0, trial_keypoints=tkp, trial_jac=tjac, **kw)
    rot = state['rot']
    expr = state['expression'] if ne else None
    pr = {name: rot[:, j:j + n] for name, j, n in parts}
    with torch.no_grad():
        out = _forward_2d(body_model, rot[:, :1], rot[:, 1:22], state['betas'], state[last], intr, pr, expr)
        per_body = _kp2d_loss(out['proj_joints'], x, w, sigma, pw, rot, anchor, bw, state['betas'], jw, ew, expr)
        if mt is not None:      # _kp2d_loss already counted betas_weight |betas|^2
            per_body = per_body + mt.loss(state['meas'], state['betas'], 0.0)
        if intr is not None:
            per_body = _depth_rule(per_body, out['joints'][:], w)
    res = _kp_lm_result(state, last, keypoints=out['joints'][:], proj_joints=out['proj_joints'], loss=per_body)
    if parts:
        raw = rot[..., :2].reshape(B, 6 * n_rot)
        res['body_pose'], res['body_pose_mat'] = raw[:, 6:132].contiguous(), rot[:, 1:22]
        for name, j, n in parts:
            res[name] = raw[:, 6 * j:6 * (j + n)].contiguous()
    if wide:
        res['full_pose_mat'] = rot
    if ne:
        res['expression'] = state['expression']
    return res


# the pose parts past the body in SMPL-X's joint order (SMPLX.forward's names) and their joint counts
POSE_PARTS = (('jaw_pose', 1), ('leye_pose', 1), ('reye_pose', 1), ('left_hand_pose', 15), ('right_hand_pose', 15))
POSE_WIDTHS = (22, 23, 24, 25, 40, 55)
# the widest wide LM step: 55 rotations, 27 betas, 5 expression coefficients and the camera (or 16 and 16)
LM_WIDE_MAX_PARAMS = 200


def _parts_in(width):
    """The pose parts inside a pose width: [(name, first joint, joint count)]."""
    out, j = [], 22
    for name, n in POSE_PARTS:
        if j + n > width:
            break
        out.append((name, j, n))
        j += n
    return out


class _SortedBatch:
    """A batch sorted by group once: labels (B,) with group_plan's rules, or None for one group of every row.  order
    (B,), group_plan's stable sort, and inv its inverse; offsets (G + 1,) int32 on the CPU, group g the sorted rows
    [offsets[g], offsets[g + 1]); gidx (B,) each sorted row's group, first (G,) each group's first sorted row and
    counts (G,) its number of rows (float).  All but offsets on `device`."""

    def __init__(self, labels, B, device):
        if labels is None:
            order, offsets = torch.arange(B), torch.tensor([0, B] if B else [0], dtype=torch.int32)
        else:
            order, offsets = group_plan(labels, B)
        counts = (offsets[1:] - offsets[:-1]).long()
        self.G, self.offsets = offsets.numel() - 1, offsets
        self.order = _to_device(order, device)
        self.inv = torch.argsort(self.order)
        self.gidx = _to_device(torch.repeat_interleave(torch.arange(self.G), counts), device)
        self.first = _to_device(offsets[:-1].long(), device)
        self.counts = _to_device(counts.float(), device)

    def mean(self, betas):
        """Per group, the mean (G, NB) of the sorted rows' betas (B, NB), summed in row order: a group's start."""
        if self.G == 0:
            return betas.new_zeros(0, betas.shape[1])
        return (_group_sum(betas, self.offsets) / self.counts[:, None]).contiguous()


def _fit_keypoints_2d_groups(body_model, x, w, params, rot0, anchor, method, iterations, sigma, pw, bw, lr, groups,
                             body_measurements, measurements, measurement_weights, cd, share_pose=False):
    """fit_body_to_keypoints_2d with groups: the images sorted by group once, fitted, and returned in the caller's
    order; share_pose: the body pose per group too, anchor None or the caller's per-group anchor."""
    from . import ops
    from .autograd import Rot6dFunction
    device = x.device
    B, K = x.shape[0], x.shape[1]
    plan = _SortedBatch(groups, B, device)
    G, offsets, gidx, nb = plan.G, plan.offsets, plan.gidx, params['betas'].shape[1]
    x, w, rot0 = (t[plan.order].contiguous() for t in (x, w, rot0))
    sp = {k: v.detach()[plan.order].contiguous() for k, v in params.items()}
    betas0 = plan.mean(sp['betas'])
    if share_pose:
        raw0 = _shared_body_raw(rot0, offsets, plan.counts)
        body0 = ops.decode_rot6d(raw0) if G else rot0.new_zeros(0, 21, 3, 3)
        rot0 = torch.cat([rot0[:, :1], body0[gidx]], 1).contiguous()
        if anchor is None:
            anchor = torch.cat([rot0[plan.first, :1], body0], 1).contiguous()
        elif anchor.numel() != G * 22 * 9:
            raise ValueError(f'fit_body_to_keypoints_2d: with share_pose, pose_anchor must be ({G}, 22, 3, 3)')
        else:
            anchor = anchor.reshape(G, 22, 3, 3).contiguous()
    else:
        anchor = anchor[plan.order].contiguous()
    mt = _measurement_term(measurements, measurement_weights, G, device, body_measurements, cd)
    if method == 'lm':
        packed = body_model.packed(device)
        trial = {'rot': rot0.clone(), 'betas': betas0, 'image_betas': betas0[gidx].contiguous(),
                 'camera': sp['camera']}
        state = _kp_lm_state(B, K, 22, nb, 'camera', device, G)
        if mt is not None:
            state.update(mt.state(nb, device))
        pose_anchor = anchor if pw > 0 else None
        if B > 0:
            ws = (ops.fit_lm_shared_pose_workspace if share_pose else ops.fit_lm_groups_workspace)(B, G, 22, nb, device)
            step = ops.fit_lm_keypoints_2d_shared_pose_step if share_pose else ops.fit_lm_keypoints_2d_groups_step
            mstep = (ops.fit_lm_keypoints_2d_shared_pose_measurements_step if share_pose else
                     ops.fit_lm_keypoints_2d_groups_measurements_step)
            if mt is not None:
                mt.prime(body_model)
            for it in range(iterations + 1):
                tkp, tjac = ops.smplx_keypoint_jacobian(packed, trial['image_betas'], trial['rot'])
                if mt is None:
                    step(state, trial, x, w, sigma, pw, bw, LM_UP, LM_DOWN, it == 0, tkp, tjac, offsets, ws,
                         pose_anchor=pose_anchor)
                else:
                    tm, tmj = mt.trial(packed, body_model, trial['betas'])
                    mstep(state, trial, x, w, sigma, pw, bw, mt.tgt, mt.wt, LM_UP, LM_DOWN, it == 0, tkp, tjac, tm,
                          tmj, offsets, ws, pose_anchor=pose_anchor)
        rot = state['rot']
        with torch.no_grad():
            out = body_model(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=state['betas'][gidx],
                             camera=state['camera'], return_shaped=False)
        res = _kp_lm_result(state, 'camera', keypoints=out['joints'][:], proj_joints=out['proj_joints'],
                            loss=state['loss'])
        if share_pose:
            for k in ('body_pose', 'body_pose_mat'):
                res[k] = res[k][plan.first]
    else:
        p = {k: sp[k].clone().requires_grad_(True) for k in ('global_rot', 'body_pose', 'camera')}
        if share_pose:
            p['body_pose'] = raw0.clone().requires_grad_(True)
        p['betas'] = betas0.clone().requires_grad_(True)

        def loss_fn():
            grot = Rot6dFunction.apply(p['global_rot'])
            bpose = Rot6dFunction.apply(p['body_pose'])
            body = bpose[gidx] if share_pose else bpose
            out = body_model(global_rot=grot, body_pose=body, betas=p['betas'][gidx], camera=p['camera'],
                             return_shaped=False)
            if share_pose:      # the keypoint terms per image, the pose prior once per group
                per_group = _group_sum(_kp2d_loss(out['proj_joints'], x, w, sigma, 0.0, None, None, 0.0, None),
                                       offsets)
                if pw > 0:
                    per_group = per_group + 0.5 * pw * (bpose - anchor[:, 1:]).pow(2).sum((1, 2, 3))
            else:
                rot = torch.cat([grot, bpose], 1)
                per_group = _group_sum(_kp2d_loss(out['proj_joints'], x, w, sigma, pw, rot, anchor, 0.0, None),
                                       offsets)
            meas = None
            if mt is not None:
                meas = mt.measure(body_model, p['betas'])
                per_group = per_group + mt.loss(meas, p['betas'], 0.0)
            if bw > 0:
                per_group = per_group + bw * p['betas'].pow(2).sum(1)
            return per_group, out, grot, bpose, meas

        per_group, out, grot, bpose, meas = _adam(list(p.values()), lr, iterations, loss_fn)
        res = _adam_result(p, grot, bpose, meas, keypoints=out['joints'][:], proj_joints=out['proj_joints'],
                           loss=per_group)
    per_image = ('global_rot', 'camera', 'global_rot_mat', 'keypoints', 'proj_joints')
    for k in per_image if share_pose else per_image + ('body_pose', 'body_pose_mat'):
        res[k] = res[k][plan.inv]
    return res


def _shared_body_raw(rot0, offsets, cnt):
    """A group's starting body pose as raw 6D (G, 126): the image-order mean of its images' (sorted by group) rotations
    of joints 1 .., as the 6D decoder's input, its first two columns; the decoder's Gram-Schmidt makes it rotations."""
    G = offsets.numel() - 1
    if G == 0:
        return rot0.new_zeros(0, 6 * 21)
    mean = _group_sum(rot0[:, 1:], offsets) / cnt[:, None, None, None]
    return mean[..., :2].reshape(G, 6 * 21).contiguous()


# the global rotation of the regressor's mean pose (6D (1, 0, 0, -1, 0, 0)): upright and facing a y-down camera
MEAN_GLOBAL_ROT = ((1.0, 0.0, 0.0), (0.0, -1.0, 0.0), (0.0, 0.0, -1.0))
# the weight, relative to one ray, that keeps the default start of a calibrated fit near START_DEPTH along its first
# view's ray: it fixes the point along a single ray or parallel rays and moves a crossing by about 1e-6 of its distance
RAY_START_WEIGHT = 1e-6


def _root_joint(body_model, betas):
    """J_0(betas) (B, 3): the root joint of the shaped body, about which SMPL-X applies the global rotation (a few
    small products on any device: the start of a fit, not its hot path)."""
    with torch.no_grad():
        v = body_model.v_template + torch.einsum('bl,mkl->bmk', betas, body_model.shapedirs[..., :betas.shape[1]])
        return torch.einsum('m,bmk->bk', body_model.J_regressor[0].to(v.dtype), v)


def calibrated_start(body_model, global_rot_mat, transl, betas, cam_rot, cam_transl):
    """Maps a camera-frame start of one view into the world frame of a calibrated fit: global_rot_mat (B, 3, 3) and
    transl (B, 3) of a body in the frame of a camera with world-to-camera extrinsics cam_rot (B, 3, 3), cam_transl
    (B, 3), for example a perspective fit of that view or perspective_start of the regressor's crop camera; betas
    (B, NB).  SMPL-X rotates about the root joint J_0(betas), so the world start is R_0' = R_v^T R_0 and
    t' = R_v^T (J_0 + t - T_v) - J_0.  Returns (global_rot_mat', transl')."""
    f = lambda t: torch.as_tensor(t, dtype=torch.float32, device=body_model.shapedirs.device)  # noqa: E731
    R0, t, Rv, Tv = f(global_rot_mat).reshape(-1, 3, 3), f(transl).reshape(-1, 3), f(cam_rot), f(cam_transl)
    j0 = _root_joint(body_model, f(betas).reshape(R0.shape[0], -1).contiguous())
    Rt = Rv.reshape(-1, 3, 3).transpose(1, 2)
    return Rt @ R0, (Rt @ (j0 + t - Tv.reshape(-1, 3))[..., None])[..., 0] - j0


def _ray_start(x, w, intr, cam_rot, cam_transl, offsets):
    """The default world translation of each body of a calibrated fit (G, 3), without synchronising: the least-squares
    point nearest the rays of its views (sorted by body) through the centroids of their weighted keypoints (the
    principal point without one), plus RAY_START_WEIGHT times the squared distance to the point START_DEPTH in front of
    its first view on that view's ray.  Solved in float64."""
    keep = (w > 0)[..., None]
    c = torch.where(keep, x, torch.zeros_like(x)).sum(1) / keep.sum(1).clamp(min=1)
    c = torch.where(keep.any(1), c, intr[:, 1:])
    u = torch.cat([(c - intr[:, 1:]) / intr[:, :1], torch.ones_like(c[:, :1])], 1).double()   # the ray, camera frame
    Rt = cam_rot.double().transpose(1, 2)
    centre = -(Rt @ cam_transl.double()[..., None])[..., 0]
    d = (Rt @ u[..., None])[..., 0]
    d = d / d.norm(dim=1, keepdim=True)
    M = torch.eye(3, dtype=torch.float64, device=x.device) - d[:, :, None] * d[:, None, :]
    first = _to_device(offsets[:-1].long(), x.device)
    p0 = centre[first] + START_DEPTH * (Rt[first] @ u[first][..., None])[..., 0]
    eps = RAY_START_WEIGHT
    A = _group_sum(M, offsets) + eps * torch.eye(3, dtype=torch.float64, device=x.device)
    rhs = _group_sum((M @ centre[..., None])[..., 0], offsets) + eps * p0
    return torch.linalg.solve_ex(A, rhs)[0].float()


def _calibrated_loss(joints, x, w, intr, cam_rot, cam_transl, gidx, offsets, sigma, pw, bpose, anchor, bw, betas):
    """The calibrated fit's loss per body, through PerspectiveCamera(rotation=, translation=): joints (G, K, 3) in the
    world frame, the views (B, ...) sorted by body, gidx (B,) each view's body.  The keypoint terms per view summed in
    view order, + the pose prior once per body + betas_w |betas|^2.  Returns (per_body (G,), proj_joints (B, K, 2),
    behind (G,) bool: the step's depth rule, a weighted keypoint at Y_z <= 0 or not finite in one of the body's views,
    or a view whose focal length is not finite and > 0)."""
    from .human_shape.models.camera.camera_projection import PerspectiveCamera
    jv = joints[gidx]
    proj = PerspectiveCamera()(jv, focal_length=intr[:, 0], rotation=cam_rot, translation=cam_transl,
                               camera_center=intr[:, 1:])
    per_body = _group_sum(_kp2d_loss(proj, x, w, sigma, 0.0, None, None, 0.0, None), offsets)
    if pw > 0:
        per_body = per_body + 0.5 * pw * (bpose - anchor[:, 1:]).pow(2).sum((1, 2, 3))
    if bw > 0:
        per_body = per_body + bw * betas.pow(2).sum(1)
    y = torch.einsum('bji,bmi->bmj', cam_rot, jv.detach()) + cam_transl[:, None]
    f = intr[:, 0]
    behind = _depth_rule(torch.zeros_like(proj[:, 0, 0]), y, w).isinf() | ~(f > 0) | ~torch.isfinite(f)
    return per_body, proj, _group_sum(behind.float(), offsets) > 0


def fit_body_to_calibrated_views(body_model, keypoints2d, focal_length, principal_point, cam_rot, cam_transl,
                                 groups=None, weights=None, init=None, method='lm', iterations=None, robust_sigma=None,
                                 pose_prior_weight=0.0, betas_weight=0.0, pose_anchor=None, lr=0.05,
                                 body_measurements=None, measurements=None, measurement_weights=None,
                                 circumference_derivative='reference'):
    """Fits bodies seen by a synchronised rig of calibrated cameras: pose, shape and world translation of each body so
    that its keypoints, projected into every view that sees it, match `keypoints2d` (B, K, 2), one row per view.

    Each view v has intrinsics (focal_length a scalar or (B,), principal_point (2,) or (B, 2), as
    fit_body_to_keypoints_2d's) and world-to-camera extrinsics cam_rot (B, 3, 3), cam_transl (B, 3): Y = R_v X + T_v,
    camera frame x right, y down, z forward, p = f (Y_x / Y_z, Y_y / Y_z) + pp, X = joint + transl in the world frame.
    groups: None (every view sees one body) or (B,) labels 0 .. G-1 (group_plan's rules), the body each view sees.
    Loss per body: the sum over its views (in the caller's order) of sum_{w_k > 0} w_k rho(|p_k - x_k|^2), +
    pose_prior_weight / 2 sum_{j >= 1} |R_j - R0_j|_F^2, + the measurement terms of fit_body_to_keypoints_2d, +
    betas_weight |betas|^2; +inf for a body with a weighted keypoint behind one of its cameras, or with a view whose
    focal length is not finite and > 0 (the step's depth rule).  The baseline between
    the cameras fixes the body's metric size and position, which no single view does.  weights: None, (K,) or (B, K)
    per view.  init: per body, fit_body_to_keypoints' init with 'transl' in the world frame (calibrated_start maps a
    camera-frame start of one view); without a global rotation a body starts at the mean pose seen from its first view
    (R_0 = R_v^T MEAN_GLOBAL_ROT), without a translation at the least-squares point nearest the rays through its views'
    weighted-keypoint centroids.  pose_anchor (G, 22, 3, 3), by default the start.  method: 'lm' (per iteration the
    keypoint Jacobian of the G trial bodies and one ops.fit_lm_keypoints_2d_calibrated_step, two launches, four with
    measurements, no host synchronisation) or 'adam' (SMPLX.forward(transl=) and PerspectiveCamera(rotation=,
    translation=)).  iterations: None means 50 for LM and 600 for Adam.
    Returns per body {'global_rot', 'body_pose' (raw 6D), 'betas', 'transl', 'global_rot_mat' (G, 1, 3, 3),
    'body_pose_mat' (G, 21, 3, 3), 'keypoints' (G, K, 3) in the world frame, 'loss' (G,) recomputed through
    PerspectiveCamera}, with measurements 'measurements' (G, 5), and per view in the caller's order 'proj_joints'
    (B, K, 2)."""
    iterations, sigma = _check_kp_fit('fit_body_to_calibrated_views', body_model, method, iterations,
                                      circumference_derivative, body_measurements, measurements, robust_sigma,
                                      pose_prior_weight, betas_weight)
    from . import ops
    from .autograd import Rot6dFunction
    device = body_model.shapedirs.device
    x, w = _keypoints_2d('fit_body_to_calibrated_views', keypoints2d, weights, device)
    B, K = x.shape[0], x.shape[1]
    nb = body_model.num_betas
    intr = _intrinsics(focal_length, principal_point, B, device)
    R = torch.as_tensor(cam_rot, dtype=torch.float32, device=device)
    T = torch.as_tensor(cam_transl, dtype=torch.float32, device=device)
    if R.shape != (B, 3, 3) or T.shape != (B, 3):
        raise ValueError(f'fit_body_to_calibrated_views: cam_rot must be ({B}, 3, 3) and cam_transl ({B}, 3), got '
                         f'{tuple(R.shape)} and {tuple(T.shape)}')
    plan = _SortedBatch(groups, B, device)
    G, offsets, gidx = plan.G, plan.offsets, plan.gidx
    x, w, intr, R, T = (t[plan.order].contiguous() for t in (x, w, intr, R, T))
    init = _raw_init(init)
    if init.get('global_rot') is None:
        mean = torch.ones(3, device=device)          # MEAN_GLOBAL_ROT, filled on the device: no host-to-device copy
        mean[1:].fill_(-1.0)
        init['global_rot'] = (R[plan.first].transpose(1, 2) * mean)[..., :2].reshape(G, 6)
    if init.get('transl') is None:
        init['transl'] = _ray_start(x, w, intr, R, T, offsets) if G else torch.zeros(0, 3, device=device)
    params = _start_params(init, G, nb, device, method, 'transl')
    rot0, anchor = _start_rotations(params, pose_anchor, G)
    pw, bw = float(pose_prior_weight), float(betas_weight)
    mt = _measurement_term(measurements, measurement_weights, G, device, body_measurements, circumference_derivative)
    def loss(joints, bpose, betas):
        return _calibrated_loss(joints, x, w, intr, R, T, gidx, offsets, sigma, pw, bpose, anchor, bw, betas)
    if method == 'lm':
        state = _kp_lm_state(G, K, 22, nb, 'transl', device)
        if mt is not None:
            state.update(mt.state(nb, device))
        if G > 0:
            trial = {'rot': rot0.clone(), 'betas': params['betas'].contiguous(),
                     'transl': params['transl'].contiguous()}
            ext = torch.cat([R.reshape(B, 9), T], 1).contiguous()
            ws = ops.fit_lm_calibrated_workspace(B, G, device)
            packed = body_model.packed(device)
            pose_anchor = anchor if pw > 0 else None
            if mt is not None:
                mt.prime(body_model)
            for it in range(int(iterations) + 1):
                tkp, tjac = ops.smplx_keypoint_jacobian(packed, trial['betas'], trial['rot'])
                if mt is None:
                    ops.fit_lm_keypoints_2d_calibrated_step(state, trial, x, w, intr, ext, sigma, pw, bw, LM_UP,
                                                            LM_DOWN, it == 0, tkp, tjac, offsets, ws,
                                                            pose_anchor=pose_anchor)
                else:
                    tm, tmj = mt.trial(packed, body_model, trial['betas'])
                    ops.fit_lm_keypoints_2d_calibrated_measurements_step(
                        state, trial, x, w, intr, ext, sigma, pw, bw, mt.tgt, mt.wt, LM_UP, LM_DOWN, it == 0, tkp,
                        tjac, tm, tmj, offsets, ws, pose_anchor=pose_anchor)
        rot = state['rot']
        with torch.no_grad():
            out = body_model(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=state['betas'], transl=state['transl'],
                             return_shaped=False)
            joints = out['joints'][:]
            per_body, proj, behind = loss(joints, rot[:, 1:], state['betas'])
            if mt is not None:
                per_body = per_body + mt.loss(state['meas'], state['betas'], 0.0)
            per_body = torch.where(behind, torch.full_like(per_body, float('inf')), per_body)
        return _kp_lm_result(state, 'transl', keypoints=joints, proj_joints=proj[plan.inv], loss=per_body)

    def loss_fn():
        grot = Rot6dFunction.apply(params['global_rot'])
        bpose = Rot6dFunction.apply(params['body_pose'])
        out = body_model(global_rot=grot, body_pose=bpose, betas=params['betas'], transl=params['transl'],
                         return_shaped=False)
        joints = out['joints'][:]
        per_body, proj, behind = loss(joints, bpose, params['betas'])
        meas = None
        if mt is not None:
            meas = mt.measure(body_model, params['betas'])
            per_body = per_body + mt.loss(meas, params['betas'], 0.0)
        return per_body, joints, proj, grot, bpose, meas, behind

    per_body, joints, proj, grot, bpose, meas, behind = _adam(list(params.values()), lr, iterations, loss_fn)
    per_body = torch.where(behind, torch.full_like(per_body, float('inf')), per_body)
    return _adam_result(params, grot, bpose, meas, keypoints=joints, proj_joints=proj[plan.inv], loss=per_body)


def _smoothness(rot, transl, gidx, srw, stw):
    """Per frame (sorted by sequence) the smoothness term of the pair (t, t + 1), 0 for a sequence's last frame:
    srw / 2 sum_j |R_{t+1},j - R_t,j|_F^2 + stw |tau_{t+1} - tau_t|^2."""
    out = torch.zeros(rot.shape[0], dtype=rot.dtype, device=rot.device)
    if rot.shape[0] < 2 or not (srw > 0 or stw > 0):
        return out
    d = torch.zeros_like(out[1:])
    if srw > 0:
        d = d + 0.5 * srw * (rot[1:] - rot[:-1]).pow(2).sum((1, 2, 3))
    if stw > 0:
        d = d + stw * (transl[1:] - transl[:-1]).pow(2).sum(1)
    return torch.cat([torch.where(gidx[1:] == gidx[:-1], d, torch.zeros_like(d)), out[:1]])


def fit_body_to_sequence(body_model, keypoints2d, focal_length, principal_point, sequences=None, weights=None,
                         init=None, method='lm', iterations=None, robust_sigma=None, pose_prior_weight=0.0,
                         betas_weight=0.0, pose_anchor=None, smooth_rot_weight=0.0, smooth_transl_weight=0.0, lr=0.05):
    """Fits videos of one person filmed by one camera: per frame the pose and the camera-frame translation, per
    sequence one betas, with smoothness between consecutive frames, to the full-image 2D keypoints (B, K, 2) of every
    frame under a perspective camera with known intrinsics (focal_length a scalar or (B,), principal_point (2,) or
    (B, 2), as fit_body_to_keypoints_2d's; camera frame x right, y down, z forward).
    sequences: None (the whole batch is one sequence) or (B,) integer labels 0 .. S-1 (group_plan's rules); the frames
    of a label, in the caller's order, are that sequence in time order.  Loss per sequence: the sum over its frames of
    fit_body_to_keypoints_2d's perspective loss (keypoint term and pose prior), + smooth_rot_weight / 2 sum_{j >= 0}
    |R_{t+1},j - R_t,j|_F^2 (the global rotation included) + smooth_transl_weight |transl_{t+1} - transl_t|^2 over
    consecutive frames, + betas_weight |betas|^2; +inf when a frame has a weighted keypoint at Y_z <= 0.  The smoothness
    weights are in the targets' units: with pixel targets a 1 cm jump of the translation between two frames costs
    smooth_transl_weight * 1e-4 px^2, and a small rotation change of theta rad costs about smooth_rot_weight * theta^2
    px^2.  With both weights 0 this is the grouped perspective fit: one betas per sequence, independent frames.
    weights, init and pose_anchor (B, 22, 3, 3) are per frame; init as fit_body_to_keypoints_2d's perspective init
    ('transl', by default 3 m in front of the camera on the ray through the weighted keypoints' centroid), a sequence
    starts from the frame-order mean of its frames' init betas.  method: 'lm' (per iteration the keypoint Jacobian of
    every frame and ops.fit_lm_keypoints_2d_sequence_step, whose three launches solve the sequence's block-tridiagonal
    normal matrix exactly; no host synchronisation, every sequence's loss non-increasing) or 'adam' (SMPLX.forward
    (transl=), PerspectiveCamera and the smoothness terms in torch).  iterations: None means 50 for LM, 600 for Adam.
    Returns per sequence 'betas' (S, NB) and 'loss' (S,) (with 'lm' the step's fp64 loss of the final state), and per
    frame in the caller's order 'global_rot', 'body_pose' (raw 6D), 'transl', 'global_rot_mat', 'body_pose_mat',
    'keypoints' (B, K, 3) in the camera frame and 'proj_joints' (B, K, 2)."""
    iterations, sigma = _check_kp_fit('fit_body_to_sequence', body_model, method, iterations,
                                      robust_sigma=robust_sigma, pose_prior_weight=pose_prior_weight,
                                      betas_weight=betas_weight)
    srw, stw = float(smooth_rot_weight), float(smooth_transl_weight)
    if not (0 <= srw < float('inf') and 0 <= stw < float('inf')):
        raise ValueError('fit_body_to_sequence: the smoothness weights must be finite and >= 0')
    from . import ops
    from .autograd import Rot6dFunction
    device = body_model.shapedirs.device
    x, w = _keypoints_2d('fit_body_to_sequence', keypoints2d, weights, device)
    B, K = x.shape[0], x.shape[1]
    nb = body_model.num_betas
    intr = _intrinsics(focal_length, principal_point, B, device)
    params = _init_2d(init, B, nb, device, method, x, w, intr)
    rot0, anchor = _start_rotations(params, pose_anchor, B)
    pw, bw = float(pose_prior_weight), float(betas_weight)
    plan = _SortedBatch(sequences, B, device)
    S, offsets, gidx = plan.G, plan.offsets, plan.gidx
    x, w, intr, rot0, anchor = (t[plan.order].contiguous() for t in (x, w, intr, rot0, anchor))
    sp = {k: v.detach()[plan.order].contiguous() for k, v in params.items()}
    betas0 = plan.mean(sp['betas'])
    if method == 'lm':
        state = _kp_lm_state(B, K, 22, nb, 'transl', device, S)
        if B > 0:
            trial = {'rot': rot0.clone(), 'betas': betas0, 'image_betas': betas0[gidx].contiguous(),
                     'transl': sp['transl']}
            ws = ops.fit_lm_sequence_workspace(B, S, 22, nb, device)
            packed = body_model.packed(device)
            pose_anchor = anchor if pw > 0 else None
            for it in range(int(iterations) + 1):
                tkp, tjac = ops.smplx_keypoint_jacobian(packed, trial['image_betas'], trial['rot'])
                ops.fit_lm_keypoints_2d_sequence_step(state, trial, x, w, intr, sigma, pw, bw, srw, stw, LM_UP,
                                                      LM_DOWN, it == 0, tkp, tjac, offsets, ws,
                                                      pose_anchor=pose_anchor)
        rot = state['rot']
        with torch.no_grad():
            out = _forward_2d(body_model, rot[:, :1], rot[:, 1:], state['betas'][gidx], state['transl'], intr)
        # a start that breaks the depth rule leaves the kernel's loss NaN: its loss is +inf
        loss = torch.where(torch.isnan(state['loss']), torch.full_like(state['loss'], float('inf')), state['loss'])
        res = _kp_lm_result(state, 'transl', keypoints=out['joints'][:], proj_joints=out['proj_joints'], loss=loss)
    else:
        p = {k: sp[k].clone().requires_grad_(True) for k in ('global_rot', 'body_pose', 'transl')}
        p['betas'] = betas0.clone().requires_grad_(True)

        def loss_fn():
            grot = Rot6dFunction.apply(p['global_rot'])
            bpose = Rot6dFunction.apply(p['body_pose'])
            out = _forward_2d(body_model, grot, bpose, p['betas'][gidx], p['transl'], intr)
            rot = torch.cat([grot, bpose], 1)
            per_frame = _kp2d_loss(out['proj_joints'], x, w, sigma, pw, rot, anchor, 0.0, None) + \
                _smoothness(rot, p['transl'], gidx, srw, stw)
            per_seq = _group_sum(per_frame, offsets)
            if bw > 0:
                per_seq = per_seq + bw * p['betas'].pow(2).sum(1)
            return per_seq, out, grot, bpose

        per_seq, out, grot, bpose = _adam(list(p.values()), lr, iterations, loss_fn)
        joints = out['joints'][:]
        behind = _group_sum(_depth_rule(torch.zeros_like(x[:, 0, 0]), joints, w).isinf().float(), offsets) > 0
        res = _adam_result(p, grot, bpose, None, keypoints=joints, proj_joints=out['proj_joints'],
                           loss=torch.where(behind, torch.full_like(per_seq, float('inf')), per_seq))
    for k in ('global_rot', 'body_pose', 'transl', 'global_rot_mat', 'body_pose_mat', 'keypoints', 'proj_joints'):
        res[k] = res[k][plan.inv]
    return res


def main(argv=None):
    p = argparse.ArgumentParser(description='Fit SMPL-X betas to virtual measurements (batched, on the GPU)')
    src = p.add_mutually_exclusive_group(required=True)
    src.add_argument('--model-folder', type=str, help='folder with SMPLX_{GENDER}.{ext}')
    src.add_argument('--synthetic', action='store_true', help='the seeded synthetic SMPL-X model of shapy_b200.synth')
    p.add_argument('--gender', type=str, default='neutral')
    p.add_argument('--num-betas', dest='num_betas', type=int, default=10)
    p.add_argument('--ext', type=str, default='npz')
    p.add_argument('--height', type=float, default=1.80, help='height in metres')
    p.add_argument('--mass', type=float, default=-1, help='mass in kilograms')
    p.add_argument('--chest', type=float, default=-1, help='chest circumference in metres')
    p.add_argument('--waist', type=float, default=-1, help='waist circumference in metres')
    p.add_argument('--hips', type=float, default=-1, help='hips circumference in metres')
    p.add_argument('--targets', type=str, default=None,
                   help='npz with per-body arrays mass / height / chest / waist / hips (overrides the single targets); '
                        'with --keypoints-2d, the known measurements fitted together with the keypoints (the single '
                        'targets are not used there)')
    p.add_argument('--meas-definition-path', dest='meas_definition_path', type=str, default=None)
    p.add_argument('--meas-vertices-path', dest='meas_vertices_path', type=str, default=None)
    p.add_argument('--betas-weight', dest='betas_weight', type=float, default=0.0)
    p.add_argument('--method', choices=('adam', 'lm'), default='adam',
                   help='optimiser: Adam, or batched Levenberg-Marquardt on the measurement Jacobian')
    p.add_argument('--circumference-derivative', dest='circumference_derivative', choices=CIRCUMFERENCE_DERIVATIVES,
                   default='reference', help="how the circumferences are differentiated: the reference's autograd "
                                             "semantics, or their exact derivative")
    p.add_argument('--iterations', type=int, default=None, help='default 500 for adam, 50 for lm')
    p.add_argument('--lr', type=float, default=0.05, help='Adam step size (ignored by lm)')
    p.add_argument('--output', type=str, default='fit_betas.npz')
    p.add_argument('--keypoints-2d', dest='keypoints_2d', type=str, default=None,
                   help='npz with keypoints (B, K, 2) in the crop frame of proj_joints and optional weights (B, K), or '
                        'raw OpenPose detections openpose (B, 135, 3) in pixels with the crop descriptors center '
                        '(B, 2) and scale (B,) (and optionally crop_size, default 256; needs --keypoint-map): fit pose, '
                        'shape and camera to them instead of betas to measurements; with focal_length (and '
                        'principal_point, or image_size (W, H) for its centre) in the npz the keypoints and detections '
                        'are in pixels and the fit is perspective')
    p.add_argument('--keypoint-map', dest='keypoint_map', type=str, default=None,
                   help='JSON OpenPose -> model keypoint map (shapy_b200.keypoints2d), e.g. '
                        'tests/golden/openpose_smplx_map.json')
    p.add_argument('--init', type=str, default=None,
                   help='npz with raw_global_rot / raw_body_pose (or global_rot / body_pose raw 6D), betas and camera, '
                        'e.g. a saved regressor prediction; a perspective fit converts the camera with '
                        'perspective_start and the npz center / scale, or takes transl')
    p.add_argument('--robust-sigma', dest='robust_sigma', type=float, default=None)
    p.add_argument('--pose-prior-weight', dest='pose_prior_weight', type=float, default=0.0)
    p.add_argument('--pose-width', dest='pose_width', type=int, default=22, choices=POSE_WIDTHS,
                   help='with --keypoints-2d: rotations fitted, 22 (body), 25 (+ jaw and eyes) or 55 (+ hands)')
    p.add_argument('--fit-expression', dest='fit_expression', action='store_true',
                   help='with --keypoints-2d: also fit the facial expression')
    p.add_argument('--expression-weight', dest='expression_weight', type=float, default=0.0,
                   help='with --fit-expression: the regulariser weight on |expression|^2')
    p.add_argument('--share-pose', dest='share_pose', action='store_true',
                   help="with --keypoints-2d and a `groups` array: the images of a group are simultaneous views of "
                        "one posed body and share its body pose as well as its shape")
    p.add_argument('--calibrated', action='store_true',
                   help='with --keypoints-2d, a focal_length and cam_rot (B, 3, 3) / cam_transl (B, 3) in the npz: the '
                        'rows are views of a calibrated rig, fitted in its world frame (fit_body_to_calibrated_views); '
                        'an optional `groups` array labels the body each view sees')
    p.add_argument('--sequence', action='store_true',
                   help='with --keypoints-2d and a focal_length in the npz: the rows are the frames of videos of one '
                        'person filmed by one camera, in time order (fit_body_to_sequence); an optional `sequences` '
                        'array labels the video of each frame')
    p.add_argument('--smooth-rot', dest='smooth_rot', type=float, default=0.0,
                   help='with --sequence: the weight of |R_{t+1} - R_t|_F^2 / 2 between consecutive frames')
    p.add_argument('--smooth-transl', dest='smooth_transl', type=float, default=0.0,
                   help='with --sequence: the weight of |transl_{t+1} - transl_t|^2 between consecutive frames')
    a = p.parse_args(argv)
    if (a.pose_width != 22 or a.fit_expression or a.expression_weight) and \
            (not a.keypoints_2d or a.calibrated or a.sequence):
        raise SystemExit('--pose-width, --fit-expression and --expression-weight need --keypoints-2d and are not '
                         'supported with --calibrated or --sequence')

    from . import synth
    from .body_measurements import BodyMeasurements
    from .human_shape.models.body_models.body_models import SMPLX
    if a.synthetic:
        model = SMPLX(data_struct=synth.make_smplx())
    else:
        model = SMPLX(model_folder=a.model_folder, gender=a.gender, ext=a.ext, betas={'num': a.num_betas})
    model = model.cuda()
    if a.meas_definition_path and a.meas_vertices_path:
        cfg = {'meas_definition_path': a.meas_definition_path, 'meas_vertices_path': a.meas_vertices_path}
    else:
        cfg = {'landmarks': synth.load_landmarks()}
    targets = None
    if a.targets:
        d = np.load(a.targets)
        targets = {k: d[k].astype(np.float32) for k in NAMES if k in d.files}
    if a.keypoints_2d:      # known measurements only from --targets: --height has a default and is not used here
        return _main_keypoints_2d(a, model, BodyMeasurements(cfg).cuda() if targets else None, targets)
    bm = BodyMeasurements(cfg).cuda()
    if targets is None:
        targets = {k: getattr(a, k) for k in NAMES}
    res = fit_betas_to_measurements(model, bm, targets, betas_weight=a.betas_weight, iterations=a.iterations, lr=a.lr,
                                    method=a.method, circumference_derivative=a.circumference_derivative)
    meas = res['measurements'].cpu().numpy()
    np.savez(a.output, betas=res['betas'].cpu().numpy(), measurements=meas, names=np.array(NAMES),
             loss=res['loss'].cpu().numpy())
    print(json.dumps({'bodies': int(meas.shape[0]), 'output': a.output,
                      'first_body': {k: float(meas[0, i]) for i, k in enumerate(NAMES)}}))


def _main_keypoints_2d(a, model, bm, targets):
    d = np.load(a.keypoints_2d)
    persp = 'focal_length' in d.files
    focal = pp = None
    if persp:
        focal = d['focal_length'].astype(np.float32)
        if 'principal_point' in d.files:
            pp = d['principal_point'].astype(np.float32)
        elif 'image_size' in d.files:
            pp = d['image_size'].astype(np.float32).reshape(-1, 2) / 2.0
        else:
            raise SystemExit('--keypoints-2d with a focal_length needs principal_point or image_size (W, H)')
    if 'openpose' in d.files:
        from . import keypoints2d as k2d
        if not a.keypoint_map:
            raise SystemExit('--keypoints-2d with raw OpenPose detections needs --keypoint-map')
        kmap = k2d.load_keypoint_map(a.keypoint_map)
        op = k2d.threshold_confidence(d['openpose'].reshape(-1, k2d.NUM_OPENPOSE, 3), kmap)
        if not persp:       # the perspective fit takes the detections in pixels
            size = int(d['crop_size']) if 'crop_size' in d.files else 256
            op = k2d.to_crop(op, d['center'], d['scale'], size)
        x, w = k2d.map_keypoints(op, kmap, model.packed().K)
    else:
        x = d['keypoints'].astype(np.float32)
        x = x[None] if x.ndim == 2 else x
        w = d['weights'].astype(np.float32).reshape(x.shape[:2]) if 'weights' in d.files else None
    init = None
    if a.calibrated and not (persp and 'cam_rot' in d.files and 'cam_transl' in d.files):
        raise SystemExit('--calibrated needs focal_length, cam_rot and cam_transl in --keypoints-2d')
    if a.init and not a.calibrated:
        init = _load_init(a.init, x.shape[0], ('camera', 'transl', 'expression') + tuple(n for n, _ in POSE_PARTS))
        if persp and 'transl' not in init and 'camera' in init:
            if not ('center' in d.files and 'scale' in d.files):
                raise SystemExit('--init with a camera and a focal_length needs center and scale in --keypoints-2d')
            init['transl'] = perspective_start(init['camera'], d['center'], d['scale'], focal, pp)
    groups = d['groups'].astype(np.int64).reshape(-1) if 'groups' in d.files else None
    if a.calibrated:
        return _main_calibrated(a, model, bm, targets, d, x, w, focal, pp, groups)
    if a.sequence:
        return _main_sequence(a, model, d, x, w, focal, pp, init)
    res = fit_body_to_keypoints_2d(model, x, w, init=init, method=a.method, iterations=a.iterations,
                                   robust_sigma=a.robust_sigma, pose_prior_weight=a.pose_prior_weight,
                                   betas_weight=a.betas_weight, lr=a.lr, body_measurements=bm, measurements=targets,
                                   circumference_derivative=a.circumference_derivative, groups=groups,
                                   share_pose=a.share_pose, focal_length=focal, principal_point=pp,
                                   pose_width=a.pose_width, fit_expression=a.fit_expression,
                                   expression_weight=a.expression_weight)
    _save_result(a.output, res, {'bodies': int(x.shape[0])}, groups=groups)


def _load_init(path, n, last):
    """An --init npz as a fit's init of n rows: its raw 6D pose (raw_ entries first), betas and the `last` entries."""
    p = np.load(path)
    return {k: torch.as_tensor(p[k].astype(np.float32)).reshape(n, -1)
            for k in ('raw_global_rot', 'raw_body_pose', 'global_rot', 'body_pose', 'betas') + last
            if k in p.files and not (k in ('global_rot', 'body_pose') and 'raw_' + k in p.files)}


def _save_result(path, res, counts, **labels):
    """Saves a keypoint fit's result and the labels that are not None to the npz `path`, and prints its summary:
    `counts`, the path and the median loss, as one JSON line."""
    out = {k: v.detach().cpu().numpy() for k, v in res.items()}
    out.update({k: v for k, v in labels.items() if v is not None})
    np.savez(path, **out)
    print(json.dumps({**counts, 'output': path, 'median_loss': float(np.median(out['loss']))}))


def _main_calibrated(a, model, bm, targets, d, x, w, focal, pp, groups):
    """--keypoints-2d --calibrated: the per-body result (G rows) and each view's proj_joints (B rows, the npz's order).
    An --init npz is per body, with transl in the world frame."""
    G = int(groups.max()) + 1 if groups is not None and groups.size else 1
    init = _load_init(a.init, G, ('transl',)) if a.init else None
    res = fit_body_to_calibrated_views(model, x, focal, pp, d['cam_rot'].astype(np.float32),
                                       d['cam_transl'].astype(np.float32), groups=groups, weights=w, init=init,
                                       method=a.method, iterations=a.iterations, robust_sigma=a.robust_sigma,
                                       pose_prior_weight=a.pose_prior_weight, betas_weight=a.betas_weight, lr=a.lr,
                                       body_measurements=bm, measurements=targets,
                                       circumference_derivative=a.circumference_derivative)
    _save_result(a.output, res, {'bodies': int(res['loss'].shape[0]), 'views': int(x.shape[0])}, groups=groups)


def _main_sequence(a, model, d, x, w, focal, pp, init):
    """--keypoints-2d --sequence: per frame (B rows, the npz's order) and per sequence ('betas', 'loss') results."""
    if focal is None:
        raise SystemExit('--sequence needs focal_length in --keypoints-2d')
    seq = d['sequences'].astype(np.int64).reshape(-1) if 'sequences' in d.files else None
    res = fit_body_to_sequence(model, x, focal, pp, sequences=seq, weights=w, init=init, method=a.method,
                               iterations=a.iterations, robust_sigma=a.robust_sigma,
                               pose_prior_weight=a.pose_prior_weight, betas_weight=a.betas_weight,
                               smooth_rot_weight=a.smooth_rot, smooth_transl_weight=a.smooth_transl, lr=a.lr)
    _save_result(a.output, res, {'frames': int(x.shape[0]), 'sequences': int(res['loss'].shape[0])}, sequences=seq)


if __name__ == '__main__':
    main()
