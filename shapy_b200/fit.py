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

    python -m shapy_b200.fit --synthetic --keypoints-2d kp.npz --init pred.npz --method lm --robust-sigma 0.05

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
    exact = exact_circumferences(circumference_derivative)
    if iterations is None:
        iterations = 500 if method == 'adam' else 50
    device = body_model.shapedirs.device
    B = batch_size or max([torch.as_tensor(v).numel() for v in targets.values()] + [1])
    if betas_init is not None:
        B = betas_init.shape[0]
    tgt, wt = _measurement_terms(targets, weights, B, device)
    faces = body_model.faces_i32
    if method == 'lm':
        return _fit_lm(body_model, body_measurements, tgt.contiguous(), wt.contiguous(), betas_weight, iterations,
                       betas_init, B, device, exact)
    nb = body_model.shapedirs.shape[-1]
    betas = (torch.zeros(B, nb, device=device) if betas_init is None else betas_init.detach().clone().float())
    betas.requires_grad_(True)
    opt = torch.optim.Adam([betas], lr=lr)
    # the step size decays geometrically to lr / 100 over the run, so the last iterations refine instead of orbiting
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda i: 0.01 ** (i / max(1, int(iterations))))

    def loss_fn(b):
        v = body_model.forward_shape(betas=b)['v_shaped']
        m = body_measurements.forward_vertices(v, faces, circumference_derivative)['measurements']
        meas = torch.stack([m[k]['tensor'] for k in NAMES], 1)
        return _measurement_loss(tgt, wt, meas, b, betas_weight), meas

    for _ in range(int(iterations)):
        opt.zero_grad(set_to_none=True)
        per_body, _ = loss_fn(betas)
        per_body.sum().backward()
        opt.step()
        sched.step()
    with torch.no_grad():
        per_body, meas = loss_fn(betas)
    return {'betas': betas.detach(), 'measurements': meas, 'loss': per_body}


# Levenberg-Marquardt damping: divided by LM_DOWN after an accepted step, multiplied by LM_UP after a rejected one
LM_UP, LM_DOWN = 10.0, 3.0
# parameters of one body the keypoint LM step takes (kLmKpMaxP of fit.cu): 22 rotations, the betas and the translation
LM_KP_MAX_PARAMS = 96


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


def _fit_lm(body_model, body_measurements, tgt, wt, betas_weight, iterations, betas_init, B, device, exact):
    from . import ops
    packed = body_model.packed(device)
    faces = body_model.faces_i32
    lm = body_measurements.landmarks()
    nb = packed.NB
    trial = (torch.zeros(B, nb, device=device) if betas_init is None
             else betas_init.detach().to(device=device, dtype=torch.float32).clone().contiguous())
    mk = lambda *s: torch.empty(*s, dtype=torch.float32, device=device)  # noqa: E731
    state = {'betas': mk(B, nb), 'meas': mk(B, 5), 'jac': mk(B, 5, nb), 'loss': mk(B), 'lambda': mk(B),
             'accepted': torch.zeros(B, dtype=torch.int32, device=device)}
    if B == 0:
        return {'betas': state['betas'], 'measurements': state['meas'], 'loss': state['loss']}
    ops.face_incidence(faces)          # built (one copy to the host) before the loop, which never synchronises
    for it in range(int(iterations) + 1):
        v = ops.smplx_forward_shape(packed, trial)
        meas, jac, _ = ops.measure_jacobian_betas(packed, lm, v, faces, exact=exact)
        ops.fit_lm_step(state, tgt, wt, betas_weight, LM_UP, LM_DOWN, it == 0, trial, meas, jac)
    return {'betas': state['betas'], 'measurements': state['meas'], 'loss': state['loss']}


IDENT6 = (1.0, 0.0, 0.0, 1.0, 0.0, 0.0)      # the 6D code of the identity rotation (row-major 3x2)


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
    if method not in ('adam', 'lm'):
        raise ValueError(f"method must be 'adam' or 'lm', got {method!r}")
    exact_circumferences(circumference_derivative)
    if measurements is not None and body_measurements is None:
        raise ValueError('fit_body_to_keypoints: measurements need body_measurements')
    if measurements is None and betas_weight != 0:
        raise ValueError('fit_body_to_keypoints: betas_weight needs measurements (the keypoint fit has no betas prior)')
    if not betas_weight >= 0:
        raise ValueError(f'fit_body_to_keypoints: betas_weight must be >= 0, got {betas_weight}')
    if method == 'lm' and 3 * 22 + body_model.num_betas + 3 > LM_KP_MAX_PARAMS:
        raise ValueError(f"fit_body_to_keypoints(method='lm'): 22 rotations, {body_model.num_betas} betas and the "
                         f'translation are {3 * 22 + body_model.num_betas + 3} parameters, at most {LM_KP_MAX_PARAMS} '
                         f'are supported (at most {LM_KP_MAX_PARAMS - 3 * 22 - 3} betas)')
    if iterations is None:
        iterations = 600 if method == 'adam' else 50
    from .autograd import Rot6dFunction
    device = body_model.shapedirs.device
    kp = torch.as_tensor(keypoints, dtype=torch.float32, device=device)
    B, K = kp.shape[0], kp.shape[1]
    w = torch.ones(K, device=device) if weights is None else torch.as_tensor(weights, dtype=torch.float32,
                                                                             device=device)
    w = w.expand(B, K).contiguous()
    mterms = None
    if measurements is not None:
        tgt, wt = _measurement_terms(measurements, measurement_weights, B, device)
        mterms = (tgt.contiguous(), wt.contiguous(), float(betas_weight), circumference_derivative)
    init = init or {}
    ident = torch.zeros(6, device=device)      # IDENT6, filled on the device: no host-to-device copy
    ident[0::3].fill_(1.0)
    start = {'global_rot': ident.repeat(B, 1), 'body_pose': ident.repeat(B, 21),
             'betas': torch.zeros(B, body_model.num_betas, device=device), 'transl': torch.zeros(B, 3, device=device)}
    params = {}
    for k, v in start.items():
        t = init.get(k)
        t = v if t is None else torch.as_tensor(t, dtype=torch.float32, device=device).reshape(v.shape)
        params[k] = t.detach().clone().contiguous().requires_grad_(method == 'adam')
    if method == 'lm':
        return _fit_keypoints_lm(body_model, kp, w, params, int(iterations), body_measurements, mterms)
    opt = torch.optim.Adam(list(params.values()), lr=lr)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda i: 0.01 ** (i / max(1, int(iterations))))

    def loss_fn():
        grot = Rot6dFunction.apply(params['global_rot'])
        bpose = Rot6dFunction.apply(params['body_pose'])
        out = body_model(global_rot=grot, body_pose=bpose, betas=params['betas'], transl=params['transl'],
                         return_shaped=False)
        joints = out['joints'][:]                  # the KeypointTensor's tensor, still in the graph
        per_body = ((joints - kp).pow(2).sum(-1) * w).sum(1)
        meas = None
        if mterms is not None:
            v = body_model.forward_shape(betas=params['betas'])['v_shaped']
            m = body_measurements.forward_vertices(v, body_model.faces_i32, mterms[3])['measurements']
            meas = torch.stack([m[k]['tensor'] for k in NAMES], 1)
            per_body = per_body + _measurement_loss(mterms[0], mterms[1], meas, params['betas'], mterms[2])
        return per_body, joints, grot, bpose, meas

    for _ in range(int(iterations)):
        opt.zero_grad(set_to_none=True)
        per_body = loss_fn()[0]
        per_body.sum().backward()
        opt.step()
        sched.step()
    with torch.no_grad():
        per_body, joints, grot, bpose, meas = loss_fn()
    res = {k: v.detach() for k, v in params.items()}
    res.update(global_rot_mat=grot, body_pose_mat=bpose, keypoints=joints, loss=per_body)
    if meas is not None:
        res['measurements'] = meas
    return res


def _fit_keypoints_lm(body_model, kp, w, params, iterations, body_measurements=None, mterms=None):
    from . import ops
    device = kp.device
    packed = body_model.packed(device)
    B, K = kp.shape[0], kp.shape[1]
    n_rot, nb = 22, params['betas'].shape[1]
    P = 3 * n_rot + nb + 3
    trial = {'rot': ops.decode_rot6d(torch.cat([params['global_rot'], params['body_pose']], 1)).contiguous(),
             'betas': params['betas'].contiguous(), 'transl': params['transl'].contiguous()}
    mk = lambda *s: torch.empty(*s, dtype=torch.float32, device=device)  # noqa: E731
    state = {'rot': mk(B, n_rot, 3, 3), 'betas': mk(B, nb), 'transl': mk(B, 3), 'keypoints': mk(B, K, 3),
             'jac': mk(B, 3 * K, P), 'loss': mk(B), 'lambda': mk(B),
             'accepted': torch.zeros(B, dtype=torch.int32, device=device)}
    tg = kp.contiguous()
    if mterms is not None:
        state.update(meas=mk(B, 5), meas_jac=mk(B, 5, nb))
    if B > 0 and mterms is None:
        for it in range(iterations + 1):
            tkp, tjac = ops.smplx_keypoint_jacobian(packed, trial['betas'], trial['rot'], trial['transl'])
            ops.fit_lm_keypoints_step(state, trial, tg, w, LM_UP, LM_DOWN, it == 0, tkp, tjac)
    elif B > 0:
        tgt, wt, rho, cd = mterms
        exact = exact_circumferences(cd)
        faces, lm = body_model.faces_i32, body_measurements.landmarks()
        ops.face_incidence(faces)          # built (one copy to the host) before the loop, which never synchronises
        for it in range(iterations + 1):
            tkp, tjac = ops.smplx_keypoint_jacobian(packed, trial['betas'], trial['rot'], trial['transl'])
            v = ops.smplx_forward_shape(packed, trial['betas'])
            tm, tmj, _ = ops.measure_jacobian_betas(packed, lm, v, faces, exact=exact)
            ops.fit_lm_keypoints_measurements_step(state, trial, tg, w, tgt, wt, rho, LM_UP, LM_DOWN, it == 0, tkp,
                                                   tjac, tm, tmj)
    rot = state['rot']
    with torch.no_grad():
        out = body_model(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=state['betas'], transl=state['transl'],
                         return_shaped=False)
        joints = out['joints'][:]
        per_body = ((joints - kp).pow(2).sum(-1) * w).sum(1)
        if mterms is not None:
            per_body = per_body + _measurement_loss(mterms[0], mterms[1], state['meas'], state['betas'], mterms[2])
    raw = rot[..., :2].reshape(B, n_rot * 6)       # the first two columns in the decoder's row-major 3x2 layout
    res = {'global_rot': raw[:, :6].contiguous(), 'body_pose': raw[:, 6:].contiguous(), 'betas': state['betas'],
           'transl': state['transl'], 'global_rot_mat': rot[:, :1], 'body_pose_mat': rot[:, 1:], 'keypoints': joints,
           'loss': per_body}
    if mterms is not None:
        res['measurements'] = state['meas']
    return res


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


def _kp2d_loss(proj, target, w, sigma, pose_w, rot, anchor, betas_w, betas):
    """The 2D fit's per-body loss: sum_{w_k > 0} w_k rho(|proj_k - target_k|^2) + pose_w / 2 sum_{j >= 1}
    |R_j - R0_j|_F^2 + betas_w |betas|^2, rho(e) = e (sigma None) or sigma^2 e / (sigma^2 + e)."""
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
    return per_body


def _init_2d(init, B, nb, device, method):
    """The raw 6D global and body pose, betas and camera to start from: fit_body_to_keypoints' init with 'camera' in
    place of 'transl'; the regressor's stage output (raw_global_rot, raw_body_pose, betas, camera) works as-is."""
    init = dict(init or {})
    for k in ('global_rot', 'body_pose'):
        if init.get('raw_' + k) is not None:
            init[k] = init['raw_' + k]
    ident = torch.zeros(6, device=device)      # IDENT6, filled on the device: no host-to-device copy
    ident[0::3].fill_(1.0)
    cam = torch.zeros(B, 3, device=device)     # scale softplus(0.9) ~ 1.24, the regressor's mean scale
    cam[:, 0].fill_(0.9)
    start = {'global_rot': ident.repeat(B, 1), 'body_pose': ident.repeat(B, 21),
             'betas': torch.zeros(B, nb, device=device), 'camera': cam}
    params = {}
    for k, v in start.items():
        t = init.get(k)
        t = v if t is None else torch.as_tensor(t, dtype=torch.float32, device=device).reshape(v.shape)
        params[k] = t.detach().clone().contiguous().requires_grad_(method == 'adam')
    return params


def fit_body_to_keypoints_2d(body_model, keypoints2d, weights=None, init=None, method='adam', iterations=None,
                             robust_sigma=None, pose_prior_weight=0.0, betas_weight=0.0, pose_anchor=None, lr=0.05):
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
    Returns {'global_rot', 'body_pose' (raw 6D), 'betas', 'camera', 'global_rot_mat' (B, 1, 3, 3), 'body_pose_mat'
    (B, 21, 3, 3), 'keypoints' (B, K, 3) and 'proj_joints' (B, K, 2) of the final parameters, 'loss' (B,)}."""
    if method not in ('adam', 'lm'):
        raise ValueError(f"method must be 'adam' or 'lm', got {method!r}")
    if robust_sigma is not None and not robust_sigma > 0:
        raise ValueError(f'fit_body_to_keypoints_2d: robust_sigma must be > 0 or None, got {robust_sigma}')
    if not (pose_prior_weight >= 0 and betas_weight >= 0):
        raise ValueError('fit_body_to_keypoints_2d: pose_prior_weight and betas_weight must be >= 0')
    nb = body_model.num_betas
    if method == 'lm' and 3 * 22 + nb + 3 > LM_KP_MAX_PARAMS:
        raise ValueError(f"fit_body_to_keypoints_2d(method='lm'): 22 rotations, {nb} betas and the camera are "
                         f'{3 * 22 + nb + 3} parameters, at most {LM_KP_MAX_PARAMS} are supported')
    if iterations is None:
        iterations = 600 if method == 'adam' else 50
    from . import ops
    from .autograd import Rot6dFunction
    device = body_model.shapedirs.device
    x = torch.as_tensor(keypoints2d, dtype=torch.float32, device=device).contiguous()
    if x.dim() != 3 or x.shape[2] != 2:
        raise ValueError(f'fit_body_to_keypoints_2d: keypoints2d must be (B, K, 2), got {tuple(x.shape)}')
    B, K = x.shape[0], x.shape[1]
    w = torch.ones(K, device=device) if weights is None else torch.as_tensor(weights, dtype=torch.float32,
                                                                             device=device)
    w = w.expand(B, K).contiguous()
    params = _init_2d(init, B, nb, device, method)
    rot0 = ops.decode_rot6d(torch.cat([params['global_rot'], params['body_pose']], 1).detach()).contiguous()
    anchor = rot0 if pose_anchor is None else torch.as_tensor(pose_anchor, dtype=torch.float32,
                                                              device=device).reshape(B, 22, 3, 3).contiguous()
    sigma = None if robust_sigma is None or robust_sigma == float('inf') else float(robust_sigma)
    pw, bw = float(pose_prior_weight), float(betas_weight)
    if method == 'lm':
        return _fit_keypoints_2d_lm(body_model, x, w, params, rot0, anchor, int(iterations), sigma, pw, bw)
    opt = torch.optim.Adam(list(params.values()), lr=lr)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda i: 0.01 ** (i / max(1, int(iterations))))

    def loss_fn():
        grot = Rot6dFunction.apply(params['global_rot'])
        bpose = Rot6dFunction.apply(params['body_pose'])
        out = body_model(global_rot=grot, body_pose=bpose, betas=params['betas'], camera=params['camera'],
                         return_shaped=False)
        rot = torch.cat([grot, bpose], 1)
        per_body = _kp2d_loss(out['proj_joints'], x, w, sigma, pw, rot, anchor, bw, params['betas'])
        return per_body, out, grot, bpose

    for _ in range(int(iterations)):
        opt.zero_grad(set_to_none=True)
        loss_fn()[0].sum().backward()
        opt.step()
        sched.step()
    with torch.no_grad():
        per_body, out, grot, bpose = loss_fn()
    res = {k: v.detach() for k, v in params.items()}
    res.update(global_rot_mat=grot, body_pose_mat=bpose, keypoints=out['joints'][:], proj_joints=out['proj_joints'],
               loss=per_body)
    return res


def _fit_keypoints_2d_lm(body_model, x, w, params, rot0, anchor, iterations, sigma, pw, bw):
    from . import ops
    device = x.device
    packed = body_model.packed(device)
    B, K = x.shape[0], x.shape[1]
    n_rot, nb = 22, params['betas'].shape[1]
    P = 3 * n_rot + nb + 3
    trial = {'rot': rot0.clone(), 'betas': params['betas'].contiguous(), 'camera': params['camera'].contiguous()}
    mk = lambda *s: torch.empty(*s, dtype=torch.float32, device=device)  # noqa: E731
    state = {'rot': mk(B, n_rot, 3, 3), 'betas': mk(B, nb), 'camera': mk(B, 3), 'keypoints': mk(B, K, 3),
             'jac': mk(B, 3 * K, P), 'loss': mk(B), 'lambda': mk(B),
             'accepted': torch.zeros(B, dtype=torch.int32, device=device)}
    if B > 0:
        for it in range(iterations + 1):
            tkp, tjac = ops.smplx_keypoint_jacobian(packed, trial['betas'], trial['rot'])
            ops.fit_lm_keypoints_2d_step(state, trial, x, w, sigma, pw, bw, LM_UP, LM_DOWN, it == 0, tkp, tjac,
                                         pose_anchor=anchor if pw > 0 else None)
    rot = state['rot']
    with torch.no_grad():
        out = body_model(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=state['betas'], camera=state['camera'],
                         return_shaped=False)
        per_body = _kp2d_loss(out['proj_joints'], x, w, sigma, pw, rot, anchor, bw, state['betas'])
    raw = rot[..., :2].reshape(B, n_rot * 6)       # the first two columns in the decoder's row-major 3x2 layout
    return {'global_rot': raw[:, :6].contiguous(), 'body_pose': raw[:, 6:].contiguous(), 'betas': state['betas'],
            'camera': state['camera'], 'global_rot_mat': rot[:, :1], 'body_pose_mat': rot[:, 1:],
            'keypoints': out['joints'][:], 'proj_joints': out['proj_joints'], 'loss': per_body}


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
                   help='npz with per-body arrays mass / height / chest / waist / hips (overrides the single targets)')
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
                        'shape and camera to them instead of betas to measurements')
    p.add_argument('--keypoint-map', dest='keypoint_map', type=str, default=None,
                   help='JSON OpenPose -> model keypoint map (shapy_b200.keypoints2d), e.g. '
                        'tests/golden/openpose_smplx_map.json')
    p.add_argument('--init', type=str, default=None,
                   help='npz with raw_global_rot / raw_body_pose (or global_rot / body_pose raw 6D), betas and camera, '
                        'e.g. a saved regressor prediction')
    p.add_argument('--robust-sigma', dest='robust_sigma', type=float, default=None)
    p.add_argument('--pose-prior-weight', dest='pose_prior_weight', type=float, default=0.0)
    a = p.parse_args(argv)

    from . import synth
    from .body_measurements import BodyMeasurements
    from .human_shape.models.body_models.body_models import SMPLX
    if a.synthetic:
        model = SMPLX(data_struct=synth.make_smplx())
    else:
        model = SMPLX(model_folder=a.model_folder, gender=a.gender, ext=a.ext, betas={'num': a.num_betas})
    model = model.cuda()
    if a.keypoints_2d:
        return _main_keypoints_2d(a, model)
    if a.meas_definition_path and a.meas_vertices_path:
        cfg = {'meas_definition_path': a.meas_definition_path, 'meas_vertices_path': a.meas_vertices_path}
    else:
        cfg = {'landmarks': synth.load_landmarks()}
    bm = BodyMeasurements(cfg).cuda()
    if a.targets:
        d = np.load(a.targets)
        targets = {k: d[k].astype(np.float32) for k in NAMES if k in d.files}
    else:
        targets = {k: getattr(a, k) for k in NAMES}
    res = fit_betas_to_measurements(model, bm, targets, betas_weight=a.betas_weight, iterations=a.iterations, lr=a.lr,
                                    method=a.method, circumference_derivative=a.circumference_derivative)
    meas = res['measurements'].cpu().numpy()
    np.savez(a.output, betas=res['betas'].cpu().numpy(), measurements=meas, names=np.array(NAMES),
             loss=res['loss'].cpu().numpy())
    print(json.dumps({'bodies': int(meas.shape[0]), 'output': a.output,
                      'first_body': {k: float(meas[0, i]) for i, k in enumerate(NAMES)}}))


def _main_keypoints_2d(a, model):
    d = np.load(a.keypoints_2d)
    if 'openpose' in d.files:
        from . import keypoints2d as k2d
        if not a.keypoint_map:
            raise SystemExit('--keypoints-2d with raw OpenPose detections needs --keypoint-map')
        kmap = k2d.load_keypoint_map(a.keypoint_map)
        op = k2d.threshold_confidence(d['openpose'].reshape(-1, k2d.NUM_OPENPOSE, 3), kmap)
        size = int(d['crop_size']) if 'crop_size' in d.files else 256
        x, w = k2d.map_keypoints(k2d.to_crop(op, d['center'], d['scale'], size), kmap, model.packed().K)
    else:
        x = d['keypoints'].astype(np.float32)
        x = x[None] if x.ndim == 2 else x
        w = d['weights'].astype(np.float32).reshape(x.shape[:2]) if 'weights' in d.files else None
    init = None
    if a.init:
        p = np.load(a.init)
        init = {k: torch.as_tensor(p[k].astype(np.float32)).reshape(x.shape[0], -1)
                for k in ('raw_global_rot', 'raw_body_pose', 'global_rot', 'body_pose', 'betas', 'camera')
                if k in p.files and not (k in ('global_rot', 'body_pose') and 'raw_' + k in p.files)}
    res = fit_body_to_keypoints_2d(model, x, w, init=init, method=a.method, iterations=a.iterations,
                                   robust_sigma=a.robust_sigma, pose_prior_weight=a.pose_prior_weight,
                                   betas_weight=a.betas_weight, lr=a.lr)
    out = {k: v.detach().cpu().numpy() for k, v in res.items()}
    np.savez(a.output, **out)
    print(json.dumps({'bodies': int(x.shape[0]), 'output': a.output, 'median_loss': float(np.median(out['loss']))}))


if __name__ == '__main__':
    main()
