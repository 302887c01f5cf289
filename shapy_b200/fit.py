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
loss.  keypoint_jacobian(body_model, rot, betas, transl) exposes the Jacobian itself.
"""
import argparse
import json

import numpy as np
import torch

NAMES = ('mass', 'height', 'chest', 'waist', 'hips')
DEFAULT_WEIGHTS = {'height': 100.0, 'mass': 1.0, 'chest': 2000.0, 'waist': 1000.0, 'hips': 1000.0}


def _targets(targets, B, device):
    out = {}
    for k in NAMES:
        v = targets.get(k, -1.0)
        t = torch.as_tensor(v, dtype=torch.float32, device=device).reshape(-1)
        out[k] = t.expand(B).contiguous() if t.numel() == 1 else t
        if out[k].numel() != B:
            raise ValueError(f'target `{k}` has {out[k].numel()} values for {B} bodies')
    return out


def fit_betas_to_measurements(body_model, body_measurements, targets, weights=None, betas_weight=0.0, iterations=None,
                              lr=0.05, betas_init=None, batch_size=None, method='adam'):
    """Fits betas (B, NB) so that the model's T-pose measurements match `targets`.

    body_model: shapy_b200 SMPLX (its forward_shape and faces are used); body_measurements: shapy_b200
    BodyMeasurements on the same device.  targets: {name: float or (B,) values} for mass [kg], height, chest, waist,
    hips [m]; a missing name or a value <= 0 drops that term.  batch_size: B when every target is a scalar (default 1).
    method: 'adam' (the default) or 'lm' (Levenberg-Marquardt, see the top; `lr` is ignored).  iterations: None means
    500 for Adam and 50 for LM.
    Returns {'betas': (B, NB), 'measurements': (B, 5) of the final betas (mass, height, chest, waist, hips),
    'loss': (B,) final per-body loss}."""
    if method not in ('adam', 'lm'):
        raise ValueError(f"method must be 'adam' or 'lm', got {method!r}")
    if iterations is None:
        iterations = 500 if method == 'adam' else 50
    device = body_model.shapedirs.device
    B = batch_size or max([torch.as_tensor(v).numel() for v in targets.values()] + [1])
    if betas_init is not None:
        B = betas_init.shape[0]
    tg = _targets(targets, B, device)
    w = dict(DEFAULT_WEIGHTS, **(weights or {}))
    # per-body weight: 0 where the target is <= 0 or the weight is <= 1e-3 (fit_measurements.py:111-133)
    wt = torch.stack([torch.where(tg[k] > 0, torch.full_like(tg[k], w[k]), torch.zeros_like(tg[k]))
                      if w[k] > 1e-3 else torch.zeros_like(tg[k]) for k in NAMES], 1)
    tgt = torch.stack([tg[k].clamp(min=0) for k in NAMES], 1)
    faces = body_model.faces_i32
    if method == 'lm':
        return _fit_lm(body_model, body_measurements, tgt.contiguous(), wt.contiguous(), betas_weight, iterations,
                       betas_init, B, device)
    nb = body_model.shapedirs.shape[-1]
    betas = (torch.zeros(B, nb, device=device) if betas_init is None else betas_init.detach().clone().float())
    betas.requires_grad_(True)
    opt = torch.optim.Adam([betas], lr=lr)
    # the step size decays geometrically to lr / 100 over the run, so the last iterations refine instead of orbiting
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda i: 0.01 ** (i / max(1, int(iterations))))

    def loss_fn(b):
        v = body_model.forward_shape(betas=b)['v_shaped']
        m = body_measurements.forward_vertices(v, faces)['measurements']
        meas = torch.stack([m[k]['tensor'] for k in NAMES], 1)
        diff = torch.where(wt > 0, tgt - meas, torch.zeros_like(meas))    # a dropped term passes no (NaN) gradient
        per_body = (wt * diff.pow(2)).sum(1) + betas_weight * b.pow(2).sum(1)
        return per_body, meas

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


def measurement_jacobian(body_model, body_measurements, betas):
    """The measurements of forward_shape(betas) and their Jacobian with respect to betas, without autograd:
    {'measurements': (B, 5) (mass, height, chest, waist, hips, bit-identical to BodyMeasurements.forward_vertices),
    'jacobian': (B, 5, NB)}.  The Jacobian has the semantics of the measurements' backward (constant barycentrics, no
    gradient through the plane heights); a NaN circumference gives a NaN row."""
    from . import ops
    betas = torch.as_tensor(betas, dtype=torch.float32, device=body_model.shapedirs.device).detach().contiguous()
    packed = body_model.packed(betas.device)
    v = ops.smplx_forward_shape(packed, betas)
    out, jac, status = ops.measure_jacobian_betas(packed, body_measurements.landmarks(), v, body_model.faces_i32)
    body_measurements.last_status = status
    return {'measurements': out, 'jacobian': jac}


def _fit_lm(body_model, body_measurements, tgt, wt, betas_weight, iterations, betas_init, B, device):
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
        meas, jac, _ = ops.measure_jacobian_betas(packed, lm, v, faces)
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


def fit_body_to_keypoints(body_model, keypoints, weights=None, iterations=None, lr=0.05, init=None, method='adam'):
    """Fits pose and shape so that the model's keypoints match `keypoints` (B, K, 3), K = body_model's keypoint count.

    weights: None (all 1), (K,) or (B, K) per-keypoint weights.  init: optional {'global_rot': (B, 6),
    'body_pose': (B, 126) raw 6D, 'betas': (B, NB), 'transl': (B, 3)}; a missing entry starts at the identity pose,
    zero betas or zero transl.  method: 'adam' (the default: the step size decays geometrically from lr to lr / 100)
    or 'lm' (batched Levenberg-Marquardt on the keypoint Jacobian, see the top; `lr` is ignored, a keypoint with
    weight <= 0 is dropped).  iterations: None means 600 for Adam and 50 for LM.
    Returns {'global_rot', 'body_pose' (raw 6D), 'betas', 'transl', 'global_rot_mat' (B, 1, 3, 3),
    'body_pose_mat' (B, 21, 3, 3), 'keypoints' (B, K, 3) of the final parameters, 'loss' (B,) final per-body loss}."""
    if method not in ('adam', 'lm'):
        raise ValueError(f"method must be 'adam' or 'lm', got {method!r}")
    if iterations is None:
        iterations = 600 if method == 'adam' else 50
    from .autograd import Rot6dFunction
    device = body_model.shapedirs.device
    kp = torch.as_tensor(keypoints, dtype=torch.float32, device=device)
    B, K = kp.shape[0], kp.shape[1]
    w = torch.ones(K, device=device) if weights is None else torch.as_tensor(weights, dtype=torch.float32,
                                                                             device=device)
    w = w.expand(B, K).contiguous()
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
        return _fit_keypoints_lm(body_model, kp, w, params, int(iterations))
    opt = torch.optim.Adam(list(params.values()), lr=lr)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda i: 0.01 ** (i / max(1, int(iterations))))

    def loss_fn():
        grot = Rot6dFunction.apply(params['global_rot'])
        bpose = Rot6dFunction.apply(params['body_pose'])
        out = body_model(global_rot=grot, body_pose=bpose, betas=params['betas'], transl=params['transl'],
                         return_shaped=False)
        joints = out['joints'][:]                  # the KeypointTensor's tensor, still in the graph
        per_body = ((joints - kp).pow(2).sum(-1) * w).sum(1)
        return per_body, joints, grot, bpose

    for _ in range(int(iterations)):
        opt.zero_grad(set_to_none=True)
        per_body = loss_fn()[0]
        per_body.sum().backward()
        opt.step()
        sched.step()
    with torch.no_grad():
        per_body, joints, grot, bpose = loss_fn()
    res = {k: v.detach() for k, v in params.items()}
    res.update(global_rot_mat=grot, body_pose_mat=bpose, keypoints=joints, loss=per_body)
    return res


def _fit_keypoints_lm(body_model, kp, w, params, iterations):
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
    if B > 0:
        for it in range(iterations + 1):
            tkp, tjac = ops.smplx_keypoint_jacobian(packed, trial['betas'], trial['rot'], trial['transl'])
            ops.fit_lm_keypoints_step(state, trial, tg, w, LM_UP, LM_DOWN, it == 0, tkp, tjac)
    rot = state['rot']
    with torch.no_grad():
        out = body_model(global_rot=rot[:, :1], body_pose=rot[:, 1:], betas=state['betas'], transl=state['transl'],
                         return_shaped=False)
        joints = out['joints'][:]
        per_body = ((joints - kp).pow(2).sum(-1) * w).sum(1)
    raw = rot[..., :2].reshape(B, n_rot * 6)       # the first two columns in the decoder's row-major 3x2 layout
    return {'global_rot': raw[:, :6].contiguous(), 'body_pose': raw[:, 6:].contiguous(), 'betas': state['betas'],
            'transl': state['transl'], 'global_rot_mat': rot[:, :1], 'body_pose_mat': rot[:, 1:], 'keypoints': joints,
            'loss': per_body}


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
    p.add_argument('--iterations', type=int, default=None, help='default 500 for adam, 50 for lm')
    p.add_argument('--lr', type=float, default=0.05, help='Adam step size (ignored by lm)')
    p.add_argument('--output', type=str, default='fit_betas.npz')
    a = p.parse_args(argv)

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
    bm = BodyMeasurements(cfg).cuda()
    if a.targets:
        d = np.load(a.targets)
        targets = {k: d[k].astype(np.float32) for k in NAMES if k in d.files}
    else:
        targets = {k: getattr(a, k) for k in NAMES}
    res = fit_betas_to_measurements(model, bm, targets, betas_weight=a.betas_weight, iterations=a.iterations, lr=a.lr,
                                    method=a.method)
    meas = res['measurements'].cpu().numpy()
    np.savez(a.output, betas=res['betas'].cpu().numpy(), measurements=meas, names=np.array(NAMES),
             loss=res['loss'].cpu().numpy())
    print(json.dumps({'bodies': int(meas.shape[0]), 'output': a.output,
                      'first_body': {k: float(meas[0, i]) for i, k in enumerate(NAMES)}}))


if __name__ == '__main__':
    main()
