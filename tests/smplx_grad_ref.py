"""Float64 reference gradients of the SMPL-X forward for the gradient tests.

forward_differentiable is oracle.smplx_oracle.smplx_forward_full with its inputs kept in the autograd graph (the
oracle detaches them), assembled from the oracle's own differentiable pieces (rigid_chain, dynamic_landmarks,
weak_persp).  tests/test_smplx_grad_cpu.py pins its gradients to the reference's own autograd
(tests/golden/ref_smplx_grad.npz) and its values to the oracle's.

Convention of shapy_b200's SMPLX.forward: transl is added to vertices and joints after the forward, and proj_joints
projects the joints before transl."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import smplx_oracle

LEAVES = ('betas', 'expression', 'rot', 'transl', 'camera')


def _opt(model, name):
    t = model.get(name)
    return None if t is None or (torch.is_tensor(t) and t.numel() == 0) else t


def forward_differentiable(model: dict, betas, rot, expression=None, use_face_contour=True, dtype=torch.float64):
    """smplx_forward_full (body_models.py:628-767) without transl or camera, differentiable in betas, rot (B, n_rot,
    3, 3) and expression.  The dynamic-contour row is picked through round / long and stays a constant, as in the
    reference.  Returns vertices, joints (before transl), v_shaped."""
    c = lambda t: t.cpu().to(dtype)  # noqa: E731
    B, n_rot = rot.shape[0], rot.shape[1]
    J_reg = c(model['J_regressor'])
    NJ = J_reg.shape[0]
    eye = torch.eye(3, dtype=dtype)
    full_pose = torch.cat([c(rot), eye.expand(B, NJ - n_rot, 3, 3)], dim=1)
    betas = c(betas)
    sd = c(model['shapedirs'])
    shapedirs, comps = sd, betas
    ed = _opt(model, 'expr_dirs')
    if ed is not None:
        e = torch.zeros(B, ed.shape[-1], dtype=dtype) if expression is None else c(expression)
        shapedirs = torch.cat([sd, c(ed)], dim=-1)
        comps = torch.cat([betas, e], dim=-1)
    v_template = c(model['v_template'])
    v_shaped_e = v_template + torch.einsum('bl,mkl->bmk', comps, shapedirs)
    J = torch.einsum('bik,ji->bjk', v_shaped_e, J_reg)
    pose_feature = (full_pose[:, 1:] - eye).reshape(B, -1)
    v_posed = v_shaped_e + torch.matmul(pose_feature, c(model['posedirs'])).view(B, -1, 3)
    posed_J, A = smplx_oracle.rigid_chain(full_pose, J, model['parents'])
    T = torch.einsum('vj,bjmn->bvmn', c(model['lbs_weights']), A)
    vertices = torch.matmul(T, F.pad(v_posed, [0, 1], value=1.0).unsqueeze(-1))[:, :, :3, 0]
    lf = torch.zeros(B, 0, dtype=torch.long)
    lb = torch.zeros(B, 0, 3, dtype=dtype)
    if _opt(model, 'lmk_faces_idx') is not None:
        lf = model['lmk_faces_idx'].unsqueeze(0).expand(B, -1)
        lb = c(model['lmk_bary_coords']).unsqueeze(0).expand(B, -1, -1)
    if use_face_contour and _opt(model, 'dynamic_lmk_faces_idx') is not None:
        df, db = smplx_oracle.dynamic_landmarks(full_pose.detach(), model['dynamic_lmk_faces_idx'],
                                                c(model['dynamic_lmk_bary_coords']), model['neck_kin_chain'])
        lf = torch.cat([lf, df], 1)
        lb = torch.cat([lb, db], 1)
    tri = model['faces_tensor'][lf]
    lv = torch.stack([vertices[b][tri[b]] for b in range(B)])
    joints = torch.cat([posed_J, (lv * lb.unsqueeze(-1)).sum(2)], dim=1)
    if _opt(model, 'extra_joint_regressor') is not None:
        reg = torch.einsum('ji,bik->bjk', c(model['extra_joint_regressor']), vertices)
        joints[:, model['source_idxs']] = reg[:, model['target_idxs']]
    v_shaped = v_template + torch.einsum('bl,mkl->bmk', betas, sd)
    return dict(vertices=vertices, joints=joints, v_shaped=v_shaped)


def pattern(golden, name, shape):
    """The closed-form cotangent `name` of ref_smplx_grad.npz (tools/make_golden.py, grad_pattern), float64."""
    names = [str(n) for n in golden['pattern_names']]
    f, ph, amp = golden['pattern'][names.index(name)]
    return amp * np.sin(f * np.arange(int(np.prod(shape)), dtype=np.float64) + ph).reshape(shape)


def oracle_grads(model, cot, betas, rot, expression=None, transl=None, camera=None, use_face_contour=True):
    """Gradients of sum_k <cot[k], out[k]> over out = vertices, joints, v_shaped, proj_joints (a missing cotangent is
    zero) with respect to the given inputs, in float64.  Returns ({input: grad}, {output: value})."""
    leaves = {k: torch.as_tensor(v).detach().double().clone().requires_grad_(True)
              for k, v in dict(betas=betas, rot=rot, expression=expression, transl=transl, camera=camera).items()
              if v is not None}
    out = forward_differentiable(model, leaves['betas'], leaves['rot'], expression=leaves.get('expression'),
                                 use_face_contour=use_face_contour)
    ys = dict(vertices=out['vertices'], joints=out['joints'], v_shaped=out['v_shaped'])
    if 'transl' in leaves:
        t = leaves['transl'].unsqueeze(1)
        ys['vertices'], ys['joints'] = ys['vertices'] + t, ys['joints'] + t
    if 'camera' in leaves:
        ys['proj_joints'] = smplx_oracle.weak_persp(out['joints'], leaves['camera'])
    loss = 0
    for k, y in ys.items():
        if cot.get(k) is not None:
            loss = loss + (torch.as_tensor(cot[k]).double() * y).sum()
    loss.backward()
    return {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in leaves.items()}, \
        {k: v.detach() for k, v in ys.items()}
