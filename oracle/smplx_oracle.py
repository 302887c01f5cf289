"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference SMPL-X body model.

Pinned by tests/test_oracle_pins.py against (a) the reference's own lbs.py run in the
build container (tests/golden/ref_smplx.npz, written by tools/make_golden.py) and
(b) img_00.npz for the 6D decoder and the camera.  Real-weights parity of lbs()
itself is UNPINNED (the licensed SMPL-X file is not in the reference repo).

smplx_forward_full is the same forward for any pose prefix, expression and transl, in any
dtype (float64 by default); tests/golden/ref_smplx_full.npz pins it to the reference's own
lbs() run in float64.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may import this.
Plain torch-on-CPU, written op by op after:

  decode_6d          regressor/human_shape/models/common/pose_utils.py:138-153
  lbs chain          regressor/human_shape/models/body_models/lbs.py:99-196, 199-295
  transform_mat      regressor/human_shape/models/body_models/utils.py:14-24
  dynamic landmarks  lbs.py:20-49, rot_mat_to_euler utils/rotation_utils.py:86-92
  landmarks          lbs.py:52-94
  SMPLX.forward glue body_models.py:628-767 (smplx_forward: identity hands/jaw/eyes, zero
                     expression; J14 overwrite 738-744, transl 746-748, v_shaped recomputed
                     without expression 763-765)
  camera             models/camera/camera_projection.py:181-213, iterative_regressor.py:715-728
"""
import math

import torch
import torch.nn.functional as F


def decode_6d(x: torch.Tensor) -> torch.Tensor:
    """(B, 6n) -> (B, n, 3, 3).  The 6 numbers are a row-major 3x2 matrix."""
    B = x.shape[0]
    m = x.reshape(-1, 3, 2)
    a1, a2 = m[:, :, 0], m[:, :, 1]
    b1 = a1 / a1.norm(dim=1, keepdim=True).clamp_min(1e-12)
    d = (b1 * a2).sum(1, keepdim=True)
    u = a2 - d * b1
    b2 = u / u.norm(dim=1, keepdim=True).clamp_min(1e-12)
    b3 = torch.linalg.cross(b1, b2, dim=1)
    return torch.stack([b1, b2, b3], dim=-1).reshape(B, -1, 3, 3)


def full_pose_of(global_rot, body_pose):
    B = global_rot.shape[0]
    eye = torch.eye(3, dtype=global_rot.dtype).view(1, 1, 3, 3)
    # [global, body(21), jaw, leye, reye, lhand(15), rhand(15)]  body_models.py:687-690
    return torch.cat([global_rot, body_pose, eye.expand(B, 33, 3, 3)], dim=1)


def rigid_chain(rot_mats, J, parents):
    """batch_rigid_transform (lbs.py:242-295) without TorchScript."""
    B, N = rot_mats.shape[:2]
    rel = J.clone()
    rel[:, 1:] = J[:, 1:] - J[:, parents[1:]]
    T = torch.zeros(B, N, 4, 4, dtype=J.dtype)
    T[:, :, :3, :3] = rot_mats
    T[:, :, :3, 3] = rel
    T[:, :, 3, 3] = 1
    chain = [T[:, 0]]
    for i in range(1, N):
        chain.append(torch.bmm(chain[int(parents[i])], T[:, i]))
    G = torch.stack(chain, dim=1)
    posed = G[:, :, :3, 3].clone()
    Jh = F.pad(J, [0, 1], value=0.0).unsqueeze(-1)
    A = G.clone()
    A[:, :, :, 3] = G[:, :, :, 3] - torch.matmul(G, Jh)[..., 0]
    return posed, A


def dynamic_landmarks(full_pose, dyn_faces, dyn_bary, neck_kin_chain):
    rel = torch.eye(3, dtype=full_pose.dtype).expand(full_pose.shape[0], 3, 3)
    for idx in neck_kin_chain.tolist():
        rel = torch.matmul(full_pose[:, idx], rel)
    sy = torch.sqrt(rel[:, 0, 0] * rel[:, 0, 0] + rel[:, 1, 0] * rel[:, 1, 0])
    ang = torch.atan2(-rel[:, 2, 0], sy)
    y = torch.round(torch.clamp(-ang * 180.0 / math.pi, max=39)).long()
    neg = (y < 0).long()
    big = (y < -39).long()
    negv = big * 78 + (1 - big) * (39 - y)
    y = neg * negv + (1 - neg) * y
    return dyn_faces[y], dyn_bary[y]


def smplx_forward(model: dict, betas, global_rot, body_pose) -> dict:
    full_pose = full_pose_of(global_rot, body_pose)
    return smplx_forward_full(model, betas, full_pose, dtype=betas.dtype)


def _opt(model, name):
    t = model.get(name)
    return None if t is None or (torch.is_tensor(t) and t.numel() == 0) else t


def smplx_forward_full(model: dict, betas, rot, expression=None, transl=None, camera=None, dtype=torch.float64,
                       use_face_contour=True) -> dict:
    """The whole SMPL-X forward (body_models.py:628-767) in `dtype`, for any model dict with the reference's buffer
    names (optional buffers may be missing: expr_dirs, static / dynamic landmarks, the J14 regressor).

    rot (B, n_rot, 3, 3): rotations of the first n_rot joints of the full pose, in the reference's order
    [global, body(21), jaw, leye, reye, lhand(15), rhand(15)]; the remaining joints are identity.  `expression`
    enters the blend shapes and the joints, never v_shaped (763-765).  `transl` is added to vertices and joints after
    the J14 overwrite.  With `camera` (B, 3), proj_joints is the weak-perspective projection of the returned joints."""
    c = lambda t: t.detach().cpu().to(dtype)  # noqa: E731
    B, n_rot = rot.shape[0], rot.shape[1]
    J_reg = c(model['J_regressor'])
    NJ = J_reg.shape[0]
    eye = torch.eye(3, dtype=dtype)
    full_pose = torch.cat([c(rot), eye.expand(B, NJ - n_rot, 3, 3)], dim=1)
    betas = c(betas)
    sd = c(model['shapedirs'])
    ed = _opt(model, 'expr_dirs')
    shapedirs, comps = sd, betas
    if ed is not None:
        NE = ed.shape[-1]
        e = torch.zeros(B, NE, dtype=dtype) if expression is None else c(expression)
        shapedirs = torch.cat([sd, c(ed)], dim=-1)
        comps = torch.cat([betas, e], dim=-1)
    v_template = c(model['v_template'])
    v_shaped_e = v_template + torch.einsum('bl,mkl->bmk', comps, shapedirs)
    J = torch.einsum('bik,ji->bjk', v_shaped_e, J_reg)
    pose_feature = (full_pose[:, 1:] - eye).reshape(B, -1)
    v_posed = v_shaped_e + torch.matmul(pose_feature, c(model['posedirs'])).view(B, -1, 3)
    posed_J, A = rigid_chain(full_pose, J, model['parents'])
    T = torch.einsum('vj,bjmn->bvmn', c(model['lbs_weights']), A)
    vh = F.pad(v_posed, [0, 1], value=1.0).unsqueeze(-1)
    vertices = torch.matmul(T, vh)[:, :, :3, 0]
    # landmarks: static, then the dynamic contour row picked by the neck chain's rotation
    lf = torch.zeros(B, 0, dtype=torch.long)
    lb = torch.zeros(B, 0, 3, dtype=dtype)
    if _opt(model, 'lmk_faces_idx') is not None:
        lf = model['lmk_faces_idx'].unsqueeze(0).expand(B, -1)
        lb = c(model['lmk_bary_coords']).unsqueeze(0).expand(B, -1, -1)
    if use_face_contour and _opt(model, 'dynamic_lmk_faces_idx') is not None:
        df, db = dynamic_landmarks(full_pose, model['dynamic_lmk_faces_idx'], c(model['dynamic_lmk_bary_coords']),
                                   model['neck_kin_chain'])
        lf = torch.cat([lf, df], 1)
        lb = torch.cat([lb, db], 1)
    tri = model['faces_tensor'][lf]                     # (B, L, 3)
    lv = torch.stack([vertices[b][tri[b]] for b in range(B)])   # (B, L, 3, 3)
    landmarks = (lv * lb.unsqueeze(-1)).sum(2)
    joints = torch.cat([posed_J, landmarks], dim=1)
    if _opt(model, 'extra_joint_regressor') is not None:
        reg = torch.einsum('ji,bik->bjk', c(model['extra_joint_regressor']), vertices)
        joints[:, model['source_idxs']] = reg[:, model['target_idxs']]
    if transl is not None:
        joints = joints + c(transl).unsqueeze(1)
        vertices = vertices + c(transl).unsqueeze(1)
    v_shaped = v_template + torch.einsum('bl,mkl->bmk', betas, sd)
    out = dict(vertices=vertices, joints=joints, v_shaped=v_shaped, A=A, posed_joints=posed_J, full_pose=full_pose)
    if camera is not None:
        out['proj_joints'] = weak_persp(joints, c(camera))
    return out


def forward_shape(model: dict, betas) -> torch.Tensor:
    """SMPL.forward_shape (body_models.py:292-302)."""
    return model['v_template'] + torch.einsum('bl,mkl->bmk', betas, model['shapedirs'])


def weak_persp(joints, camera):
    """scale = softplus(camera[:, 0]); proj = scale * (joints_xy + camera[:, 1:3])."""
    s = F.softplus(camera[:, 0]).view(-1, 1, 1)
    return s * (joints[:, :, :2] + camera[:, 1:3].view(-1, 1, 2))
