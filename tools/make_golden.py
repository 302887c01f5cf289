#!/usr/bin/env python
"""Writes tests/golden/* by running the REFERENCE's own code (build container only).

    python tools/make_golden.py            # needs /root/reference

Everything written here is a small fixture that travels to the GPU box, where
/root/reference does not exist.  Fixtures:

  img00_body.npz        real SHAPY_A output shipped by the reference
                        (samples/shapy_fit_for_virtual_measurements/img_00.npz): v_shaped,
                        faces (int32), raw/decoded poses, camera, joints, proj_joints,
                        golden measurements; plus 3 more real v_shaped bodies from
                        regressor/hbw_evaluation/example_shapy_prediction.npz.
  measurement_landmarks.json   the 5 (face_idx, bc) landmarks BodyMeasurements reads from
                        mesh-mesh-intersection/data/{measurement_defitions,smplx_measurements}.yaml
  ref_smplx.npz         reference lbs()/SMPLX.forward outputs on the seeded synthetic model
  ref_head.npz          reference IterativeRegression + ContinuousRotReprDecoder outputs
  ref_hrnet.npz         reference HighResolutionNet outputs on the seeded synthetic checkpoint
  hrnet_keys.json       the 1 967 state-dict keys/shapes of the reference backbone (sha256 + list)
  ref_measure.json      oracle/measure (quirk-faithful op.cu emulation) results on the 4 real bodies
  b2a.npz               reference Polynomial (B2A head) outputs with seeded male / female weights, routed by gender
  p2p.npz               reference v2vhdError (P2P metric) outputs on seeded sparse point regressors and meshes
  v2v.npz               reference PointError(TranslationAlignment / NoAlignment) outputs (`v2v_t` / `v2v`) on two seeded meshes
  align.npz             reference PointError(ScaleAlignment / RootAlignment) outputs on seeded meshes and joints, and mpjpe14
                        end to end through a seeded dense J14 regressor
  ref_smplx_live.npz    reference SMPL-X forward (ref_shim) of tests/test_oracle_pins.py's seeded bodies
  ref_smplx_full.npz    reference SMPL-X forward in float64 with every pose part, expression and transl (float64)
  ref_smplx_grad.npz    gradients of the reference's SMPL-X forward (ref_shim.smplx_forward_ref, its own lbs() under autograd)
                        in float64 with respect to betas, expression, every pose rotation, transl and camera, for
                        closed-form cotangents on vertices, joints, v_shaped and proj_joints (grad_pattern)
  ref_weak_persp_to_blender.npz   reference demo.py weak_persp_to_blender on tests/test_writer_cpu.py's inputs
  ref_keypoint_tensor.{npz,json}  reference KeypointTensor under the tensor methods of tests/test_keypoint_tensor_cpu.py
  ref_mmi_{plane,soup}.npz        reference mesh_to_mesh_forward (oracle/_ref via oracle/run_ref_mmi.py) collisions on
                        the inputs of tests/test_gpu_zz_reference_op.py; GPU only: `python tools/make_golden.py mmi`
  ref_mmi_{plane,soup,quirk}_f64.npz   the same in float64 on the inputs of tests/test_mmi_f64_cpu.py (same recipe)
  ref_measure_grad.npz  reference BodyMeasurements autograd gradients (its own body_measurements.py, loaded by oracle/ref_body_measurements.py with
                        the C operator oracle) of each measurement with respect to v_shaped, on img_00 and the 3 extra
                        bodies: dense rows for mass, (rows, values) for height and the circumferences
  ref_openpose.npz      the reference's OpenPose reading on its 22 sample JSONs (samples/openpose): read_keypoints per
                        person, the confidences after the OpenPose dataset's per-part thresholds and binarisation,
                        keyps_to_bbox -> bbox_to_center_scale (factor 1.2), and Keypoints2D.crop + normalize at 256
  openpose_smplx_map.json   index data of the reference's name tables: the (SMPL-X keypoint, OpenPose keypoint) pairs of
                        map_keypoints('openpose25_v1' -> 'smplx') and the OpenPose part index lists the thresholds use
  preprocess.npz        reference input stage (transf_utils.crop with cv2 + ToTensor + Normalize) on seeded uint8 images:
                        crop windows, crops with OpenCV's portable path (IPP off) and with this container's IPP build
  ref_penetration.npz   the reference's DistanceFieldPenetrationLoss (mesh_mesh_intersection/loss.py, its own code) in
                        float64 on seeded triangle soups with (receiver, intruder) rows padded with -1: the loss and its
                        gradient with respect to the triangles for each (sigma, penalize_outside, linear_max,
                        point2plane) setting, and a batch without a row
"""
import hashlib
import json
import os
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shim  # noqa: E402

G = os.path.join(ROOT, 'tests', 'golden')
os.makedirs(G, exist_ok=True)
REF = ref_shim.REF


def body_fixture():
    d = ref_shim.load_img00()
    ex = np.load(os.path.join(REF, 'regressor/hbw_evaluation/example_shapy_prediction.npz'))
    np.savez_compressed(
        os.path.join(G, 'img00_body.npz'),
        v_shaped=d['v_shaped'].astype(np.float32), faces=d['faces'].astype(np.int32),
        vertices=d['vertices'].astype(np.float32),
        raw_global_rot=d['raw_global_rot'], global_rot=d['global_rot'],
        raw_body_pose=d['raw_body_pose'], body_pose=d['body_pose'], betas=d['betas'],
        camera=d['camera'], joints=d['joints'], proj_joints=d['proj_joints'],
        meas_names=np.array(['mass', 'height', 'chest', 'waist', 'hips']),
        meas_values=np.array([d['measurements'][k] for k in ['mass', 'height', 'chest', 'waist', 'hips']],
                             dtype=np.float64),
        extra_v_shaped=ex['v_shaped'].astype(np.float32))
    import yaml
    mv = yaml.safe_load(open(os.path.join(REF, 'mesh-mesh-intersection/data/smplx_measurements.yaml')))
    md = yaml.safe_load(open(os.path.join(REF, 'mesh-mesh-intersection/data/measurement_defitions.yaml')))
    lm = {}
    for out_name, src in [('head_top', 'HeadTop'), ('left_heel', 'HeelLeft'), ('chest', md['CW_p'][0]),
                          ('waist', md['BW_p'][0]), ('hips', md['IW_p'][0])]:
        lm[out_name] = dict(name=src, face_idx=int(mv[src]['face_idx']), bc=[float(x) for x in mv[src]['bc']])
    json.dump(lm, open(os.path.join(G, 'measurement_landmarks.json'), 'w'), indent=1)
    print('img00_body.npz, measurement_landmarks.json', lm)


def smplx_fixture():
    from shapy_b200 import synth
    ref = ref_shim.load()
    model = synth.make_smplx()
    g = torch.Generator().manual_seed(11)
    B = 3
    betas = torch.randn(B, 10, generator=g)
    raw = torch.randn(B, 22 * 6, generator=g) * 0.4 + synth.mean_params()[:132]
    dec1, dec21 = ref.pu.ContinuousRotReprDecoder(1), ref.pu.ContinuousRotReprDecoder(21)
    with torch.no_grad():
        grot = dec1(raw[:, :6].contiguous())
        bpose = dec21(raw[:, 6:].contiguous())
        out = ref_shim.smplx_forward_ref(model, betas, grot, bpose)
        # config 1: T-pose, B=1
        eye = torch.eye(3).view(1, 1, 3, 3)
        out_t = ref_shim.smplx_forward_ref(model, betas[:1], eye.clone(), eye.expand(1, 21, -1, -1).contiguous())
        # large head rotation to exercise the dynamic-contour LUT on both sides
        raw2 = raw.clone()
        aa = torch.tensor([[0.0, 0.9, 0.0], [0.0, -1.2, 0.1], [0.2, 0.3, 0.0]])
        R = ref.rot.batch_rodrigues(aa)
        # neck joint 12 sits at body_pose index 11 -> flat offset 6 + 11 * 6
        raw2[:, 6 + 11 * 6: 6 + 12 * 6] = R[:, :, :2].reshape(B, 6)
        grot2, bpose2 = dec1(raw2[:, :6].contiguous()), dec21(raw2[:, 6:].contiguous())
        out2 = ref_shim.smplx_forward_ref(model, betas, grot2, bpose2)
    np.savez_compressed(
        os.path.join(G, 'ref_smplx.npz'), betas=betas.numpy(), raw=raw.numpy(), global_rot=grot.numpy(),
        body_pose=bpose.numpy(), vertices=out['vertices'].numpy(), joints=out['joints'].numpy(),
        v_shaped=out['v_shaped'].numpy(), t_vertices=out_t['vertices'].numpy(), t_joints=out_t['joints'].numpy(),
        raw2=raw2.numpy(), joints2=out2['joints'].numpy(), vertices2_sub=out2['vertices'][:, ::97].numpy())
    print('ref_smplx.npz', out['vertices'].shape, out['joints'].shape)


def head_fixture():
    from shapy_b200 import synth
    ref = ref_shim.load()
    mlp = ref.net.MLP(2048 + 145, 145, layers=[1024, 1024], activation={'type': 'none'},
                      normalization={'type': 'none'}, dropout=0.5, gain=0.01)
    it = ref.net.IterativeRegression(mlp, synth.mean_params().view(1, -1), num_stages=3).eval()
    sd = synth.make_head_state_dict()
    it.load_state_dict({k[len('regressor.'):]: v for k, v in sd.items()})
    g = torch.Generator().manual_seed(12)
    feats = torch.randn(5, 2048, generator=g).abs() * 0.5
    with torch.no_grad():
        params, _ = it(feats)
    np.savez_compressed(os.path.join(G, 'ref_head.npz'), feats=feats.numpy(),
                        params=np.stack([p.numpy() for p in params]))
    print('ref_head.npz', params[-1].shape)


def hrnet_fixture():
    from shapy_b200 import synth
    m = ref_shim.build_hrnet()
    sd0 = m.state_dict()
    keys = [[k, list(v.shape)] for k, v in sd0.items()]
    digest = hashlib.sha256('\n'.join(f'{k} {s}' for k, s in keys).encode()).hexdigest()
    json.dump(dict(sha256=digest, n=len(keys), keys=keys), open(os.path.join(G, 'hrnet_keys.json'), 'w'))
    m.load_state_dict(synth.make_state_dict(sd0, seed=1))
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 3, 224, 224, generator=g)
    with torch.no_grad():
        out = m(x)
        x64 = torch.randn(1, 3, 64, 96, generator=g)
        out64 = m(x64)
    np.savez_compressed(
        os.path.join(G, 'ref_hrnet.npz'), concat=out['concat'].numpy(),
        layer1_sub=out['layer1'][:, ::7, ::5, ::5].numpy(), layer4=out['layer4'][:, ::16].numpy(),
        concat64=out64['concat'].numpy())
    print('ref_hrnet.npz', out['concat'].shape, float(out['concat'].abs().mean()), len(keys), digest[:12])


def preprocess_fixture():
    """Runs the reference's own crop() (regressor/human_shape/utils/transf_utils.py, loaded by path; cv2 is present in the
    build container) followed by the ToTensor / Normalize arithmetic of data/transforms/transforms.py:603-624,710-733."""
    import importlib.util
    import cv2
    import torchvision.transforms.functional as F
    spec = importlib.util.spec_from_file_location('ref_transf_utils', os.path.join(ref_shim.HS, 'utils', 'transf_utils.py'))
    tu = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tu)
    mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]      # config/datasets_defaults.py:37-38
    rng = np.random.default_rng(20240923)
    out = {'mean': np.float32(mean), 'std': np.float32(std)}
    cases = [  # (H, W, center, scale, size): inside, overhanging every border, strong down- and up-scaling
        (96, 128, (64.0, 48.0), 0.40, 64), (96, 128, (5.5, 90.25), 0.55, 64), (120, 90, (80.0, 10.0), 0.9, 32),
        (70, 70, (35.0, 35.0), 0.12, 64), (150, 200, (100.7, 75.2), 1.35, 32), (64, 48, (24.0, 32.0), 0.32, 64),
    ]
    for i, (H, W, center, scale, size) in enumerate(cases):
        # image-like content: smooth gradients plus noise, uint8
        yy, xx = np.mgrid[0:H, 0:W]
        img = np.stack([(xx * 255.0 / W), (yy * 255.0 / H), ((xx + yy) * 255.0 / (H + W))], -1)
        img = np.clip(img + rng.normal(0, 25, img.shape), 0, 255).astype(np.uint8)
        imgf = np.clip(img.astype(np.float32) / 255.0, 0, 1)                      # read_img, img_utils.py:57-61
        c = np.array(center, dtype=np.float32)
        res = {}
        for tag, ipp in (('portable', False), ('ipp', True)):
            cv2.ipp.setUseIPP(ipp)
            crop = tu.crop(imgf, c, scale, [size, size])
            t = F.to_tensor(crop)
            t = torch.clamp(t, 0, 1)
            res[tag] = F.normalize(t, mean=mean, std=std).numpy()
        cv2.ipp.setUseIPP(True)
        ul = np.array(tu.transform([1, 1], c, scale, [size, size], invert=1)) - 1
        br = np.array(tu.transform([size + 1, size + 1], c, scale, [size, size], invert=1)) - 1
        out[f'img{i}'] = img
        out[f'center{i}'] = c
        out[f'scale{i}'] = np.float64(scale)
        out[f'size{i}'] = np.int64(size)
        out[f'ul{i}'] = ul.astype(np.int64)
        out[f'br{i}'] = br.astype(np.int64)
        out[f'out{i}'] = res['portable']
        out[f'ipp_dev{i}'] = np.float64(np.abs(res['portable'] - res['ipp']).max())   # this container's IPP build vs portable
    out['n'] = np.int64(len(cases))
    np.savez_compressed(os.path.join(G, 'preprocess.npz'), **out)
    print('preprocess.npz', os.path.getsize(os.path.join(G, 'preprocess.npz')), 'bytes; max |portable - ipp| =',
          max(float(out[f'ipp_dev{i}']) for i in range(len(cases))))


def b2a_fixture():
    """Runs the reference's own Polynomial module (attributes/attributes/attributes_betas/polynomial.py, loaded by path behind
    a stub of attributes.utils.typing) with seeded male / female weights, and routes by gender exactly as
    regressor/human_shape/models/common/iterative_regressor.py:761-776 does."""
    import importlib.util
    import types
    from loguru import logger
    logger.remove()
    for name in ('attributes', 'attributes.utils', 'attributes.utils.typing'):
        if name not in sys.modules:
            m = types.ModuleType(name)
            m.__path__ = []
            sys.modules[name] = m
    sys.modules['attributes.utils.typing'].Tensor = torch.Tensor
    sys.modules['attributes.utils.typing'].Array = np.ndarray
    spec = importlib.util.spec_from_file_location(
        'ref_polynomial', os.path.join(REF, 'attributes', 'attributes', 'attributes_betas', 'polynomial.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    torch.manual_seed(31)
    males, females = mod.Polynomial(10, 15, degree=2), mod.Polynomial(10, 15, degree=2)
    for p in (males, females):                      # ratings live in [1, 5]: give the synthetic heads that scale
        with torch.no_grad():
            p.linear.weight.mul_(0.5)
            p.linear.bias.copy_(torch.rand(15) * 4 + 1)
    betas = torch.randn(9, 10) * 1.5
    gender_strs = ['male', 'Female', 'f', '', None, 'M', 'neutral', 'female', 'm']
    genders = np.array([x.lower()[0] if (x is not None and x != '') else 'n' for x in gender_strs])
    gm, gf = np.where(genders == 'm')[0], np.where(genders == 'f')[0]
    with torch.no_grad():
        am, af = males(betas[gm, :]), females(betas[gf, :])
        attributes = torch.zeros(betas.shape[0], am.shape[1])
        attributes[gm, :] = am
        attributes[gf, :] = af
    np.savez_compressed(
        os.path.join(G, 'b2a.npz'), betas=betas.numpy(), genders=np.array([g if g is not None else '<none>' for g in gender_strs]),
        w_male=males.linear.weight.detach().numpy(), b_male=males.linear.bias.detach().numpy(),
        w_female=females.linear.weight.detach().numpy(), b_female=females.linear.bias.detach().numpy(),
        indices_000=males.indices_000.numpy(), indices_001=males.indices_001.numpy(), attributes=attributes.numpy())
    print('b2a.npz', os.path.getsize(os.path.join(G, 'b2a.npz')), 'bytes')


def _load_ref_metrics():
    """The reference's regressor/human_shape/utils/metrics.py loaded by path behind stubs of open3d / .np_utils / .typing."""
    import importlib.util
    import types
    from loguru import logger
    logger.remove()
    if 'ref_hs.utils.metrics' in sys.modules:
        return sys.modules['ref_hs.utils.metrics']
    for name in ('open3d', 'ref_hs', 'ref_hs.utils', 'ref_hs.utils.np_utils', 'ref_hs.utils.typing'):
        m = types.ModuleType(name)
        m.__path__ = []
        sys.modules[name] = m
    sys.modules['ref_hs.utils.np_utils'].np2o3d_pcl = None
    for n in ('Tensor', 'Array', 'IntList'):
        setattr(sys.modules['ref_hs.utils.typing'], n, object)
    spec = importlib.util.spec_from_file_location('ref_hs.utils.metrics', os.path.join(ref_shim.HS, 'utils', 'metrics.py'))
    mod = importlib.util.module_from_spec(spec)
    mod.__package__ = 'ref_hs.utils'
    sys.modules['ref_hs.utils.metrics'] = mod
    spec.loader.exec_module(mod)
    return mod


def v2v_fixture():
    """Runs the reference's own PointError with TranslationAlignment / NoAlignment (metrics.py:232-277, 335-366), i.e. the
    `v2v_t` / `v2v` evaluation metrics (evaluation.py:192-224, 595-602), on two seeded meshes of the same topology."""
    mod = _load_ref_metrics()
    rng = np.random.default_rng(78)
    B, V = 3, 1500
    est = rng.normal(0, 0.4, (B, V, 3)).astype(np.float32)
    gt = (est + rng.normal(0, 0.01, (B, V, 3)) + rng.normal(0, 0.05, (B, 1, 3))).astype(np.float32)
    out = {}
    for tag, name in (('aligned', 'translation'), ('raw', 'none')):
        pe = mod.PointError(mod.build_alignment(name))
        out[f'error_{tag}'] = np.asarray(pe(est.copy(), gt.copy()), np.float64)
    np.savez_compressed(os.path.join(G, 'v2v.npz'), est=est, gt=gt, **out)
    print('v2v.npz', os.path.getsize(os.path.join(G, 'v2v.npz')), 'bytes; mean aligned error', out['error_aligned'].mean())


def align_fixture():
    """Runs the reference's own PointError with ScaleAlignment and RootAlignment (metrics.py:173-229, 279-303, 335-366):
    the scale-corrected `v2v_t` on two seeded same-topology meshes far from the origin (float32, as the evaluator passes
    them), the root-aligned joint error for several root lists, and mpjpe14 end to end (evaluation.py:161-190, 616-620) with
    a seeded dense float64 J14 regressor."""
    mod = _load_ref_metrics()
    rng = np.random.default_rng(79)
    B, V, J = 3, 1500, 14
    offset = np.array([0.3, 0.4, 2.5])
    est = rng.normal(0, 0.4, (B, V, 3)).astype(np.float32)
    gt = (1.1 * est + rng.normal(0, 0.02, (B, V, 3)) + offset).astype(np.float32)
    out = dict(est=est, gt=gt)
    out['error_scale'] = np.asarray(mod.PointError(mod.build_alignment('scale'))(est.copy(), gt.copy()), np.float64)
    j_est = (rng.normal(0, 0.3, (B, J, 3)) + offset).astype(np.float32)
    j_gt = (j_est + rng.normal(0, 0.03, (B, J, 3)) + [0.05, -0.02, 0.1]).astype(np.float32)
    out.update(j_est=j_est, j_gt=j_gt)
    for tag, root in ROOT_CASES:
        pe = mod.PointError(mod.build_alignment('root', root=[0]))
        pe.set_root(list(root))                         # as _compute_mpjpe does (evaluation.py:146-153)
        with warnings.catch_warnings(), np.errstate(invalid='ignore'):
            warnings.simplefilter('ignore', RuntimeWarning)           # the empty list: "Mean of empty slice"
            out[f'error_root_{tag}'] = np.asarray(pe(j_est.copy(), j_gt.copy()), np.float64)
        out[f'root_{tag}'] = np.array(root, np.int64)
    # mpjpe14: a J14-like regressor with 32 positive weights per row summing to 1, float32-representable values stored as
    # float64 (the dtype of the regressor pickle); the einsum line of evaluation.py:183-184 on float32 vertices
    J14 = np.zeros((J, V))
    for j in range(J):
        J14[j, rng.choice(V, 32, replace=False)] = rng.dirichlet(np.ones(32)).astype(np.float32)
    verts = (est + offset).astype(np.float32)
    est_joints_np = np.einsum('jv,bvn->bjn', J14, verts)
    j14_gt = (est_joints_np * 1.05 + rng.normal(0, 0.02, (B, J, 3))).astype(np.float32)
    out.update(j14=J14, j14_verts=verts, j14_gt=j14_gt, j14_joints=est_joints_np)
    for tag, name in (('root', 'root'), ('scale', 'scale')):
        pe = mod.PointError(mod.build_alignment(name, root=[2, 3]))     # evaluation.py:616-619
        out[f'error_mpjpe14_{tag}'] = np.asarray(pe(est_joints_np, j14_gt), np.float64)
    np.savez_compressed(os.path.join(G, 'align.npz'), **out)
    print('align.npz', os.path.getsize(os.path.join(G, 'align.npz')), 'bytes; mean scale error', out['error_scale'].mean(),
          'mean mpjpe14 root error', out['error_mpjpe14_root'].mean())


# (tag, root list) of the root-aligned cases in align.npz: mpjpe14's [2, 3], the default [0], a negative index and the
# empty list the evaluator's default `root_joints = ()` gives (NaN)
ROOT_CASES = (('r23', [2, 3]), ('r0', [0]), ('rm1', [-1]), ('rempty', []))


def p2p_fixture():
    """Runs the reference's own v2vhdError (regressor/human_shape/utils/metrics.py:368-456, loaded by path behind stubs of
    open3d / .np_utils / .typing) on seeded sparse point regressors (3 barycentric weights per point) and meshes, in
    float64 on the CPU as the evaluator does (evaluation.py:258-260)."""
    import pickle
    import tempfile
    import scipy.sparse as sp
    mod = _load_ref_metrics()
    rng = np.random.default_rng(77)
    P, V1, V2, B = 700, 400, 250, 3

    def regressor(V):
        cols = rng.integers(0, V, (P, 3))
        w = rng.dirichlet([1, 1, 1], P)
        # float32-representable weights stored as float64, the dtype of the reference's regressor pickles (the evaluator
        # multiplies them with .double() vertices)
        return sp.csr_matrix((w.reshape(-1).astype(np.float32).astype(np.float64), (np.repeat(np.arange(P), 3), cols.reshape(-1))),
                             shape=(P, V))
    r_in, r_tg = regressor(V1), regressor(V2)
    r_in.sum_duplicates()
    r_tg.sum_duplicates()
    tmp = tempfile.mkdtemp()
    paths = []
    for name, r in (('in', r_in), ('tg', r_tg)):
        paths.append(os.path.join(tmp, name + '.pkl'))
        with open(paths[-1], 'wb') as f:
            pickle.dump(r, f)
    v_in = (rng.normal(0, 0.3, (B, V1, 3)) + [0.1, -0.2, 0.05]).astype(np.float32)
    v_tg = (rng.normal(0, 0.3, (B, V2, 3)) + [-0.3, 0.4, 0.0]).astype(np.float32)
    out = {}
    for align in (True, False):
        metric = mod.v2vhdError(paths[0], paths[1], align=align)
        if align:
            mean, err = metric(torch.from_numpy(v_in).double(), torch.from_numpy(v_tg).double())
        else:       # metrics.py:449-452 only defines t under `if self.align`: the unaligned variant is the same formula with t = 0
            a = metric.sparse_batch_mm(metric.input_point_regressor.double(), torch.from_numpy(v_in).double())
            c = metric.sparse_batch_mm(metric.target_point_regressor.double(), torch.from_numpy(v_tg).double())
            err = torch.sqrt(torch.pow(a - c, 2).sum(axis=-1))
            mean = err.mean(1)
        out['mean_aligned' if align else 'mean_raw'] = mean.numpy()
        out['error_aligned' if align else 'error_raw'] = err.numpy()
    for name, r in (('in', r_in), ('tg', r_tg)):
        out[f'{name}_row_ptr'], out[f'{name}_col'], out[f'{name}_val'] = (r.indptr.astype(np.int32), r.indices.astype(np.int32),
                                                                             r.data.astype(np.float32))
    np.savez_compressed(os.path.join(G, 'p2p.npz'), v_in=v_in, v_tg=v_tg, **out)
    print('p2p.npz', os.path.getsize(os.path.join(G, 'p2p.npz')), 'bytes; mean aligned error', out['mean_aligned'])


def smplx_live_fixture():
    from oracle import smplx_oracle
    from shapy_b200 import synth
    model = synth.make_smplx()
    g = torch.Generator().manual_seed(5)
    betas = torch.randn(2, 10, generator=g)
    raw = torch.randn(2, 132, generator=g) * 0.3 + synth.mean_params()[:132]
    grot, bpose = smplx_oracle.decode_6d(raw[:, :6]), smplx_oracle.decode_6d(raw[:, 6:])
    ref = ref_shim.smplx_forward_ref(model, betas, grot, bpose)
    np.savez_compressed(os.path.join(G, 'ref_smplx_live.npz'),
                        **{k: ref[k].numpy().astype(np.float32) for k in ('vertices', 'joints', 'v_shaped')})


def smplx_full_fixture():
    """The reference's SMPL-X forward (ref_shim.smplx_forward_ref on the verbatim lbs(), find_dynamic_lmk_idx_and_bcoords
    and vertices2landmarks) in float64 on the float64 synthetic model: every pose part non-identity, a nonzero expression
    and transl, and the neck of bodies 0 / 1 turned past each end of the dynamic-contour LUT.  Vertices and v_shaped are
    subsampled (every 7th vertex) to keep the fixture small."""
    from shapy_b200 import synth
    ref = ref_shim.load()
    dt = torch.float64
    model = synth.make_smplx(dtype=dt)
    g = torch.Generator().manual_seed(21)
    B = 4
    betas = torch.randn(B, 10, generator=g, dtype=dt)
    expression = torch.randn(B, 10, generator=g, dtype=dt)
    transl = torch.randn(B, 3, generator=g, dtype=dt) * 0.5
    aa = torch.randn(B, 55, 3, generator=g, dtype=dt) * 0.3
    aa[:2, [0, 3, 6, 9, 15]] *= 0.1                              # the rest of the neck chain nearly straight
    aa[0, 12] = torch.tensor([0.0, 1.2, 0.0], dtype=dt)         # neck about y, both ways: LUT row 78 and the clamp at 39
    aa[1, 12] = torch.tensor([0.0, -1.2, 0.0], dtype=dt)
    rot = ref.rot.batch_rodrigues(aa.reshape(-1, 3)).reshape(B, 55, 3, 3)
    assert rot.dtype == dt
    with torch.no_grad():
        out = ref_shim.smplx_forward_ref(model, betas, rot[:, :1], rot[:, 1:22], jaw_pose=rot[:, 22:23],
                                         leye_pose=rot[:, 23:24], reye_pose=rot[:, 24:25],
                                         left_hand_pose=rot[:, 25:40], right_hand_pose=rot[:, 40:55],
                                         expression=expression, transl=transl)
    np.savez_compressed(
        os.path.join(G, 'ref_smplx_full.npz'), betas=betas.numpy(), expression=expression.numpy(),
        transl=transl.numpy(), rot=rot.numpy(), vertices_sub=out['vertices'][:, ::7].numpy(),
        joints=out['joints'].numpy(), v_shaped_sub=out['v_shaped'][:, ::7].numpy())
    print('ref_smplx_full.npz', os.path.getsize(os.path.join(G, 'ref_smplx_full.npz')), 'bytes')


# cotangent name -> (frequency, phase, amplitude): g.flat[i] = amplitude * sin(frequency * i + phase), float64
GRAD_PATTERN = {'vertices': (0.731, 0.1, 1.0), 'joints': (1.913, 0.7, 1.0), 'v_shaped': (0.377, 1.9, 0.5),
                'proj_joints': (2.71, 0.3, 1.0)}


def grad_pattern(name, shape):
    f, ph, amp = GRAD_PATTERN[name]
    return amp * np.sin(f * np.arange(int(np.prod(shape)), dtype=np.float64) + ph).reshape(shape)


def smplx_grad_fixture():
    """Gradients of the reference's SMPL-X forward under its own autograd (ref_shim.smplx_forward_ref on the verbatim
    lbs(), pose2rot=False) in float64 on the float64 synthetic model, for the loss
    <g_v, vertices> + <g_j, joints> + <g_s, v_shaped> + <g_p, proj_joints> with the closed-form cotangents of
    grad_pattern.  The bodies are smplx_full_fixture's (every pose part, expression, transl, the neck past both ends
    of the LUT) plus a camera.  transl is added to vertices and joints after the forward and proj_joints projects the
    joints before transl, as shapy_b200's SMPLX.forward does; proj = softplus(c0) (xy + c[1:3])
    (camera_projection.py:181-213)."""
    from shapy_b200 import synth
    ref = ref_shim.load()
    dt = torch.float64
    model = synth.make_smplx(dtype=dt)
    g = torch.Generator().manual_seed(21)
    B = 4
    betas = torch.randn(B, 10, generator=g, dtype=dt)
    expression = torch.randn(B, 10, generator=g, dtype=dt)
    transl = torch.randn(B, 3, generator=g, dtype=dt) * 0.5
    aa = torch.randn(B, 55, 3, generator=g, dtype=dt) * 0.3
    aa[:2, [0, 3, 6, 9, 15]] *= 0.1
    aa[0, 12] = torch.tensor([0.0, 1.2, 0.0], dtype=dt)
    aa[1, 12] = torch.tensor([0.0, -1.2, 0.0], dtype=dt)
    rot = ref.rot.batch_rodrigues(aa.reshape(-1, 3)).reshape(B, 55, 3, 3)
    camera = torch.tensor([[0.9, 0.05, -0.1], [-1.5, 0.2, 0.1], [21.0, -0.3, 0.2], [2.0, 0.0, 0.4]], dtype=dt)
    leaves = dict(betas=betas, expression=expression, transl=transl, rot=rot, camera=camera)
    leaves = {k: v.detach().clone().requires_grad_(True) for k, v in leaves.items()}
    r = leaves['rot']
    out = ref_shim.smplx_forward_ref(model, leaves['betas'], r[:, :1], r[:, 1:22], jaw_pose=r[:, 22:23],
                                     leye_pose=r[:, 23:24], reye_pose=r[:, 24:25], left_hand_pose=r[:, 25:40],
                                     right_hand_pose=r[:, 40:55], expression=leaves['expression'])
    t = leaves['transl'].unsqueeze(1)
    vertices, joints = out['vertices'] + t, out['joints'] + t
    cam = leaves['camera']
    proj = torch.nn.functional.softplus(cam[:, 0]).view(-1, 1, 1) * (out['joints'][:, :, :2] + cam[:, 1:3].view(-1, 1, 2))
    loss = 0
    for name, y in (('vertices', vertices), ('joints', joints), ('v_shaped', out['v_shaped']), ('proj_joints', proj)):
        loss = loss + (torch.from_numpy(grad_pattern(name, tuple(y.shape))) * y).sum()
    loss.backward()
    np.savez_compressed(
        os.path.join(G, 'ref_smplx_grad.npz'), **{k: v.detach().numpy() for k, v in leaves.items()},
        **{f'grad_{k}': v.grad.numpy() for k, v in leaves.items()},
        pattern_names=np.array(list(GRAD_PATTERN)), pattern=np.array(list(GRAD_PATTERN.values())))
    print('ref_smplx_grad.npz', os.path.getsize(os.path.join(G, 'ref_smplx_grad.npz')), 'bytes')


def writer_camera_fixture():
    import ast
    from collections import defaultdict
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    import test_writer_cpu as tw
    path = os.path.join(REF, 'regressor', 'demo.py')
    fn = [n for n in ast.parse(open(path).read()).body if isinstance(n, ast.FunctionDef) and n.name == 'weak_persp_to_blender'][0]
    ns = {'torch': torch, 'np': np, 'defaultdict': defaultdict}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), path, 'exec'), ns)     # executed where it lies
    targets = tw.make_targets(5, np.random.default_rng(2))
    scale = torch.rand(5, 1, generator=torch.Generator().manual_seed(3)) + 0.5
    transl = torch.randn(5, 2, generator=torch.Generator().manual_seed(4)) * 0.1
    r = ns['weak_persp_to_blender'](targets, scale, transl, H=720, W=1280, sensor_width=36, focal_length=5000)
    np.savez_compressed(os.path.join(G, 'ref_weak_persp_to_blender.npz'), **{k: np.asarray(v) for k, v in r.items()})


def keypoint_tensor_fixture():
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    import test_keypoint_tensor_cpu as tk
    path = os.path.join(REF, 'regressor', 'human_shape', 'models', 'body_models', 'utils.py')
    src = open(path).read()
    start = src.index('class KeypointTensor(object):')
    end = src.index('\nclass ', start + 10) if '\nclass ' in src[start + 10:] else len(src)
    ns = {'torch': torch}
    exec(compile(src[start:end], path, 'exec'), ns)                           # executed where it lies
    b = tk.make(ns['KeypointTensor'])
    ops = [lambda k: k.view(2, 9), lambda k: k.detach(), lambda k: k.to(torch.float64), lambda k: k.sum(dim=2),
           lambda k: k.matmul(torch.full((3, 3), 0.5)), lambda k: k.clone().reshape(3, 6), lambda k: k.permute(2, 0, 1)]
    arrs, meta = {}, []
    for i, f in enumerate(ops):
        y = f(b)
        arrs[f'op{i}'] = y._t.numpy()
        meta.append(dict(keypoint_names=list(y.keypoint_names), source=y.source, connections=[list(c) for c in y.connections],
                         part_indices={k: (v.tolist() if torch.is_tensor(v) else v) for k, v in y.part_indices.items()}))
    arrs['index1'] = b[1].numpy()
    arrs['numpy'] = b.numpy()
    np.savez(os.path.join(G, 'ref_keypoint_tensor.npz'), **arrs)
    json.dump(dict(ops=meta, index1_type=type(b[1]).__name__), open(os.path.join(G, 'ref_keypoint_tensor.json'), 'w'))


def mmi_fixtures():
    """Needs a GPU and oracle/_ref (python oracle/build_ref.py).  Stores the filled slots of the reference's output, in
    the inputs' dtype: float32 for ref_mmi_{plane,soup}, float64 for ref_mmi_{plane,soup,quirk}_f64."""
    import subprocess
    import tempfile
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    import test_gpu_zz_reference_op as t
    import test_mmi_f64_cpu as t64
    quirk_q, quirk_t, quirk_m, quirk_pairs = t64.quirk_inputs_f64()
    for name, (query, target, M) in (('ref_mmi_plane', t.plane_inputs(G)), ('ref_mmi_soup', t.soup_inputs()),
                                     ('ref_mmi_plane_f64', t64.plane_inputs_f64(G)),
                                     ('ref_mmi_soup_f64', t64.soup_inputs_f64()),
                                     ('ref_mmi_quirk_f64', (quirk_q, quirk_t, quirk_m))):
        with tempfile.TemporaryDirectory() as tmp:
            inp, outp = os.path.join(tmp, 'in.npz'), os.path.join(tmp, 'out.npz')
            np.savez(inp, query=query, target=target, max_collisions=np.int64(M))
            subprocess.run([sys.executable, os.path.join(ROOT, 'oracle', 'run_ref_mmi.py'), inp, outp], check=True)
            d = np.load(outp)
            f, bcs = d['faces'], d['bcs']
        assert bcs.dtype == query.dtype
        if name == 'ref_mmi_quirk_f64':      # the fixture exists to show these pairs reported by the reference
            t64.check_quirk(f[0], M, quirk_pairs, 'reference')
        keep = np.nonzero(f >= 0)
        np.savez_compressed(os.path.join(G, f'{name}.npz'), shape=np.int64(f.shape), idx=np.stack(keep, 1).astype(np.int32),
                            faces=f[keep].astype(np.int32), bcs=bcs[keep], query=query)


def measure_grad_fixture():
    from oracle import ref_body_measurements
    BM, cfg = ref_body_measurements.load()
    bm = BM(cfg)
    g = np.load(os.path.join(G, 'img00_body.npz'))
    bodies = np.concatenate([g['v_shaped'][None], g['extra_v_shaped']], 0).astype(np.float32)
    f = torch.from_numpy(g['faces'].astype(np.int64))
    out = {'mass': np.zeros(bodies.shape, np.float32)}
    for b in range(bodies.shape[0]):
        for i, name in enumerate(('mass', 'height', 'chest', 'waist', 'hips')):
            v = torch.from_numpy(bodies[b])[None].clone().requires_grad_(True)
            bm(v[:, f])['measurements'][name]['tensor'].sum().backward()
            gr = v.grad[0].numpy()
            if name == 'mass':
                out['mass'][b] = gr
            else:
                rows = np.nonzero(np.abs(gr).sum(1))[0].astype(np.int32)
                out[f'{name}_{b}_rows'], out[f'{name}_{b}_values'] = rows, gr[rows]
    np.savez_compressed(os.path.join(G, 'ref_measure_grad.npz'), **out)
    print('ref_measure_grad.npz', {k: v.shape for k, v in out.items() if k.endswith('rows')})


def _load_ref_keypoint_utils():
    """The reference's data/utils/keypoints.py, keypoint_names.py, bbox.py, transf_utils.get_transform and the crop /
    normalize methods of Keypoints2D, loaded where they lie behind stub parent packages (open3d and the structure
    base classes are not needed by these functions)."""
    import types
    HS = ref_shim.HS

    def stub(name):
        m = sys.modules.get(name) or types.ModuleType(name)
        m.__path__ = []
        sys.modules[name] = m
        return m
    o3 = types.ModuleType('open3d')
    o3.geometry = types.SimpleNamespace(PointCloud=object)
    sys.modules.setdefault('open3d', o3)
    for n in ('human_shape', 'human_shape.data', 'human_shape.data.utils'):
        stub(n)
    u = stub('human_shape.utils')
    ty = types.ModuleType('human_shape.utils.typing')
    ty.Array = ty.Tensor = object
    sys.modules['human_shape.utils.typing'] = ty
    npu = ref_shim._load('human_shape.utils.np_utils', HS + '/utils/np_utils.py', 'human_shape.utils')
    bu = ref_shim._load('human_shape.utils.bool_utils', HS + '/utils/bool_utils.py', 'human_shape.utils')
    for n in ('Array', 'StringList', 'IntList', 'Tensor'):
        setattr(u, n, object)
    u.binarize, u.nand = npu.binarize, bu.nand
    kpm = ref_shim._load('human_shape.data.utils.keypoints', HS + '/data/utils/keypoints.py', 'human_shape.data.utils')
    names = ref_shim._load('human_shape.data.utils.keypoint_names', HS + '/data/utils/keypoint_names.py',
                           'human_shape.data.utils')
    bbox = ref_shim._load('human_shape.data.utils.bbox', HS + '/data/utils/bbox.py', 'human_shape.data.utils')
    tu = ref_shim._load('human_shape.utils.transf_utils', HS + '/utils/transf_utils.py', 'human_shape.utils')
    path = HS + '/data/structures/keypoints.py'
    src = open(path).read()
    start = src.index('    def crop(self, center, scale, crop_size=224')
    end = src.index('    def ', src.index('    def normalize(self', start) + 10)
    ns = {'np': np, 'torch': torch, 'get_transform': tu.get_transform, 'AbstractStructure': type(None)}
    body = 'class _Methods:\n' + src[start:end]
    exec(compile(body, path, 'exec'), ns)                                    # executed where it lies

    class Kp2D:                                                              # the fields the two methods read
        def __init__(self, kp, size, flip_indices=None, source=None, apply_crop=True, flip_axis=0, dtype=None):
            kp = np.asarray(kp)
            self.keypoints, self.conf, self.size = kp[:, :-1], kp[:, -1], size
            self.apply_crop, self.flip_indices, self.source, self.flip_axis = apply_crop, flip_indices, source, flip_axis
            self.extra_fields = {}

        def add_field(self, k, v):
            self.extra_fields[k] = v
    Kp2D.crop, Kp2D.normalize = ns['_Methods'].crop, ns['_Methods'].normalize
    return kpm, names, bbox, Kp2D


def openpose_fixture(crop_size=256):
    """The OpenPose dataset's __getitem__ (datasets/openpose.py:148-215) with its defaults: body / hand / face thresholds
    0.1 / 0.2 / 0.4, binarisation, no face contour, body_dset_factor 1.2."""
    if not hasattr(np, 'int'):
        np.int = int                      # Keypoints2D.crop casts with np.int (removed from NumPy 1.24)
    kpm, names, bbox, Kp2D = _load_ref_keypoint_utils()
    src_names = names.KEYPOINT_NAMES_DICT['openpose25_v1']
    parts = kpm.get_part_idxs(src_names, names.KEYPOINT_PARTS)
    face = parts['face'][:-17]
    tgt, srcidx, n_target = kpm.map_keypoints('openpose25_v1', 'smplx', names.KEYPOINT_NAMES_DICT)
    mapping = {'source': 'openpose25_v1', 'target': 'smplx', 'num_target': int(n_target),
               'pairs': [[int(t), int(s)] for t, s in zip(tgt, srcidx)],
               'parts': {'body': parts['body'].tolist(), 'left_hand': parts['left_hand'].tolist(),
                         'right_hand': parts['right_hand'].tolist(), 'face': face.tolist()},
               'thresholds': {'body': 0.1, 'hand': 0.2, 'face': 0.4}, 'bbox_scale_factor': 1.2}
    json.dump(mapping, open(os.path.join(G, 'openpose_smplx_map.json'), 'w'), indent=1)
    out = {k: [] for k in ('raw', 'thresholded', 'center', 'scale', 'bbox_size', 'cropped', 'file_index', 'valid')}
    folder = os.path.join(REF, 'samples', 'openpose')
    files = sorted(f for f in os.listdir(folder) if f.endswith('.json'))
    for fi, f in enumerate(files):
        people = kpm.read_keypoints(os.path.join(folder, f))
        for raw in ([] if people is None else people):
            kp = raw.copy()
            kp[:, -1] = np.clip(kp[:, -1], 0, 1)
            body_conf, face_conf = kp[parts['body'], -1], kp[face, -1]
            lh, rh = kp[parts['left_hand'], -1], kp[parts['right_hand'], -1]
            body_conf[body_conf < 0.1] = 0.0
            face_conf[face_conf < 0.4] = 0.0
            lh[lh < 0.2] = 0.0
            rh[rh < 0.2] = 0.0
            kp[parts['body'], -1] = kpm.binarize(body_conf, 0.1, kp.dtype)
            kp[parts['left_hand'], -1] = kpm.binarize(lh, 0.2, kp.dtype)
            kp[parts['right_hand'], -1] = kpm.binarize(rh, 0.2, kp.dtype)
            kp[face, -1] = kpm.binarize(face_conf, 0.4, kp.dtype)
            center, scale, size = bbox.bbox_to_center_scale(bbox.keyps_to_bbox(kp[:, :-1], kp[:, -1]),
                                                            dset_scale_factor=1.2)
            valid = center is not None
            if valid:
                c = Kp2D(kp, (1000, 1000, 3)).crop(center, scale, crop_size=crop_size).normalize()
                cropped = np.concatenate([c.keypoints, c.conf[:, None]], 1)
            else:
                center, scale, size, cropped = np.full(2, np.nan), np.nan, np.nan, np.full_like(kp, np.nan)
            for k, v in (('raw', raw), ('thresholded', kp), ('center', center), ('scale', scale), ('bbox_size', size),
                         ('cropped', cropped), ('file_index', fi), ('valid', valid)):
                out[k].append(v)
    arrs = {k: np.asarray(v) for k, v in out.items()}
    arrs['files'] = np.array(files)
    arrs['crop_size'] = np.int32(crop_size)
    np.savez_compressed(os.path.join(G, 'ref_openpose.npz'), **arrs)
    print('ref_openpose.npz', {k: v.shape for k, v in arrs.items()}, len(mapping['pairs']), 'mapped keypoints')


PENETRATION_SETTINGS = [(0.5, True, 1000.0, False), (0.5, True, 1000.0, True), (0.5, False, 1000.0, False),
                        (0.05, True, 1000.0, False), (0.3, True, 0.4, False), (1.5, False, 1000.0, True)]


def penetration_fixture():
    import importlib.util
    spec = importlib.util.spec_from_file_location(
        'ref_penetration_loss', os.path.join(REF, 'mesh-mesh-intersection', 'mesh_mesh_intersection', 'loss.py'))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    rng = np.random.default_rng(20261018)
    B, F, C = 3, 24, 20
    # clusters of small triangles around shared centres, so that many rows have points inside the cones
    centres = rng.normal(size=(B, F, 1, 3)) * 0.05
    tris = centres + rng.normal(size=(B, F, 3, 3)) * 0.08
    idx = np.full((B, C, 2), -1, np.int64)
    for b, n in enumerate([C, 11, 5]):
        r = rng.integers(0, F, size=(n,))
        i = (r + rng.integers(1, F, size=(n,))) % F
        idx[b, :n, 0], idx[b, :n, 1] = r, i
    perm = rng.permutation(C)              # padding rows between real ones
    idx[1] = idx[1][perm]
    out = dict(triangles=tris, collision_idxs=idx, settings=np.array(PENETRATION_SETTINGS, np.float64))
    for k, (sigma, po, lmax, p2p) in enumerate(PENETRATION_SETTINGS):
        t = torch.from_numpy(tris).requires_grad_(True)
        loss = m.DistanceFieldPenetrationLoss(sigma=sigma, point2plane=p2p, penalize_outside=po, linear_max=lmax)(
            t, torch.from_numpy(idx))
        loss.sum().backward()
        out[f'loss_{k}'] = loss.detach().numpy()
        out[f'grad_{k}'] = t.grad.numpy()
    t = torch.from_numpy(tris).requires_grad_(True)
    out['loss_empty'] = m.DistanceFieldPenetrationLoss()(t, torch.full((B, 4, 2), -1, dtype=torch.long)).detach().numpy()
    np.savez_compressed(os.path.join(G, 'ref_penetration.npz'), **out)
    print('ref_penetration.npz', {k: v.tolist() for k, v in out.items() if k.startswith('loss')})


if __name__ == '__main__':
    which = sys.argv[1:] or ['body', 'smplx', 'head', 'hrnet', 'preprocess', 'b2a', 'p2p', 'v2v', 'align', 'smplx_live',
                             'smplx_full', 'camera', 'keypoint', 'measure_grad', 'smplx_grad', 'openpose',
                             'penetration']
    torch.set_num_threads(8)
    if 'body' in which:
        body_fixture()
    if 'smplx' in which:
        smplx_fixture()
    if 'head' in which:
        head_fixture()
    if 'hrnet' in which:
        hrnet_fixture()
    if 'preprocess' in which:
        preprocess_fixture()
    if 'b2a' in which:
        b2a_fixture()
    if 'p2p' in which:
        p2p_fixture()
    if 'v2v' in which:
        v2v_fixture()
    if 'align' in which:
        align_fixture()
    if 'smplx_live' in which:
        smplx_live_fixture()
    if 'smplx_full' in which:
        smplx_full_fixture()
    if 'smplx_grad' in which:
        smplx_grad_fixture()
    if 'camera' in which:
        writer_camera_fixture()
    if 'keypoint' in which:
        keypoint_tensor_fixture()
    if 'mmi' in which:
        mmi_fixtures()
    if 'measure_grad' in which:
        measure_grad_fixture()
    if 'openpose' in which:
        openpose_fixture()
    if 'penetration' in which:
        penetration_fixture()
