"""GPU: the self-penetration term in the Adam fits (fit_body_to_scan, fit_body_to_keypoints, single-image
fit_body_to_keypoints_2d): weight 0 is the fit without the term bit for bit, the reported penetration is that of the
final parameters, in the scan fit a weight > 0 leaves fewer intersecting pairs and a lower penetration loss from a
self-intersecting start, and the fits without the term raise before any launch."""
import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from penetration_oracle import smooth_smplx
from shapy_b200 import _lib, ops, synth
from shapy_b200.fit import fit_body_to_keypoints, fit_body_to_keypoints_2d, fit_body_to_scan

pytestmark = pytest.mark.gpu
_CACHE = {}


def _setup():
    """Two bodies with both elbows flexed into the upper arms (self-intersecting), their raw 6D pose, keypoints,
    projected keypoints and a scan of their vertices."""
    if _CACHE:
        return _CACHE
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    m = SMPLX(data_struct=smooth_smplx()).cuda()
    B = 2
    rot = np.tile(np.eye(3, dtype=np.float32), (B, 22, 1, 1))
    for b, ang in enumerate([2.6, 2.4]):
        rot[b, 18] = Rotation.from_rotvec([0, -ang, 0]).as_matrix()
        rot[b, 19] = Rotation.from_rotvec([0, ang, 0]).as_matrix()
    raw = torch.tensor(rot[..., :, :2].reshape(B, 132))   # the first two columns, row-major: the 6D layout
    rot_t = ops.decode_rot6d(raw.cuda())
    assert torch.allclose(rot_t.cpu(), torch.tensor(rot), atol=1e-5)
    with torch.no_grad():
        out = m(global_rot=rot_t[:, :1], body_pose=rot_t[:, 1:], betas=torch.zeros(B, m.num_betas, device='cuda'),
                camera=torch.tensor([[0.9, 0, 0]] * B, device='cuda'), return_shaped=False)
    init = {'global_rot': raw[:, :6].cuda(), 'body_pose': raw[:, 6:].cuda()}
    v = out['vertices']
    pen = dict(part_labels=ops.face_parts(m), ignored_part_pairs=ops.parent_child_part_pairs(m.parents))
    _CACHE.update(model=m, init=init, v=v.clone(), joints=out['joints'][:].clone(),
                  proj=out['proj_joints'].clone(), pen=pen)
    return _CACHE


def _fits(c):
    m, init = c['model'], c['init']
    return {
        'scan': lambda **kw: fit_body_to_scan(m, c['v'][:, ::4].contiguous(), init=init, iterations=20, **kw),
        'keypoints': lambda **kw: fit_body_to_keypoints(m, c['joints'], init=dict(init), iterations=20, **kw),
        'keypoints_2d': lambda **kw: fit_body_to_keypoints_2d(m, c['proj'], init=dict(init), iterations=20, **kw),
    }


@pytest.mark.parametrize('which', ['scan', 'keypoints', 'keypoints_2d'])
def test_weight_zero_is_the_fit_without_the_term(which):
    c = _setup()
    fit = _fits(c)[which]
    a, b = fit(), fit(penetration_weight=0.0, **c['pen'])
    assert a.keys() == b.keys() and 'penetration' not in a
    for k in a:
        if torch.is_tensor(a[k]):
            assert torch.equal(a[k], b[k]), k


def _penetration_of(c, res, sigma):
    """(penetration, pairs) of a fit's result, recomputed on its posed vertices with the part filter."""
    m = c['model']
    with torch.no_grad():
        v = m(global_rot=res['global_rot_mat'], body_pose=res['body_pose_mat'], betas=res['betas'],
              transl=res.get('transl'), return_shaped=False)['vertices'].contiguous()
    pairs, count = ops.self_collisions(v, m.faces_i32, 1024, **c['pen'])
    return ops.penetration_forward(v, m.faces_i32, pairs, sigma).cpu().numpy(), count.cpu().numpy()


@pytest.mark.parametrize('which', ['scan', 'keypoints', 'keypoints_2d'])
def test_term_reports_its_final_value(which):
    c = _setup()
    res = _fits(c)[which](penetration_weight=0.1, penetration_sigma=0.02, **c['pen'])
    q, n = _penetration_of(c, res, 0.02)
    np.testing.assert_allclose(res['penetration'].cpu().numpy(), q, rtol=1e-6)
    assert (res['penetration_pairs'].cpu().numpy() == n).all() and (n > 0).all()


def test_scan_term_separates_intersecting_limbs():
    """The scan of a self-intersecting body holds the fit there at weight 0; the term pushes the limbs apart."""
    c = _setup()
    fit = _fits(c)['scan']
    sigma = 0.02
    p0, n0 = _penetration_of(c, fit(), sigma)
    res = fit(penetration_weight=0.1, penetration_sigma=sigma, **c['pen'])
    p1, n1 = res['penetration'].cpu().numpy(), res['penetration_pairs'].cpu().numpy()
    print('scan penetration', p0, '->', p1, 'pairs', n0, '->', n1)
    assert (n0 > 0).all() and (p0 > 0).all()
    assert (p1 < p0).all() and (n1 < n0).all()


def test_unsupported_fits_raise_before_any_launch():
    c = _setup()
    m, init = c['model'], c['init']
    n0 = _lib.lib().shapy_launch_count()
    with pytest.raises(ValueError):
        fit_body_to_keypoints(m, c['joints'], method='lm', penetration_weight=1.0)
    with pytest.raises(ValueError):
        fit_body_to_keypoints_2d(m, c['proj'], method='lm', penetration_weight=1.0)
    with pytest.raises(ValueError):
        fit_body_to_keypoints_2d(m, c['proj'], groups=torch.tensor([0, 0]), penetration_weight=1.0)
    with pytest.raises(ValueError):
        fit_body_to_scan(m, c['v'], penetration_weight=1.0, max_penetration_pairs=ops.MAX_PENETRATION_PAIRS + 1)
    assert _lib.lib().shapy_launch_count() == n0
