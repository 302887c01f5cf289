"""GPU: the scan LM step with self-penetration rows (ops.fit_lm_scan_step(penetration=...)) against
tests/scan_pen_lm_oracle.py step by step, and fit_body_to_scan(method='lm', penetration_weight=...) from a
self-intersecting start: non-increasing loss, no host synchronisation and a lower penetration."""
import math

import numpy as np
import pytest
import torch

import lm_harness as H
import scan_lm_oracle as so
import scan_pen_lm_oracle as spo
from penetration_oracle import smooth_smplx
from test_gpu_fit_scan_lm import _check, _evaluate, _scan_case, _state
from shapy_b200 import ops

pytestmark = pytest.mark.gpu

C, PW, PS = 64, 0.5, 0.02


def _pairs(m, v):
    return ops.self_collisions(v, m.faces_i32, C)[0]


def _step(m, state, trial, pts, w, ev, pairs, first):
    B, N = pts.shape[:2]
    P = 66 + m.num_betas + 3
    ws = ops.fit_lm_scan_penetration_workspace(B, N, m.packed().V, P, C, 'cuda')
    ops.fit_lm_scan_step(state, trial, pts, w, m.faces_i32, None, 1.0, 1.0, 0.0, 0.0, 10.0, 3.0, first, *ev, ws,
                         penetration=(pairs, PW, PS))


def _oracle(m, s0, trial0, pts, w, ev, pairs, first):
    v, jac, face, bary, nearest = [t.cpu().numpy() for t in ev]
    faces = m.faces_tensor.cpu().numpy()
    B, N = pts.shape[:2]
    P, V = 66 + m.num_betas + 3, v.shape[1]
    ns = math.ceil(N / so.CHUNK)
    out = []
    for b in range(B):
        chunks = so.rows(v[b], jac[b], pts[b].cpu().numpy(), w[b].cpu().numpy(), faces, face[b], bary[b], nearest[b],
                         math.inf, P)
        pen = spo.pen_rows(v[b], jac[b], faces, pairs[b].cpu().numpy(), PW, PS, P)
        assert sum(L for _, _, L in pen) > 0
        st = {k: t[b].cpu().numpy() for k, t in s0.items()}
        st['accepted'] = int(s0['accepted'][b])
        tr = {k: t[b].cpu().numpy() for k, t in trial0.items()}
        out.append(spo.lm_scan_pen_step(st, tr, chunks, ns, pen, w[b].cpu().numpy(), V, 1.0, 1.0, 10.0, 3.0, first))
    return out


def test_step_matches_oracle_first_accept_reject():
    B, N = 2, 1500
    m, pts, w, trial = _scan_case(B, N, 11)
    P, nb = 66 + m.num_betas + 3, m.num_betas
    state = _state(B, P, nb)
    flags = []
    for it in range(5):
        t0 = {k: v.clone() for k, v in trial.items()}
        s0 = {k: v.clone() for k, v in state.items()}
        ev = _evaluate(m, trial, pts, w, 1.0)
        pairs = _pairs(m, ev[0])
        _step(m, state, trial, pts, w, ev, pairs, it == 0)
        flags.append(_check(state, trial, _oracle(m, s0, t0, pts, w, ev, pairs, it == 0)))
        if it == 0:
            trial['transl'][1] += 0.3           # body 1's next trial moved away
    # every step checked, the first accepted by both bodies, and at least one later trial rejected
    assert all(flags[0]) and any(not a for f in flags[1:] for a in f), flags


def test_weight_zero_rows_are_the_step_without_the_term():
    B, N = 2, 1500
    m, pts, w, trial = _scan_case(B, N, 21)
    P, nb = 66 + m.num_betas + 3, m.num_betas
    ev = _evaluate(m, trial, pts, w, 1.0)
    runs = []
    for pen in (None, (_pairs(m, ev[0]), 0.0, PS)):
        st, tr = _state(B, P, nb), {k: v.clone() for k, v in trial.items()}
        ws = ops.fit_lm_scan_penetration_workspace(B, N, m.packed().V, P, C, 'cuda')
        ops.fit_lm_scan_step(st, tr, pts, w, m.faces_i32, None, 1.0, 1.0, 0.0, 0.0, 10.0, 3.0, True, *ev, ws,
                             penetration=pen)
        runs.append((st, tr))
    for k in runs[0][0]:
        assert torch.equal(H.bits(runs[0][0][k]), H.bits(runs[1][0][k])), k
    for k in runs[0][1]:
        assert torch.equal(H.bits(runs[0][1][k]), H.bits(runs[1][1][k])), k


def test_iteration_without_host_sync():
    B, N = 2, 1000
    m, pts, w, trial = _scan_case(B, N, 41, nan_dropped=False)
    P, nb = 66 + m.num_betas + 3, m.num_betas
    state = _state(B, P, nb)
    ws = ops.fit_lm_scan_penetration_workspace(B, N, m.packed().V, P, C, 'cuda')
    tree = ops.ScanTree()
    v0 = _evaluate(m, trial, pts, w, 1.0)[0]
    ops.closest_points(v0, m.faces_i32, pts, w, tree)
    ops.self_collisions(v0, m.faces_i32, C, tree)           # sizes the tree's workspace for both queries
    filt = ops.make_part_filter(None, None, m.faces_i32.shape[0], 'cuda')

    def it():
        v, jac = ops.smplx_vertex_jacobian(m.packed(), trial['betas'], trial['rot'], trial['transl'])
        face, bary, _ = ops.closest_points(v, m.faces_i32, pts, w, tree)
        nearest = ops.nearest_points(v, pts, w)[0]
        pairs = ops.self_collisions(v, m.faces_i32, C, tree, part_filter=filt)[0]
        ops.fit_lm_scan_step(state, trial, pts, w, m.faces_i32, None, 1.0, 1.0, 0.0, 0.0, 10.0, 3.0, True, v, jac, face,
                             bary, nearest, ws, penetration=(pairs, PW, PS))
    n, _ = H.launches_without_sync(it)
    assert n >= 6


def _pen_of(m, res, pen, sigma):
    with torch.no_grad():
        v = m(global_rot=res['global_rot_mat'], body_pose=res['body_pose_mat'], betas=res['betas'],
              transl=res['transl'], return_shaped=False)['vertices'].contiguous()
    pairs, count = ops.self_collisions(v, m.faces_i32, 1024, **pen)
    return ops.penetration_forward(v, m.faces_i32, pairs, sigma).cpu().numpy(), count.cpu().numpy()


def test_scan_lm_term_separates_intersecting_limbs():
    """A scan of a self-intersecting body holds the LM fit there at weight 0; the term lowers the penetration at the
    pairs it sees, and every body's loss is non-increasing.  The pair count is printed, not asserted: on this model it
    is dominated by the template's own intersections past the 1 024-row cut, which the term never sees."""
    from scipy.spatial.transform import Rotation
    from shapy_b200.fit import fit_body_to_scan
    from shapy_b200.human_shape.models.body_models.body_models import SMPLX
    m = SMPLX(data_struct=smooth_smplx()).cuda()
    B = 2
    rot = np.tile(np.eye(3, dtype=np.float32), (B, 22, 1, 1))
    for b, ang in enumerate([2.6, 2.4]):
        rot[b, 18] = Rotation.from_rotvec([0, -ang, 0]).as_matrix()
        rot[b, 19] = Rotation.from_rotvec([0, ang, 0]).as_matrix()
    raw = torch.tensor(rot[..., :, :2].reshape(B, 132)).cuda()
    r = ops.decode_rot6d(raw)
    with torch.no_grad():
        v = m(global_rot=r[:, :1], body_pose=r[:, 1:], betas=torch.zeros(B, m.num_betas, device='cuda'),
              return_shaped=False)['vertices']
    pts = v[:, ::4].contiguous()
    init = {'global_rot': raw[:, :6], 'body_pose': raw[:, 6:]}
    pen = dict(part_labels=ops.face_parts(m), ignored_part_pairs=ops.parent_child_part_pairs(m.parents))
    kw = dict(method='lm', iterations=15)
    p0, n0 = _pen_of(m, fit_body_to_scan(m, pts, init=init, **kw), pen, PS)
    term = dict(penetration_weight=PW, penetration_sigma=PS, **pen)
    start = fit_body_to_scan(m, pts, init=init, iterations=0, method='lm', **term)
    res = fit_body_to_scan(m, pts, init=init, **kw, **term)
    p1, n1 = res['penetration'].cpu().numpy(), res['penetration_pairs'].cpu().numpy()
    print('scan lm penetration', p0, '->', p1, 'pairs', n0, '->', n1, 'loss', start['loss'], '->', res['loss'])
    assert bool((res['loss'] <= start['loss'] * (1 + 1e-5) + 1e-9).all())
    assert (p0 > 0).all() and (p1 < p0).all() and (n1 > 0).all()
