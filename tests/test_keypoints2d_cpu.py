"""CPU: shapy_b200.keypoints2d against the reference's own OpenPose reading, thresholds, box and crop on its 22 sample
detections (tests/golden/ref_openpose.npz, written by tools/make_golden.py), and map_keypoints with the reference's
OpenPose -> SMPL-X index map (tests/golden/openpose_smplx_map.json)."""
import json
import os

import numpy as np
import pytest

from shapy_b200 import keypoints2d as k2d

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
REF_SAMPLES = os.path.join(os.environ.get('SHAPY_REFERENCE', '/root/reference'), 'samples', 'openpose')


@pytest.fixture(scope='module')
def ref():
    return np.load(os.path.join(G, 'ref_openpose.npz'))


@pytest.fixture(scope='module')
def kmap():
    return k2d.load_keypoint_map(os.path.join(G, 'openpose_smplx_map.json'))


def _write_json(tmp_path, raw):
    """The person's arrays back into an OpenPose JSON (the fixture stores what read_keypoints returned)."""
    person = {'pose_keypoints_2d': raw[:25].reshape(-1).tolist(), 'hand_left_keypoints_2d': raw[25:46].reshape(-1).tolist(),
              'hand_right_keypoints_2d': raw[46:67].reshape(-1).tolist(),
              'face_keypoints_2d': np.concatenate([raw[67:], np.zeros((2, 3), np.float32)]).reshape(-1).tolist()}
    path = tmp_path / 'kp.json'
    path.write_text(json.dumps({'version': 1.3, 'people': [person]}))
    return str(path)


def test_read_openpose_matches_the_reference(ref, tmp_path):
    """All 22 sample files when the reference tree is there, else each fixture person round-tripped through JSON."""
    files = [str(f) for f in ref['files']]
    for i, fi in enumerate(ref['file_index']):
        path = os.path.join(REF_SAMPLES, files[fi])
        got = k2d.read_openpose(path if os.path.exists(path) else _write_json(tmp_path, ref['raw'][i]))
        assert got.shape == (1, 135, 3) and got.dtype == np.float32
        assert np.array_equal(got[0], ref['raw'][i]), files[fi]


def test_missing_parts_and_empty_files(tmp_path):
    p = tmp_path / 'a.json'
    p.write_text(json.dumps({'people': [{'pose_keypoints_2d': list(range(75))}]}))
    kp = k2d.read_openpose(str(p))
    assert kp.shape == (1, 135, 3) and np.all(kp[0, 25:] == 0) and kp[0, 24, 2] == 74
    p.write_text(json.dumps({'people': []}))
    assert k2d.read_openpose(str(p)).shape == (0, 135, 3)


def test_thresholds_box_and_crop_match_the_reference(ref, kmap):
    thr = k2d.threshold_confidence(ref['raw'], kmap)
    assert np.array_equal(thr, ref['thresholded'])
    center, scale = k2d.bbox_from_keypoints(thr, kmap['bbox_scale_factor'])
    valid = ref['valid'].astype(bool)
    assert valid.sum() == 22
    assert np.abs(center - ref['center']).max() <= 1e-6 * np.abs(ref['center']).max()
    assert np.abs(scale - ref['scale']).max() <= 1e-6 * np.abs(ref['scale']).max()
    crop = k2d.to_crop(thr, center, scale, int(ref['crop_size']))
    assert np.abs(crop - ref['cropped']).max() <= 1e-6


def test_bbox_needs_six_confident_points():
    kp = np.zeros((1, 135, 3), np.float32)
    kp[0, :5] = [[10, 20, 1], [30, 40, 1], [50, 10, 1], [20, 60, 1], [40, 30, 1]]
    c, s = k2d.bbox_from_keypoints(kp)
    assert np.isnan(c).all() and np.isnan(s).all()
    kp[0, 5] = [15, 15, 1]
    c, s = k2d.bbox_from_keypoints(kp)
    assert np.allclose(c[0], [30, 35]) and np.isclose(s[0], 1.2 * 50 / 200)


def test_map_keypoints(kmap):
    kp = np.random.default_rng(0).uniform(size=(2, 135, 3)).astype(np.float32)
    kp[1, :, 2] = 0
    tg, w = k2d.map_keypoints(kp, kmap, 123)
    assert tg.shape == (2, 123, 2) and w.shape == (2, 123)
    mapped = {t for t, s in kmap['pairs']}
    for t, s in kmap['pairs']:
        assert np.array_equal(tg[0, t], kp[0, s, :2]) and w[0, t] == kp[0, s, 2]
    assert all(w[0, k] == 0 and np.isnan(tg[0, k]).all() for k in range(123) if k not in mapped)
    assert (w[1] == 0).all() and np.isnan(tg[1]).all()
    tg, w = k2d.map_keypoints(kp, kmap, 20)                # pairs past K are dropped
    assert tg.shape == (2, 20, 2)


# Median distance in the crop frame between SHAPY's own proj_joints of img_00 and the img_00 OpenPose body detections
# (threshold, box and crop as the reference's OpenPose dataset, 256 px crop) on the 14 confident mapped body joints:
# 0.0529 on first run (deterministic, ~7 px of the crop); the bar sits just above it.  Pairing the same joints in
# reverse order gives a median far above it, so the check sees the correspondence, not just the crop frame.
IMG00_MEDIAN_BAR = 0.055


def test_img00_detections_lie_near_shapys_projection(ref, kmap):
    """The only check against real data: img_00's detections, mapped onto SMPL-X in img_00's crop, against the
    proj_joints SHAPY predicted for that image (tests/golden/img00_body.npz)."""
    body = np.load(os.path.join(G, 'img00_body.npz'))
    i = [str(f) for f in ref['files']].index('img_00.json')
    row = int(np.nonzero(ref['file_index'] == i)[0][0])
    thr = k2d.threshold_confidence(ref['raw'][row:row + 1], kmap)
    center, scale = k2d.bbox_from_keypoints(thr, kmap['bbox_scale_factor'])
    crop = k2d.to_crop(thr, center, scale, 256)
    tg, w = k2d.map_keypoints(crop, kmap, body['proj_joints'].shape[0])
    body_targets = {t for t, s in kmap['pairs'] if s in set(kmap['parts']['body'])}
    keep = [k for k in sorted(body_targets) if w[0, k] > 0]
    d = np.linalg.norm(body['proj_joints'][keep] - tg[0, keep], axis=1)
    wrong = np.linalg.norm(body['proj_joints'][keep] - tg[0, keep[::-1]], axis=1)
    print('img_00: median distance', float(np.median(d)), 'reversed pairs', float(np.median(wrong)))
    assert len(keep) >= 12
    assert float(np.median(d)) <= IMG00_MEDIAN_BAR
    assert float(np.median(wrong)) > 4 * IMG00_MEDIAN_BAR
