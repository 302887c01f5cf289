"""OpenPose detections into the fit's frame (host, NumPy): read, threshold, box, crop and map onto the model's keypoints.

    from shapy_b200 import keypoints2d as k2d
    kp = k2d.read_openpose('img_00.json')                              # (people, 135, 3): x, y, confidence
    m = k2d.load_keypoint_map('openpose_smplx_map.json')
    kp = k2d.threshold_confidence(kp, m)                               # per-part thresholds, binarised
    center, scale = k2d.bbox_from_keypoints(kp)                        # the crop descriptor InputStage takes
    crop = k2d.to_crop(kp, center, scale, 256)                         # normalised crop frame of proj_joints
    targets, weights = k2d.map_keypoints(crop, m, body_model.K)        # (people, K, 2), (people, K)
    fit_body_to_keypoints_2d(body_model, targets, weights, ...)

The layout is the reference's read_keypoints (data/utils/keypoints.py): 25 body, 21 left hand, 21 right hand and 68 face
points per person (the last two of OpenPose's 70 face points dropped), a missing part filled with zeros.  The
thresholds, the box and the crop follow the reference's OpenPose dataset (datasets/openpose.py), Keypoints2D.crop and
normalize, and bbox_to_center_scale.  Which OpenPose point is which model keypoint, and which points belong to which
part, come from the reference's name tables; they are data, passed in as a keypoint map: a JSON object with 'pairs'
([model keypoint, OpenPose keypoint] index pairs), 'parts' (index lists 'body', 'left_hand', 'right_hand', 'face'),
'thresholds' ({'body', 'hand', 'face'}) and 'bbox_scale_factor'.
"""
import json

import numpy as np

NUM_OPENPOSE = 135          # 25 body + 21 + 21 hand + 68 face
_PARTS = (('pose_keypoints_2d', 25), ('hand_left_keypoints_2d', 21), ('hand_right_keypoints_2d', 21),
          ('face_keypoints_2d', 70))


def read_openpose(path):
    """(people, 135, 3) float32 [x, y, confidence] of an OpenPose JSON file; a part a person lacks is zeros, and a file
    without people gives (0, 135, 3)."""
    with open(path) as f:
        data = json.load(f)
    people = []
    for person in data.get('people', []):
        rows = []
        for key, n in _PARTS:
            v = person.get(key, [])
            if len(v) < 1:
                v = [0] * (n * 3)
            rows.append(np.asarray(v, dtype=np.float32).reshape(-1, 3))
        rows[-1] = rows[-1][:-2]
        people.append(np.concatenate(rows, 0))
    if not people:
        return np.zeros((0, NUM_OPENPOSE, 3), np.float32)
    return np.stack(people)


def load_keypoint_map(path):
    with open(path) as f:
        return json.load(f)


def threshold_confidence(keypoints, keypoint_map, binarize=True):
    """The confidences of keypoints (..., 135, 3) as the reference's OpenPose dataset sets them: clipped to [0, 1],
    zeroed below the part's threshold, then (binarize) 1 where at or above it.  The parts are applied in the order
    body, left hand, right hand, face, so a point listed in two parts (a wrist) ends with the later part's value.
    Returns a copy."""
    kp = np.array(keypoints, dtype=np.float32, copy=True)
    kp[..., 2] = np.clip(kp[..., 2], 0, 1)
    th = keypoint_map['thresholds']
    parts = keypoint_map['parts']
    new = []
    for name, t in (('body', th['body']), ('left_hand', th['hand']), ('right_hand', th['hand']),
                    ('face', th['face'])):
        idx = np.asarray(parts[name], np.int64)
        c = kp[..., idx, 2].copy()
        if t > 0:
            c[c < t] = 0.0
        if binarize:
            c = (c >= t if t > 0 else c > 0).astype(np.float32)
        new.append((idx, c))
    for idx, c in new:
        kp[..., idx, 2] = c
    return kp


def bbox_from_keypoints(keypoints, scale_factor=1.2, min_valid=6):
    """(center (P, 2), scale (P,)) of the square crop around each person's confident keypoints, as the reference's
    keyps_to_bbox -> bbox_to_center_scale: the box of the points with confidence > 0, its larger side times
    scale_factor is the crop size, scale = size / 200.  A person with fewer than min_valid such points, or a box of
    zero area, gets NaN."""
    kp = np.asarray(keypoints, np.float32)
    single = kp.ndim == 2
    kp = kp[None] if single else kp
    center = np.full((kp.shape[0], 2), np.nan, np.float32)
    scale = np.full(kp.shape[0], np.nan, np.float32)
    for p in range(kp.shape[0]):
        v = kp[p, kp[p, :, 2] > 0, :2]
        if len(v) < min_valid:
            continue
        (xmin, ymin), (xmax, ymax) = v.min(0), v.max(0)
        w, h = xmax - xmin, ymax - ymin
        xc, yc = 0.5 * (xmax + xmin), 0.5 * (ymax + ymin)
        box = np.stack([xc - 0.5 * w, yc - 0.5 * h, xc + 0.5 * w, yc + 0.5 * h]).astype(np.float32)
        if not abs((box[2] - box[0]) * (box[3] - box[1])) > 0:
            continue
        scale[p] = scale_factor * max(box[2] - box[0], box[3] - box[1]) / 200
        center[p] = np.stack([(box[0] + box[2]) * 0.5, (box[1] + box[3]) * 0.5]).astype(np.float32)
    return (center[0], scale[0]) if single else (center, scale)


def to_crop(keypoints, center, scale, size, round_to_pixel=True):
    """Pixel keypoints (..., N, 2 or 3) into the normalised [-1, 1] frame of a size x size crop with the (center,
    scale = box / 200) descriptor InputStage crops the image with: the reference's Keypoints2D.crop (its get_transform
    in float32, then + 1 and, with round_to_pixel, truncated to integer pixels as it does) and normalize (2 x / size - 1).
    A confidence column is kept as it is."""
    kp = np.asarray(keypoints, np.float32)
    center = np.asarray(center, np.float32).reshape(-1, 2)
    scale = np.asarray(scale, np.float32).reshape(-1)
    flat = kp.reshape(-1, kp.shape[-2], kp.shape[-1])
    if center.shape[0] == 1 and flat.shape[0] > 1:
        center, scale = np.repeat(center, flat.shape[0], 0), np.repeat(scale, flat.shape[0])
    out = flat.copy()
    for p in range(flat.shape[0]):
        h = 200 * scale[p]                                        # float32, as the reference's scale
        t = np.zeros((2, 3), np.float32)                          # get_transform's first two rows, in float32
        t[0, 0], t[1, 1] = float(size) / h, float(size) / h
        t[0, 2] = size * (-float(center[p, 0]) / h + .5)
        t[1, 2] = size * (-float(center[p, 1]) / h + .5)
        xy = np.dot(flat[p, :, :2], t[:, :2].T) + t[:, 2] + 1
        if round_to_pixel:
            xy = xy.astype(np.int64)
        xy = xy.astype(np.float32)
        xy[:, 0] = 2.0 * xy[:, 0] / size - 1.0
        xy[:, 1] = 2.0 * xy[:, 1] / size - 1.0
        out[p, :, :2] = xy
    return out.reshape(kp.shape)


def map_keypoints(keypoints, keypoint_map, num_keypoints):
    """Scatters OpenPose points (P, 135, 3) onto the model's num_keypoints keypoints: (targets (P, K, 2), weights
    (P, K)), the weight the point's confidence (after threshold_confidence); a keypoint no pair maps, or that a pair maps
    past num_keypoints, gets weight 0 and a NaN target (fit_body_to_keypoints_2d never reads it)."""
    kp = np.asarray(keypoints, np.float32)
    kp = kp[None] if kp.ndim == 2 else kp
    P = kp.shape[0]
    targets = np.full((P, num_keypoints, 2), np.nan, np.float32)
    weights = np.zeros((P, num_keypoints), np.float32)
    for t, s in keypoint_map['pairs']:
        if t < num_keypoints:
            targets[:, t] = kp[:, s, :2]
            weights[:, t] = kp[:, s, 2]
    targets[weights <= 0] = np.nan
    return targets, weights
