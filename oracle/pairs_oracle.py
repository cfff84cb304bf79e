"""CPU oracle of the held-out pair generator: ProducerPurturb.generate (reference produce_train_pair_data.py:86-141).

TEST INFRASTRUCTURE ONLY, like se3_oracle.py: nothing in the product package imports it.

What it restates (file:line relative to the upstream reference tree):

  random_direction / random_gaussian_magnitude   Utils.py:372-404   (the host RNG draws, in the reference's order)
  crop_bbox_seg                                  Utils.py:320-359   (crop_bbox with its seg plane)
  visibility_counts                              produce_train_pair_data.py:97-104
  generate                                       produce_train_pair_data.py:86-141 (arrays instead of files)

on top of se3_oracle's compute_bbox, crop_bbox, render_full_frame_unlit and render_window_pyrender (the pyrender Renderer the
reference's generator uses, restated; see that file for its pinning).  The RNG draws and the seg crop are pinned bit for bit by
tests/golden/golden_pairs.npz, which oracle/make_golden_pairs.py writes with the reference's own Utils functions.
"""
import math
import random

import cv2
import numpy as np

import se3_oracle as O


def random_direction():
    theta = random.uniform(0, 1) * math.pi * 2
    phi = math.acos((2 * (random.uniform(0, 1))) - 1)
    p = np.zeros(3)
    p[0] = 1 * math.sin(phi) * math.cos(theta)
    p[1] = 1 * math.sin(phi) * math.sin(theta)
    p[2] = 1 * math.cos(phi)
    return p


def random_gaussian_magnitude(max_T, max_R):
    direction_T = random_direction()
    while True:
        magn_T = np.random.normal(0, max_T)
        if abs(magn_T) <= max_T:
            break
    direction_R = random_direction()
    direction_R = direction_R / np.linalg.norm(direction_R)
    while True:
        magn_R = np.random.normal(0, max_R)
        if abs(magn_R) <= max_R:
            break
    pose = np.eye(4)
    pose[:3, :3] = cv2.Rodrigues(direction_R * magn_R / 180.0 * np.pi)[0].reshape(3, 3)
    pose[:3, 3] = direction_T * magn_T
    return pose


def crop_bbox_seg(color, depth, boundingbox, output_size, seg):
    """Utils.py:320-359 with seg: (rgb, depth) as se3_oracle.crop_bbox, and seg copied into a uint8 zero canvas through the same
    window, nearest-resized, not masked."""
    rgb, d = O.crop_bbox(color, depth, boundingbox, output_size)
    top, left, crop_h, crop_w = O.crop_window(boundingbox)
    H, W = seg.shape[:2]
    canvas = np.zeros((crop_h, crop_w), dtype=np.uint8)
    y0, y1 = max(top, 0), min(top + crop_h, H)
    x0, x1 = max(left, 0), min(left + crop_w, W)
    cy0, cx0 = abs(min(top, 0)), abs(min(left, 0))
    cy1 = min(crop_h - (top + crop_h - H), crop_h)
    cx1 = min(crop_w - (left + crop_w - W), crop_w)
    canvas[cy0:cy1, cx0:cx1] = seg[y0:y1, x0:x1]
    return rgb, d, cv2.resize(canvas, output_size, interpolation=cv2.INTER_NEAREST)


def visibility_counts(seg, class_id, B_in_cam, K, mesh):
    """(num_visible, covered) of produce_train_pair_data.py:98-102: np.sum(seg == class_id) and np.sum(depth > 0.1) of the
    full-image render (depth float32: 0.1 compares as float32)."""
    H, W = seg.shape
    _, depth = O.render_full_frame_unlit(B_in_cam, K, mesh, H, W)
    return int(np.sum(seg == class_id)), int(np.sum(depth > 0.1))


def visible_enough(num_visible, covered):
    """The reference's two thresholds (produce_train_pair_data.py:99-104), numpy scalar division: covered == 0 gives inf, kept."""
    if num_visible <= 100:
        return False
    with np.errstate(divide='ignore', invalid='ignore'):
        ratio = np.int64(num_visible) / np.float64(covered)
    return not (ratio < 0.1)


def generate(B_in_cam, rgb, depth, seg, num_sample, class_id, K32, object_width, max_trans, max_rot, mesh, check_vis=False,
             size=176):
    """produce_train_pair_data.py:86-141 on arrays.  K32: the float32 cam_K.  -> list, one entry per drawn sample:
    dict(A_in_cam, status: 'centre' (projection outside the image) / 'seg' (< 100 segB pixels) / 'kept', and for the cropped
    samples rgbA, depthA, rgbB, depthB, segB (0/1 uint8) and count).  [] without draws when the visibility check rejects the frame."""
    H, W = seg.shape
    K = K32.astype(np.float64)
    if check_vis and not visible_enough(*visibility_counts(seg, class_id, B_in_cam, K, mesh)):
        return []
    out = []
    for _ in range(num_sample):
        B_in_A = random_gaussian_magnitude(max_trans, max_rot)
        A_in_cam = B_in_cam.dot(np.linalg.inv(B_in_A))
        projected = K32.dot(A_in_cam[:3, 3].reshape(3, 1)).reshape(-1)
        u = projected[0] / projected[2]
        v = projected[1] / projected[2]
        rec = dict(A_in_cam=A_in_cam)
        out.append(rec)
        if u < 0 or u >= W or v < 0 or v >= H:
            rec['status'] = 'centre'
            continue
        bb = O.compute_bbox(A_in_cam, K, object_width, scale=(1000, 1000, 1000))
        rgbA, depthA = O.render_window_pyrender(A_in_cam, K, object_width, mesh, H, W, size)
        rgbB, depthB, segB = crop_bbox_seg(rgb, depth, bb, (size, size), seg)
        count = int(np.sum(segB == class_id))
        rec.update(rgbA=rgbA, depthA=depthA.astype(np.uint16), rgbB=rgbB, depthB=depthB.astype(np.uint16),
                   segB=(segB == class_id).astype(np.uint8), count=count, status='seg' if count < 100 else 'kept')
    return out
