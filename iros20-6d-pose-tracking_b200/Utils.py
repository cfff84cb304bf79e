"""Drop-ins for the three reference Utils.py functions on the per-frame path, computed on the
GPU through libse3tn (numpy in / numpy out like the originals):

  compute_bbox               reference Utils.py:302-316
  crop_bbox                  reference Utils.py:320-359 (with or without the seg plane)
  normalize_rotation_matrix  reference Utils.py:363-367 (9 flops: stays numpy)
  add / adi                  reference Utils.py:72-98 (ADD, ADD-S); `model` is anything with `.points` or an (m,3) array
  random_direction / random_gaussian_magnitude   reference Utils.py:372-404 (host RNG draws: stay on the host, same order)
"""
import math
import random

import numpy as np
import torch

_engine = None


def set_engine(engine):
    """Share one Engine (and its device) with the Tracker instead of creating a private one."""
    global _engine
    _engine = engine


def _eng():
    global _engine
    if _engine is None:
        from .engine import Engine
        _engine = Engine(max_batch=1)
    return _engine


def compute_bbox(pose, K, scale_size=230, scale=(1, 1, 1)):
    eng = _eng()
    poses = torch.from_numpy(np.ascontiguousarray(pose, dtype=np.float64).reshape(1, 4, 4)).to(eng.device)
    widths = torch.tensor([float(scale_size)], dtype=torch.float64, device=eng.device)
    out = eng.compute_bbox(poses, K, widths, scale=tuple(float(s) for s in scale))
    return out[0].cpu().numpy()


def crop_bbox(color, depth, boundingbox, output_size=(100, 100), seg=None):
    """-> (rgb, depth), or (rgb, depth, seg) when seg (uint8 (H,W) labels) is given: the labels cropped through the same window
    and nearest mapping, zero outside the image (Utils.py:346-349)."""
    eng = _eng()
    rgb = torch.from_numpy(np.ascontiguousarray(color, dtype=np.uint8)).to(eng.device)
    d = torch.from_numpy(np.ascontiguousarray(depth).astype(np.uint16)).to(eng.device)
    bb = torch.from_numpy(np.ascontiguousarray(boundingbox, dtype=np.int32).reshape(1, 4, 2)).to(eng.device)
    out_hw = (int(output_size[1]), int(output_size[0]))            # cv2.resize takes (width, height)
    if seg is None:
        crgb, cdepth = eng.crop_bbox(rgb, d, bb, out_hw=out_hw)
        return crgb[0].cpu().numpy(), cdepth[0].cpu().numpy()
    seg = np.asarray(seg)
    if seg.dtype != np.uint8:
        raise ValueError('seg must be a uint8 label image (the reference crops it into a uint8 canvas, Utils.py:331)')
    s = torch.from_numpy(np.ascontiguousarray(seg)).to(eng.device)
    crgb, cdepth, cseg, _ = eng.crop_bbox_seg(rgb, d, s, bb, out_hw=out_hw)
    return crgb[0].cpu().numpy(), cdepth[0].cpu().numpy(), cseg[0].cpu().numpy()


def random_direction():
    """Utils.py:394-404: a uniform direction on the unit sphere from two random.uniform draws (theta, then phi)."""
    theta = random.uniform(0, 1) * math.pi * 2
    phi = math.acos((2 * (random.uniform(0, 1))) - 1)
    p = np.zeros(3)
    p[0] = 1 * math.sin(phi) * math.cos(theta)
    p[1] = 1 * math.sin(phi) * math.sin(theta)
    p[2] = 1 * math.cos(phi)
    return p


def random_gaussian_magnitude(max_T, max_R):
    """Utils.py:372-390, in the reference's draw order: translation direction (random), its magnitude (np.random.normal, redrawn
    until |m| <= max_T), rotation direction (random), its magnitude in degrees (redrawn until |m| <= max_R), R = cv2.Rodrigues.
    Host only: after random.seed(s); np.random.seed(s) it returns the reference's matrices bit for bit."""
    import cv2
    direction_T = random_direction()
    while 1:
        magn_T = np.random.normal(0, max_T)
        if abs(magn_T) <= max_T:
            break
    T = direction_T * magn_T
    direction_R = random_direction()
    direction_R = direction_R / np.linalg.norm(direction_R)
    while 1:
        magn_R = np.random.normal(0, max_R)
        if abs(magn_R) <= max_R:
            break
    rod = direction_R * magn_R / 180.0 * np.pi
    R = cv2.Rodrigues(rod)[0].reshape(3, 3).copy()
    pose = np.eye(4)
    pose[:3, :3] = R
    pose[:3, 3] = T.copy()
    return pose


def normalize_rotation_matrix(R):
    R[:, 0] = R[:, 0] / np.linalg.norm(R[:, 0])
    R[:, 1] = R[:, 1] / np.linalg.norm(R[:, 1])
    R[:, 2] = R[:, 2] / np.linalg.norm(R[:, 2])
    return R


def _model_points(model):
    pts = np.asarray(model.points if hasattr(model, 'points') else model, dtype=np.float64)
    return np.ascontiguousarray(pts.reshape(-1, 3))


def add(pred, gt, model):
    eng = _eng()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(eng.device)
    out, _ = eng.add_adi(t(_model_points(model)), t(np.asarray(pred).reshape(1, 4, 4)), t(np.asarray(gt).reshape(1, 4, 4)), want_adi=False)
    return float(out[0].item())


def adi(pred, gt, model):
    eng = _eng()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(eng.device)
    _, out = eng.add_adi(t(_model_points(model)), t(np.asarray(pred).reshape(1, 4, 4)), t(np.asarray(gt).reshape(1, 4, 4)), want_add=False)
    return float(out[0].item())


def fill_depth(depth, max_depth=2.0, extrapolate=False, blur_type='bilateral'):
    """Drop-in for reference Utils.py:455-514: depth in METRES (any float array, as the reference takes it) -> float32 metres,
    computed by libse3tn.  The pipeline quantises the input to whole millimetres first -- exact for the ROS node's
    `uint16 / 1e3` input (predict_ros.py:38-41)."""
    if blur_type not in ('bilateral', 'gaussian'):
        raise ValueError("blur_type must be 'bilateral' or 'gaussian'")           # the reference silently skips the blur for anything else
    eng = _eng()
    mm = np.rint(np.asarray(depth, dtype=np.float64) * 1e3)
    if mm.min() < 0 or mm.max() > 65535:
        raise ValueError('depth must be within 0 .. 65.535 m')
    _, out_m = eng.fill_depth(torch.from_numpy(mm.astype(np.uint16)).to(eng.device), max_depth=max_depth, want_metres=True,
                              extrapolate=extrapolate, blur_type=blur_type)
    return out_m.cpu().numpy()


class Compose(object):
    """Utils.py:517-524: transforms applied in order.  A chain of data_augmentation's classes is what
    TrackDataset(augmentations=...) takes; it runs on the device, not through this __call__."""
    def __init__(self, transforms):
        self.transforms = transforms

    def __call__(self, img):
        for t in self.transforms:
            img = t(img)
        return img
