"""CPU restatement of the reference's result-video drawing (getResultsYcb, predict.py:424-433; predictSequenceYcb /
predictSequenceYcbInEOAT, predict.py:549-560, 612-624) with cv2 itself: cvtColor, putText, circle, resize.

The model points are moved by the pose with x' = ((R00 x + R01 y) + R02 z) + t0 (numpy fp64, which never fuses a multiply-add)
and placed as project_points (predict.py:81-86) places them.  A point whose u or v is not finite or beyond +-2^30 is left out
before drawing (the reference would hand cv2 whatever astype(np.int32) makes of it; none of those lands on the image).
"""
import cv2
import numpy as np

MAX_COORD = 2.0 ** 30


def transform(points, pose):
    """(m,3) float64 model points moved by a 4x4 pose, each row summed left to right."""
    p = np.asarray(points, dtype=np.float64)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    T = np.asarray(pose, dtype=np.float64)
    return np.stack([((T[r, 0] * x + T[r, 1] * y) + T[r, 2] * z) + T[r, 3] for r in range(3)], 1)


def project(points, K, pose):
    """(uv int32 (k,2)) of the drawn points: u = (x' fx) / z' + cx, v = (y' fy) / z' + cy, rounded half to even."""
    q = transform(points, pose)
    K = np.asarray(K, dtype=np.float64)
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        u = np.round(np.divide(q[:, 0] * K[0, 0], q[:, 2]) + K[0, 2])
        v = np.round(np.divide(q[:, 1] * K[1, 1], q[:, 2]) + K[1, 2])
    keep = (np.abs(u) <= MAX_COORD) & (np.abs(v) <= MAX_COORD)
    return np.stack([u[keep], v[keep]], 1).astype(np.int32)


def draw(frame_rgb, uvs, text, order):
    """The half-size BGR image of one track: the label `text` (None: no label) 'under' the points, as getResultsYcb draws it, or
    'over' them, as predictSequenceYcb / YcbInEOAT draw it."""
    H, W = frame_rgb.shape[:2]
    bgr = cv2.cvtColor(np.ascontiguousarray(frame_rgb), cv2.COLOR_RGB2BGR)

    def label():
        if text is not None:
            cv2.putText(bgr, text, (W // 2, H - 50), cv2.FONT_HERSHEY_SIMPLEX, fontScale=1, thickness=4, color=(255, 0, 0))
    if order == 'under':
        label()
    for u, v in uvs:
        cv2.circle(bgr, (int(u), int(v)), radius=1, color=(0, 255, 255), thickness=-1)
    if order == 'over':
        label()
    return cv2.resize(bgr, (W // 2, H // 2))


def draw_track(frame_rgb, K, pose, points, text, order):
    return draw(frame_rgb, project(points, K, pose), text, order)
