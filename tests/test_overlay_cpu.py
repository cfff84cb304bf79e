"""The drawing rules se3tn_draw_tracks restates, checked against cv2 itself (no GPU):
  * the CPU oracle (oracle/overlay_oracle.py) draws what the reference's lines draw on project_points' pixels
    (tests/golden/golden_overlay.npz, written by oracle/make_golden_overlay.py with the reference's own project_points)
  * cv2.resize to half size (INTER_LINEAR) is (a + b + c + d + 2) >> 2 over each 2 x 2 block
  * cv2.circle(radius=1, thickness=-1) sets the plus of 5 pixels, clipped to the image
  * the label strip holds every pixel putText sets for the videos' labels, and predict.label_strip renders exactly those
"""
import importlib, os
import cv2
import numpy as np
import pytest

import overlay_oracle as OV


@pytest.fixture(scope='module')
def pr():
    return importlib.import_module('iros20-6d-pose-tracking_b200.predict')


def halve(img):
    """(a + b + c + d + 2) >> 2 over each 2 x 2 block of a uint8 (H, W, C) image."""
    s = img.astype(np.uint32)
    return ((s[0::2, 0::2] + s[0::2, 1::2] + s[1::2, 0::2] + s[1::2, 1::2] + 2) >> 2).astype(np.uint8)


def plus(H, W, u, v):
    m = np.zeros((H, W), dtype=bool)
    for x, y in ((u, v), (u - 1, v), (u + 1, v), (u, v - 1), (u, v + 1)):
        if 0 <= x < W and 0 <= y < H:
            m[y, x] = True
    return m


def test_oracle_matches_the_reference_fixture(golden_dir):
    g = np.load(os.path.join(golden_dir, 'golden_overlay.npz'))
    for c in range(3):
        for order in ('under', 'over'):
            got = OV.draw_track(g['frame_%d' % c], g['K_%d' % c], g['pose_%d' % c], g['points_%d' % c], str(g['text_%d' % c]), order)
            assert np.array_equal(got, g['out_%d_%s' % (c, order)]), (c, order)
    assert not np.array_equal(g['out_1_under'], g['out_1_over'])      # the fixture's points cross the label


def test_half_size_resize_is_the_rounded_mean_of_each_2x2_block():
    rng = np.random.default_rng(0)
    frames = [np.zeros((480, 640, 3), np.uint8), np.full((480, 640, 3), 255, np.uint8)]
    for k in range(60):                                               # random frames of assorted even sizes
        H, W = 2 * int(rng.integers(1, 120)), 2 * int(rng.integers(1, 160))
        frames.append(rng.integers(0, 256, (H, W, 3), dtype=np.uint8))
    for k in range(30):                                               # saturated 0 / 255 frames
        frames.append((rng.random((96, 128, 3)) < 0.5).astype(np.uint8) * 255)
    for k in range(20):                                               # label edges and dots over a camera-like frame
        f = cv2.resize(rng.integers(0, 256, (30, 40, 3), dtype=np.uint8), (640, 480), interpolation=cv2.INTER_CUBIC)
        cv2.putText(f, 'frame:%d' % rng.integers(0, 10 ** 7), (320, 430), cv2.FONT_HERSHEY_SIMPLEX, fontScale=1, thickness=4, color=(255, 0, 0))
        for u, v in rng.integers(-2, 642, (200, 2)):
            cv2.circle(f, (int(u), int(v)), radius=1, color=(0, 255, 255), thickness=-1)
        frames.append(f)
    assert len(frames) >= 100
    for f in frames:
        H, W = f.shape[:2]
        assert np.array_equal(cv2.resize(f, (W // 2, H // 2)), halve(f)), f.shape


def test_radius_1_filled_circle_is_a_plus_of_5_pixels_clipped_to_the_image():
    H, W = 12, 16
    centres = [(u, v) for u in (-2, -1, 0, 1, W // 2, W - 2, W - 1, W, W + 1) for v in (-2, -1, 0, 1, H // 2, H - 2, H - 1, H, H + 1)]
    for u, v in centres:
        img = np.zeros((H, W, 3), np.uint8)
        cv2.circle(img, (u, v), radius=1, color=(0, 255, 255), thickness=-1)
        assert np.array_equal(img[..., 1] == 255, plus(H, W, u, v)), (u, v)
        assert np.array_equal(img[..., 0], np.zeros((H, W), np.uint8))


def test_label_strip_holds_every_pixel_putText_sets(pr):
    H, W = 480, 640
    rng = np.random.default_rng(1)
    labels = [0, 1, 7, 8, 9, 10, 11, 42, 99, 100, 444, 999, 1000, 1111, 8888, 9999, 10000, 77777, 99999, 100000, 444444, 999999,
              1000000, 8888888, 9999999] + [int(x) for x in rng.integers(0, 10 ** 7, 40)]
    for i in labels:
        text = 'frame:%d' % i
        full = np.zeros((H, W, 3), np.uint8)
        cv2.putText(full, text, (W // 2, H - 50), cv2.FONT_HERSHEY_SIMPLEX, fontScale=1, thickness=4, color=(255, 0, 0))
        rows = np.nonzero(full.any(axis=(1, 2)))[0]
        assert rows.min() >= H - pr.LABEL_TOP and rows.max() < H - pr.LABEL_BOTTOM, (text, rows.min(), rows.max())
        assert set(np.unique(full[..., 0])) <= {0, 255} and not full[..., 1:].any()
        y0, mask = pr.label_strip(text, H, W)
        assert y0 == H - pr.LABEL_TOP and mask.shape == (pr.LABEL_TOP - pr.LABEL_BOTTOM, W)
        assert np.array_equal(mask, full[y0:H - pr.LABEL_BOTTOM, :, 0]), text
    with pytest.raises(ValueError):
        pr.label_strip('frame:1', pr.LABEL_TOP - 2, W)
