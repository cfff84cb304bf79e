"""The reference's train-time augmentations of input B (data_augmentation.py:48-121, 217-267) restated with the draws passed in.

augment() applies HSVJitter, ChangeBright, GaussianNoise, GaussianBlur and BlackCover in train.py:85-92's order to one pair,
taking every random value from `params` (se3tn_augment_draws' layout, include/se3tn.h SE3TN_AUG_*) and the two GaussianNoise
fields instead of np.random / random.  The arithmetic is the reference classes' own: cv2 for the colour conversions and the blur,
numpy's dtype chain for the rest.  A float64 stored into a uint8 / uint16 array keeps the low bits of its truncation (what numpy
does on x86-64; numpy 1.x stores BlackCover's -9999 as 55537), spelt out in store() so that the result does not hang on numpy's
casting warnings.

philox_uniform / cover_corners restate the device's draws of BlackCover's corners (csrc/augment.cuh), so that a test can replay the
reference's corner loop over the very corners the device drew.  case_inputs makes the inputs of the golden fixture
(make_golden_augment.py, tests/golden/golden_augment.npz) from a seed.
"""
import cv2
import numpy as np

HSV_ON, HSV_BRANCH, HSV_MAG, BRIGHT_ON, BRIGHT = 0, 1, 4, 7, 8
NOISE_RGB_BRANCH, NOISE_RGB_STD, NOISE_DEPTH_BRANCH, NOISE_DEPTH_STD = 9, 10, 11, 12
BLUR_RGB_BRANCH, BLUR_RGB_K, BLUR_DEPTH_BRANCH, BLUR_DEPTH_K = 13, 14, 15, 16
COVER_BRANCH, COVER_U, COVER_V, COVER_QUADRANT, COVER_CORNERS, COVER_VALID, COVER_REMAINED = 17, 18, 19, 20, 21, 22, 23
N_PARAMS = 24
DEPTH_COVER = 55537                      # -9999 stored into uint16


def store(x, dtype):
    """numpy's float64 -> uint8 / uint16 store on x86-64: truncate toward zero, keep the low bits."""
    return np.asarray(x, dtype=np.float64).astype(np.int64).astype(dtype)


def cover_slices(u, v, q):
    """BlackCover's quadrant q at corner (u, v) as (rows, cols) slices (data_augmentation.py:237-252)."""
    rows = slice(None, v) if q in (0, 1) else slice(v, None)
    cols = slice(None, u) if q in (0, 2) else slice(u, None)
    return rows, cols


def augment(rgbB, depthB, maskB, params, noise_rgb=None, noise_depth=None):
    """One pair: rgbB uint8 (176,176,3), depthB uint16 (176,176), maskB uint8 (176,176) (segB, or depthB > 100) -> the augmented
    (rgbB, depthB, maskB), new arrays.  params: the pair's SE3TN_AUG_PARAMS draws; noise_rgb / noise_depth: its N(0, std) fields
    (needed only when a GaussianNoise branch is taken)."""
    p = np.asarray(params, dtype=np.float64)
    rgbB, depthB, maskB = rgbB.copy(), depthB.copy(), maskB.copy()
    if p[HSV_ON]:                                                            # HSVJitter, :55-70
        mask = depthB > 100
        hsv = cv2.cvtColor(rgbB, cv2.COLOR_RGB2HSV).astype(np.float32)
        for c in range(3):
            if p[HSV_BRANCH + c]:
                hsv[:, :, c] += float(p[HSV_MAG + c])   # a python float joins float32 arithmetic as float32
        hsv = np.clip(hsv, 0, 255)
        rgbB[mask] = cv2.cvtColor(hsv.astype(np.uint8), cv2.COLOR_HSV2RGB)[mask]
    if p[BRIGHT_ON]:                                                         # ChangeBright, :77-81
        rgbB = np.clip(rgbB * float(p[BRIGHT]), 0, 255).astype(np.uint8)
    mask = depthB > 100                                                      # GaussianNoise, :91-102
    if p[NOISE_RGB_BRANCH]:
        rgbB[mask] = store(rgbB[mask] + noise_rgb[mask], np.uint8)
    if p[NOISE_DEPTH_BRANCH]:
        depthB[mask] = store(depthB[mask] + noise_depth[mask], np.uint16)
    if p[BLUR_RGB_BRANCH]:                                                   # GaussianBlur, :111-121
        k = int(p[BLUR_RGB_K])
        rgbB = cv2.GaussianBlur(rgbB, (k, k), sigmaX=2)
    if p[BLUR_DEPTH_BRANCH]:
        k = int(p[BLUR_DEPTH_K])
        depthB = cv2.GaussianBlur(depthB, (k, k), sigmaX=2)
    if p[COVER_BRANCH] and p[COVER_QUADRANT] >= 0:                           # BlackCover, :223-267, the accepted corner
        rows, cols = cover_slices(int(p[COVER_U]), int(p[COVER_V]), int(p[COVER_QUADRANT]))
        rgbB[rows, cols, :] = 0
        depthB[rows, cols] = DEPTH_COVER
        maskB[rows, cols] = 0
    return rgbB, depthB, maskB


def cover_search(maskB, corners):
    """BlackCover's loop (:228-265) over drawn corners [(u, v, first quadrant), ...] -> (u, v, quadrant, corners used), or None when
    every corner fails.  num_valid is the sum of maskB's values, the kept test counts pixels equal to 1, as the reference does."""
    m = np.asarray(maskB).astype(np.uint8)
    num_valid = int(m.sum(dtype=np.int64))
    for a, (u, v, q0) in enumerate(corners):
        for t in range(4):
            q = (q0 + t) % 4
            rows, cols = cover_slices(u, v, q)
            kept = m.copy()
            kept[rows, cols] = 0
            remained = int((kept == 1).sum())
            if not (num_valid and remained / float(num_valid) < 0.5):
                return u, v, q, a + 1
    return None


MASK32 = 0xFFFFFFFF


def philox(ctr, key):
    """Philox4x32-10 of a counter (4 words) and a key (2 words)."""
    x, y, z, w = ctr
    k0, k1 = key
    for _ in range(10):
        p0, p1 = 0xD2511F53 * x, 0xCD9E8D57 * z
        x, y, z, w = ((p1 >> 32) ^ y ^ k0) & MASK32, p1 & MASK32, ((p0 >> 32) ^ w ^ k1) & MASK32, p0 & MASK32
        k0, k1 = (k0 + 0x9E3779B9) & MASK32, (k1 + 0xBB67AE85) & MASK32
    return x, y, z, w


def philox_uniform(seed, pair, slot):
    """The device's scalar draw `slot` of pair `pair`: a 53-bit uniform in [0, 1)."""
    pair &= (1 << 64) - 1
    x, y, _, _ = philox((pair & MASK32, pair >> 32, 0, slot), (seed & MASK32, (seed >> 32) & MASK32))
    return ((x >> 5) * 67108864.0 + (y >> 6)) * (1.0 / 9007199254740992.0)


def philox_randint(seed, pair, slot, count):
    return min(int(philox_uniform(seed, pair, slot) * count), count - 1)


CORNER_SLOT = 16


def cover_corners(seed, pair, count):
    """The first `count` corners (u, v, first quadrant) the device draws for BlackCover in pair `pair`."""
    return [(philox_randint(seed, pair, CORNER_SLOT + 3 * a, 176), philox_randint(seed, pair, CORNER_SLOT + 3 * a + 1, 176),
             philox_randint(seed, pair, CORNER_SLOT + 3 * a + 2, 4)) for a in range(count)]


def case_inputs(seed, seg_kind):
    """One golden case's rgbB uint8 (176,176,3), depthB uint16 (176,176), maskB uint8 (176,176) and its rgbA.  The images are
    smooth (they compress) with saturated patches under the mask (the rgb noise wraps there) and a band of depth at 95..105 mm.
    seg_kind: 'seg' a 0/1 disc, 'none' maskB = depthB > 100 (no segB file), 'two' a disc of 1 with a ring of 2 (num_valid counts
    the 2s twice, so whole corners can fail the keep test)."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[:176, :176].astype(np.float64)
    cy, cx, r = rng.uniform(50, 126), rng.uniform(50, 126), rng.uniform(25, 45)
    d2 = (yy - cy) ** 2 + (xx - cx) ** 2
    rgb = np.stack([(xx * 1.4 + 10 * c) % 256 for c in range(3)], -1)
    rgb = np.clip(rgb + rng.integers(0, 3, rgb.shape), 0, 255).astype(np.uint8)
    rgb[20:40, 20:60] = 255
    rgb[130:150, 100:140] = 0
    depth = (600 + 3 * yy + 2 * xx).astype(np.uint16)
    depth[d2 < r * r] -= 200
    depth[:6] = (95 + xx[:6] % 11).astype(np.uint16)
    depth[160:, :30] = 0
    if seg_kind == 'none':
        mask = (depth > 100).astype(np.uint8)
    else:
        mask = (d2 < r * r).astype(np.uint8)
        if seg_kind == 'two':
            mask[(d2 >= r * r) & (d2 < (1.15 * r) ** 2)] = 2
    return rgb, depth, mask, np.zeros((176, 176, 3), np.uint8)
