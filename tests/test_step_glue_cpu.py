"""CPU: the restatements tests/test_gpu_step_glue.py compares the fp64 / fp32 glue of a tracking step with, checked against the
oracle's literal restatements, and the inputs the two files share.

* process_predict_exact (oracle/se3_oracle.py) keeps the reference's two float32 steps of the pose update (datasets.py:159-175):
  the Rodrigues matrix rounded to float32 and the translation increment formed in float32.  Dropping either changes nearly
  every element it touches, each by less than 1e-7, so only a bit-for-bit comparison can tell the kernel's chain from a
  float64 one.  The device's cos / sin are not glibc's: a float64 Rodrigues entry within a few ulps of a float32 rounding
  midpoint may round the other way there; exempt_rows() finds those entries, and they are rare.
* crop_bbox_indexed is crop_bbox through cv2's nearest-neighbour index formula, so windows tens of thousands of pixels
  wide can be cut without their canvas.  Such windows have source indices above 32,767.
* edge_frame / edge_views hold every raw depth 0..2100, 65535 and every 8-bit colour, so each entry of the preprocessing
  kernel's per-track tables is read."""
import importlib
import cv2
import numpy as np
import pytest
import se3_oracle as O

synth = importlib.import_module('iros20-6d-pose-tracking_b200.synth')
K = synth.CAMERA_K                                      # the YCB-Video camera
TN, RN = 0.03, 5 * np.pi / 180
NORMALIZERS = [(0.03, 5 * np.pi / 180), (0.02, 15 * np.pi / 180)]     # tracking, validation (dataset_info.yml)
EXEMPT_ULPS = 8
DEPTH_VALUES = np.append(np.arange(2101), 65535).astype(np.uint16)    # LUT edges 100 / 101 and 1999 / 2000, and no reading

# (label, translation, object_width) of the windows the preprocessing tests cut; rotations do not move a window
SPECIAL_TRACKS = [
    ('42671 x 42699 px window', (-0.056, 0.0, 0.005), 200.0),         # frame columns at window columns 32,970 and up
    ('42699 x 42672 px window', (0.0, -0.056, 0.005), 200.0),         # frame rows at window rows 33,064 and up
    ('176 px window', (0.01, 0.02, 1.2079), 200.0),                   # identity resize
    ('window over the top border', (0.0, -0.2, 0.6), 200.0),
    ('window over the bottom border', (0.0, 0.2, 0.6), 200.0),
    ('window over the left border', (-0.25, 0.0, 0.6), 200.0),
    ('window over the right border', (0.25, 0.0, 0.6), 200.0),
    ('window outside the frame', (2.0, 2.0, 0.5), 200.0),
    ('zero-width window', (0.0, 0.0, 0.5), 0.0),
    ('z < 0 (GL pose)', (0.05, 0.03, -0.6), 200.0),
    ('window larger than the frame', (0.0, 0.0, 0.25), 200.0),
    ('far object, 112 px window', (0.01, 0.02, 1.9), 200.0),
]
IDENTITY = 2
CANVAS_LIMIT = 1 << 22                                  # crop_bbox allocates h x w canvases; above this crop_bbox_indexed cuts


def window(pose, width):
    return O.crop_window(O.compute_bbox(pose, K, width, scale=(1000, 1000, 1000)))


def _pose(t):
    p = np.eye(4); p[:3, 3] = t
    return p


# ------------------------------------------------------------------------------------------- shared inputs
def edge_image(rng, size=176):
    """rgb (size,size,3) uint8 and depth (size,size) uint16 holding every colour value per channel and every DEPTH_VALUES entry."""
    depth = rng.permutation(np.resize(DEPTH_VALUES, size * size)).reshape(size, size)
    rgb = np.stack([rng.permutation(np.resize(np.arange(256, dtype=np.uint8), size * size)).reshape(size, size)
                    for _ in range(3)], axis=-1)
    return rgb, depth


def edge_views(n, seed):
    rng = np.random.default_rng(seed)
    views = [edge_image(rng) for _ in range(n)]
    return np.stack([v[0] for v in views]), np.stack([v[1] for v in views])


def edge_frame(seed=0):
    """A synthetic 480 x 640 frame whose block under the 176 px window holds every colour and depth value."""
    rgb, depth = synth.raw_frame(seed)
    top, left, h, w = window(_pose(SPECIAL_TRACKS[IDENTITY][1]), SPECIAL_TRACKS[IDENTITY][2])
    rgb[top:top + h, left:left + w], depth[top:top + h, left:left + w] = edge_image(np.random.default_rng(seed + 100))
    return rgb, depth


def step_tracks(n, seed=0):
    """n tracks, SPECIAL_TRACKS first, then random poses of synth.raw_poses -> (poses, widths, weight ids over two sets, labels)."""
    poses = synth.raw_poses(n, seed=seed)
    widths = np.full(n, 200.0)
    labels = ['random pose'] * n
    for i, (label, t, w) in enumerate(SPECIAL_TRACKS[:n]):
        poses[i, :3, 3] = t; widths[i] = w; labels[i] = label
    widths[len(SPECIAL_TRACKS)::7] = 187.3
    ids = np.random.default_rng(seed + 1).integers(0, 2, n).astype(np.int32)
    return poses, widths, ids, labels


def oracle_crop(rgb, depth, pose, width):
    """crop_bbox where its canvas can be allocated, crop_bbox_indexed otherwise (and for the empty window)."""
    top, left, h, w = window(pose, width)
    bb = O.compute_bbox(pose, K, width, scale=(1000, 1000, 1000))
    if h <= 0 or w <= 0 or h * w > CANVAS_LIMIT:
        return O.crop_bbox_indexed(rgb, depth, bb, (176, 176))
    return O.crop_bbox(rgb, depth, bb, (176, 176))


def pose_update_cases(n=10000, seed=0):
    """(A (n,4,4) float64, trans (n,3) float32, rot (n,3) float32): the network's tanh range, with rot = 0 (the identity
    branch), rot = +-1 on a single axis and rot = (+-1, +-1, +-1)."""
    rng = np.random.default_rng(seed)
    A = synth.raw_poses(n, seed=seed)
    trans = rng.uniform(-1, 1, (n, 3)).astype(np.float32)
    rot = rng.uniform(-1, 1, (n, 3)).astype(np.float32)
    rot[0] = 0
    for k in range(3):
        rot[1 + 2 * k] = 0; rot[1 + 2 * k, k] = 1
        rot[2 + 2 * k] = 0; rot[2 + 2 * k, k] = -1
    rot[7:15] = np.array(np.meshgrid([1, -1], [1, -1], [1, -1])).reshape(3, -1).T
    trans[1:4] = np.eye(3); trans[4:7] = -np.eye(3)
    return A, trans, rot


def near_f32_midpoint(x, ulps=EXEMPT_ULPS):
    """float64 values within `ulps` float64 ulps of a midpoint between two adjacent float32 values."""
    x = np.asarray(x, dtype=np.float64)
    f = x.astype(np.float32)
    g = np.nextafter(f, np.where(x >= f, np.float32(np.inf), np.float32(-np.inf)))
    mid = (f.astype(np.float64) + g.astype(np.float64)) * 0.5            # exact: two float32 values
    return np.abs(x - mid) <= ulps * np.spacing(np.abs(x))


def exempt_rows(rot, rn):
    """(n,3) bool: rotation rows r of the update whose float64 Rodrigues entries R[r, :] (OpenCV's, before the float32
    rounding) lie near a float32 rounding midpoint.  Output element (r, c) of the pose depends on row r of R only."""
    r32 = np.asarray(rot, dtype=np.float32) * np.float32(rn)
    R64 = np.stack([cv2.Rodrigues(r.astype(np.float64))[0] for r in r32])
    return near_f32_midpoint(R64).any(axis=2)


def assert_pose_update_equal(got, want, rot, rn, what):
    """got == want bit for bit, except rotation elements in exempt rows; at most 0.1 % of the rotation elements exempt."""
    ex = exempt_rows(rot, rn)
    assert ex.mean() <= 1e-3, '%s: %.3f %% of the rotation rows exempt' % (what, 100 * ex.mean())
    allowed = np.zeros(got.shape, bool)
    allowed[:, :3, :3] = ex[:, :, None]
    bad = (got != want) & ~allowed
    if bad.any():
        where = np.argwhere(bad)[:8]
        raise AssertionError('%s: %d pose elements differ from process_predict_exact (%d exempt rows); first (track, row, col, '
                             'got, want): %s' % (what, bad.sum(), ex.sum(),
                                                 [(int(i), int(r), int(c), got[i, r, c], want[i, r, c]) for i, r, c in where]))


def near_pi_cases():
    """(rotation vectors (m,3), deltas (m,)): angle pi - delta about axes in all eight octants (x the smallest or the
    largest component) and along +-x, +-y, +-z; the deltas straddle the small-sine branch (s < 1e-5) of the so(3) log."""
    axes = []
    for base in ((1.0, 2.0, 3.0), (3.0, 1.0, 2.0)):
        for sg in np.array(np.meshgrid([1, -1], [1, -1], [1, -1])).reshape(3, -1).T:
            a = np.array(base) * sg
            axes.append(a / np.linalg.norm(a))
    axes += [s * e for e in np.eye(3) for s in (1.0, -1.0)]
    deltas = [1e-9, 1e-7, 5e-6, 9.9e-6, 1.01e-5, 1e-4]
    ws = np.array([(np.pi - d) * a for d in deltas for a in axes])
    return ws, np.repeat(deltas, len(axes))


# ------------------------------------------------------------------------------------------- tests
def test_special_windows_are_what_they_say():
    got = {label: window(_pose(t), w) for label, t, w in SPECIAL_TRACKS}
    H, W = 480, 640
    top, left, h, w = got['176 px window']
    assert (h, w) == (176, 176) and 0 <= top and top + h <= H and 0 <= left and left + w <= W
    assert got['42671 x 42699 px window'] == (-21108, -32970, 42699, 42671)
    assert got['42699 x 42672 px window'] == (-33064, -21023, 42699, 42672)
    assert got['window over the top border'][0] < 0 < got['window over the top border'][0] + got['window over the top border'][2] < H
    assert 0 < got['window over the bottom border'][0] < H < sum(got['window over the bottom border'][0::2])
    assert got['window over the left border'][1] < 0 < got['window over the left border'][1] + got['window over the left border'][3] < W
    assert 0 < got['window over the right border'][1] < W < sum(got['window over the right border'][1::2])
    assert got['window outside the frame'][0] >= H and got['window outside the frame'][1] >= W
    assert got['zero-width window'][2:] == (0, 0)
    assert got['window larger than the frame'][2] > H and got['window larger than the frame'][3] > W


def test_edge_content_covers_every_table_entry():
    rgb, depth = edge_frame()
    rB, dB = oracle_crop(rgb, depth, _pose(SPECIAL_TRACKS[IDENTITY][1]), SPECIAL_TRACKS[IDENTITY][2])
    rgbA, depthA = edge_views(3, seed=1)
    for r, d in [(rB, dB)] + list(zip(rgbA, depthA)):
        assert np.array_equal(np.unique(d), DEPTH_VALUES)
        assert all(np.array_equal(np.unique(r[..., c]), np.arange(256)) for c in range(3))


def test_crop_bbox_indexed_is_crop_bbox():
    rgb, depth = edge_frame()
    poses, widths, _, labels = step_tracks(40, seed=3)
    checked = 0
    for p, w, label in zip(poses, widths, labels):
        top, left, h, cw = window(p, w)
        bb = O.compute_bbox(p, K, w, scale=(1000, 1000, 1000))
        got = O.crop_bbox_indexed(rgb, depth, bb, (176, 176))
        if h <= 0 or cw <= 0:
            assert not got[0].any() and not got[1].any(), label
            continue
        if h * cw > CANVAS_LIMIT:
            continue
        want = O.crop_bbox(rgb, depth, bb, (176, 176))
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), label
        small = O.crop_bbox_indexed(rgb, depth, bb, (100, 120)), O.crop_bbox(rgb, depth, bb, (100, 120))
        assert np.array_equal(small[0][0], small[1][0]) and np.array_equal(small[0][1], small[1][1]), label
        checked += 1
    assert checked >= 35


def test_sixteen_bit_source_indices_lose_frame_pixels():
    """The defect the 16-bit index tables of the preprocessing kernel had: source indices of 32,768 and up wrap negative,
    and frame pixels of the two widest windows turn into zeros."""
    rgb, depth = edge_frame()
    for label, t, w in SPECIAL_TRACKS[:2]:
        top, left, h, cw = window(_pose(t), w)
        sy = np.minimum(np.floor(np.arange(176) * (1.0 / (176 / h))).astype(np.int64), h - 1)
        sx = np.minimum(np.floor(np.arange(176) * (1.0 / (176 / cw))).astype(np.int64), cw - 1)
        assert max(sy.max(), sx.max()) > 32767
        fy, fx = top + sy.astype(np.int16).astype(np.int64), left + sx.astype(np.int16).astype(np.int64)
        ok = ((fy >= 0) & (fy < 480))[:, None] & ((fx >= 0) & (fx < 640))[None, :]
        wrapped = np.where(ok, depth[np.clip(fy, 0, 479)[:, None], np.clip(fx, 0, 639)[None, :]], 0)
        _, want = O.crop_bbox_indexed(rgb, depth, O.compute_bbox(_pose(t), K, w, scale=(1000, 1000, 1000)), (176, 176))
        print('%s: %d of %d frame pixels lost' % (label, (wrapped != want).sum(), (want > 0).sum()))
        assert (wrapped != want).sum() >= 3, label


def test_process_predict_exact_is_process_predict():
    """The restatement against the literal one: translations bit for bit, rotations to the last bits (BLAS's dot)."""
    for tn, rn in NORMALIZERS:
        A, tr, ro = pose_update_cases(500, seed=1)
        got = O.process_predict_exact(A, tr, ro, tn, rn)
        want = np.stack([O.process_predict(A[i], (tr[i], ro[i]), tn, rn) for i in range(len(A))])
        assert np.array_equal(got[:, :, 3], want[:, :, 3]) and np.array_equal(got[:, 3], want[:, 3])
        assert np.abs(got - want).max() <= 4e-16
        assert np.array_equal(got[0, :3, :3], A[0, :3, :3])                 # rot = 0: the identity, exactly


@pytest.mark.parametrize('tn,rn', NORMALIZERS)
def test_float64_shortcuts_hide_below_old_tolerance(tn, rn):
    """Each float32 step of the reference, dropped, changes >= 90 % of the elements it touches, by less than 1e-7."""
    A, tr, ro = pose_update_cases()
    exact = O.process_predict_exact(A, tr, ro, tn, rn)
    r32 = ro * np.float32(rn)
    R64 = np.stack([cv2.Rodrigues(r.astype(np.float64))[0] for r in r32])
    no_r_rounding = O.pose_compose_exact(A, R64, tr * np.float32(tn))
    f64_increment = O.pose_compose_exact(A, np.stack([cv2.Rodrigues(r)[0] for r in r32]), tr.astype(np.float64) * tn)
    for what, mutant, sl in (('R not rounded to float32', no_r_rounding, np.s_[:, :3, :3]),
                             ('float64 translation increment', f64_increment, np.s_[:, :3, 3])):
        d = np.abs(mutant[sl] - exact[sl])
        print('%s: %.2f %% of the elements change, max %.2e' % (what, 100 * (d > 0).mean(), d.max()))
        assert (d > 0).mean() >= 0.9 and d.max() < 1e-7, what
        others = np.ones(exact.shape, bool); others[sl] = False
        assert np.array_equal(mutant[others], exact[others]), what


@pytest.mark.parametrize('tn,rn', NORMALIZERS)
def test_exemptions_are_rare_and_real(tn, rn):
    _, _, ro = pose_update_cases()
    ex = exempt_rows(ro, rn)
    assert ex.mean() <= 1e-3
    f = np.float32(1.25)
    mid = (np.float64(f) + np.float64(np.nextafter(f, np.float32(2)))) / 2
    probe = np.array([mid, np.nextafter(mid, 0), mid + 8 * np.spacing(mid), mid + 9 * np.spacing(mid), np.float64(f), 0.0])
    assert near_f32_midpoint(probe).tolist() == [True, True, True, False, False, False]


def test_near_pi_cases_straddle_the_small_sine_branch():
    ws, deltas = near_pi_cases()
    for w, d in zip(ws, deltas):
        R = cv2.Rodrigues(w)[0]
        s = np.linalg.norm([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]]) / 2
        assert (s < 1e-5) == (d < 1e-5), (w, d, s)
    assert set(deltas[deltas < 1e-5]) and set(deltas[deltas > 1e-5])
