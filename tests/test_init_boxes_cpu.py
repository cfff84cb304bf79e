"""CPU-only: se3tn_init_boxes' binding, oracle/init_box_ref.py's box statistics and depth candidates on hand-made frames, the
candidate numbering, and the argument checks of Engine.box_spec / Engine.box_pixels."""
import ctypes as C
import fractions
import importlib
import os
import re
import sys
import numpy as np
import pytest

PKG = 'iros20-6d-pose-tracking_b200'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import init_box_ref as ibr  # noqa: E402
import init_ref  # noqa: E402

L = importlib.import_module(PKG + '._lib')
Engine = importlib.import_module(PKG + '.engine').Engine
K = np.array([[600.0, 0, 320.0], [0, 610.0, 240.0], [0, 0, 1]])


def test_binding_mirrors_the_header():
    src = open(os.path.join(ROOT, 'include', 'se3tn.h')).read()
    decl = re.search(r'int se3tn_init_boxes\((.*?)\);', src, re.S).group(1)
    args = [a.strip() for a in re.sub(r'/\*.*?\*/', '', decl).split(',')]
    kinds = [C.c_int if re.match(r'(const )?int\b', a) and '*' not in a else C.c_void_p for a in args]
    res, argtypes = L.SIGNATURES['se3tn_init_boxes']
    assert res is C.c_int and argtypes == kinds and len(args) == 19
    assert [a.split()[-1].lstrip('*') for a in args][5:7] == ['boxes', 'depths']
    lib = L.load()
    assert hasattr(lib, 'se3tn_init_boxes')


def test_quantile_index_against_sorted_depths():
    rng = np.random.default_rng(0)
    for P in list(range(1, 40)) + [100, 101, 4096, 4097]:
        for D in range(1, 9):
            d = np.sort(rng.integers(1, 65536, P))
            for q in range(D):
                k = ibr.quantile_index(q, D, P)
                exact = fractions.Fraction((2 * q + 1) * P - D, 2 * D)       # floor of the quantile (2q+1)/2D's position
                assert k == max(0, exact.numerator // exact.denominator) and 0 <= k < P
                assert d[k] == np.sort(d)[k]
            ks = [ibr.quantile_index(q, D, P) for q in range(D)]
            assert ks == sorted(ks)
            if D == 1:
                assert ks == [(P - 1) // 2]                               # the lower median, the mask rule's z_med


def _frame(H=12, W=16, seed=0):
    rng = np.random.default_rng(seed)
    return rng.integers(300, 2000, (H, W)).astype(np.uint16)


def test_box_statistics_on_hand_made_frames():
    depth = _frame()
    depth[3, 5] = 0; depth[4, 6] = 0
    box = (4, 2, 9, 6)                                   # u 4..8, v 2..5: 20 pixels, two without depth
    stats, t0 = ibr.box_stats(depth, box, 1, K, 3)
    d = np.sort(depth[2:6, 4:9].reshape(-1).astype(np.int64))
    d = d[d > 0]
    assert list(stats) == [0, 20, 18, sum(range(4, 9)) * 4, sum(range(2, 6)) * 5, d[(18 - 1) // 2]]
    assert 2 * stats[3] == (4 + 9 - 1) * stats[1]        # sum_u / mask is (x0 + x1 - 1) / 2 exactly
    for q in range(3):
        z = d[ibr.quantile_index(q, 3, 18)] / 1000.0
        u, v = stats[3] / 20.0, stats[4] / 20.0
        assert np.array_equal(t0[q], [z * ((u - K[0, 2]) / K[0, 0]), z * ((v - K[1, 2]) / K[1, 1]), z])
    # half-open: column x1 and row y1 are outside; a value placed there changes nothing
    d2 = depth.copy()
    d2[:, 9] = 1; d2[6, :] = 1
    assert np.array_equal(ibr.box_stats(d2, box, 1, K, 3)[0], stats)
    d2[2, 4] = 0                                         # (x0, y0) is inside
    assert not np.array_equal(ibr.box_stats(d2, box, 1, K, 3)[0], stats)


@pytest.mark.parametrize('P', [7, 8])
def test_even_and_odd_depth_counts(P):
    depth = np.zeros((4, 10), np.uint16)
    depth[1, :P] = np.arange(P, 0, -1) * 100 + 50
    stats, t0 = ibr.box_stats(depth, (0, 0, 10, 4), 1, K, 2)
    assert stats[2] == P and stats[5] == np.sort(depth[1, :P])[(P - 1) // 2]
    srt = np.sort(depth[1, :P])
    assert [round(z * 1000) for z in t0[:, 2]] == [srt[max(0, (P - 2) // 4)], srt[max(0, (3 * P - 2) // 4)]]


def test_fewer_depths_than_candidates_clamp_to_the_first():
    depth = np.zeros((5, 5), np.uint16)
    depth[2, 2], depth[3, 3] = 900, 700
    stats, t0 = ibr.box_stats(depth, (0, 0, 5, 5), 1, K, 8)
    assert stats[2] == 2
    ks = [ibr.quantile_index(q, 8, 2) for q in range(8)]
    assert ks == [0] * 6 + [1] * 2                       # floor((2 d + 1) / 8 - 1 / 2), at least 0
    assert list(np.round(t0[:, 2] * 1000)) == [700] * 6 + [900] * 2


def test_empty_boxes_and_too_few_depths():
    depth = _frame()
    for box in [(3, 3, 3, 9), (2, 5, 9, 5), (0, 0, 0, 0)]:
        stats, t0 = ibr.box_stats(depth, box, 1, K, 4)
        assert stats[0] == 1 and stats[1] == 0 and np.array_equal(t0, np.tile([0.0, 0.0, 1.0], (4, 1)))
    stats, t0 = ibr.box_stats(depth, (0, 0, 3, 3), 10, K, 2)
    assert stats[0] == 2 and stats[2] == 9 and np.array_equal(t0, np.tile([0.0, 0.0, 1.0], (2, 1)))


def test_a_box_on_the_frame_border():
    depth = _frame()
    H, W = depth.shape
    stats, _ = ibr.box_stats(depth, (W - 3, 0, W, H), 1, K, 1)
    assert stats[1] == 3 * H and stats[3] == sum(range(W - 3, W)) * H and stats[4] == sum(range(H)) * 3
    # box membership under a crop window that hangs over the right border: M marks exactly the crop pixels whose source
    # pixel lies in the box
    big = np.full((480, 640), 800, np.uint16)
    pose = np.eye(4)
    pose[:3, 3] = (0.2625, 0.0, 0.5)                     # projects to u = 635
    box = (600, 200, 640, 300)
    O, M = ibr.crop(pose, K, 200.0, big, box)
    top, left, ch, cw = init_ref.so.crop_window(init_ref.so.compute_bbox(pose, K, 200.0, scale=(1000, 1000, 1000)))
    fy, fx = init_ref.icp_ref.window_indices(top, left, ch, cw, 176)
    assert left + cw > 640 and (fx >= 640).any()
    want = ((fy >= 200) & (fy < 300))[:, None] & ((fx >= 600) & (fx < 640))[None, :]
    assert M.any() and np.array_equal(M, want) and (O[:, fx >= 640] == 0).all()


def test_candidate_numbering_and_grid():
    V, R, D = 5, 3, 2
    t0 = np.array([[0.1, 0.0, 0.8], [0.12, 0.0, 0.96]])
    G = ibr.grid(V, R, t0)
    assert G.shape == (D * V * R, 4, 4)
    for d in range(D):
        for v in range(V):
            for r in range(R):
                c = ibr.candidate(d, v, r, V, R)
                assert c == d * V * R + v * R + r
                assert np.array_equal(G[c][:3, :3], init_ref.grid_rotation(v * R + r, V, R))
                assert np.array_equal(G[c][:3, 3], t0[d])
    assert np.array_equal(ibr.grid(V, R, t0[:1]), init_ref.grid(V, R, t0[0]))


def test_tight_box_and_background():
    seg = np.zeros((10, 12), np.uint8)
    seg[2:5, 3:8] = 4
    seg[9, 11] = 4
    assert list(ibr.tight_box(seg, 4)) == [3, 2, 12, 10]
    assert list(ibr.tight_box(seg, 5)) == [0, 0, 0, 0]
    depth = np.zeros((480, 640), np.uint16)
    depth[100:200, 100:200] = 600
    bg = ibr.with_background(depth, K)
    assert (bg[100:200, 100:200] == 600).all() and bg[depth == 0].min() >= 1090 and bg.max() <= 1310


def test_box_arguments():
    b, D = Engine.box_spec([[1, 2, 3, 4]], 4)
    assert b.dtype == np.int32 and b.shape == (1, 4) and D == 4
    assert Engine.box_spec(np.zeros((0, 4), np.int64))[0].shape == (0, 4)
    for depths in (0, 9, 2.0, True, None):
        with pytest.raises(ValueError, match='depths'):
            Engine.box_spec([[1, 2, 3, 4]], depths)
    for boxes in ([[1.5, 2, 3, 4]], [[True, False, True, True]], [[1, 2, 3]], [1, 2, 3, 4, 5, 6, 7, 8, 9], [[0, 0, 2 ** 31, 4]]):
        with pytest.raises(ValueError):
            Engine.box_spec(boxes)
    assert list(Engine.box_pixels((10.2, 5.9, 20.1, 30.0), 480, 640)) == [10, 5, 21, 30]
    assert list(Engine.box_pixels((-5.5, -1, 700, 500.5), 480, 640)) == [0, 0, 640, 480]
    assert list(Engine.box_pixels((650, 490, 700, 500), 480, 640)) == [640, 480, 640, 480]     # wholly outside: empty
    assert list(Engine.box_pixels((30, 10, 20, 5), 480, 640)) == [30, 10, 30, 10]              # reversed: empty
    for box in ((0, 0, float('nan'), 3), (0, 0, 1), (0, 0, float('inf'), 3)):
        with pytest.raises(ValueError, match='four finite'):
            Engine.box_pixels(box, 480, 640)
