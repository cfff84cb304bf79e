"""Start poses from a mask without a GPU: se3tn_init_opts / se3tn_init_arrays in include/se3tn.h against _lib, the entry point's
binding, Engine.init_spec's parsing and refusals, oracle/init_ref.py's rotation grid, and its mask statistics and score /
delta / rank rules on hand-made frames and crops."""
import ctypes as C
import importlib
import os
import re
import sys
import numpy as np
import pytest

PKG = 'iros20-6d-pose-tracking_b200'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import init_ref  # noqa: E402

L = importlib.import_module(PKG + '._lib')


def _header():
    return re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', 'se3tn.h')).read(), flags=re.S)


def _fields(name):
    m = re.search(r'\bstruct\s+%s\s*\{([^}]*)\}' % name, _header())
    assert m, 'struct %s is not defined' % name
    out = []
    for decl in filter(None, (' '.join(d.split()) for d in m.group(1).split(';'))):
        typ, names = re.match(r'((?:const )?\w+\s*\*?)\s*(.*)', decl).groups()
        typ = typ.replace(' ', '')
        for f in names.split(','):
            if typ == 'constse3tn_icp_opts*':
                out.append((f.strip(), C.POINTER(L.IcpOpts)))
            elif typ.endswith('*'):
                out.append((f.strip(), L._vp))
            else:
                out.append((f.strip(), {'int32_t': C.c_int32}[typ]))
    return out


def test_init_structs_match_the_header():
    assert L.InitOpts._fields_ == _fields('se3tn_init_opts') and C.sizeof(L.InitOpts) == 32
    assert L.InitArrays._fields_ == _fields('se3tn_init_arrays') and C.sizeof(L.InitArrays) == 8 * C.sizeof(C.c_void_p)
    assert [f[0] for f in L.InitArrays._fields_] == list(importlib.import_module(PKG + '.engine').Engine.INIT_ARRAYS)
    src = open(os.path.join(ROOT, 'include', 'se3tn.h')).read()
    for name, value in (('SE3TN_INIT_COLS', L.INIT_COLS), ('SE3TN_INIT_STATS', L.INIT_STATS), ('SE3TN_MAX_INIT_KEEP', L.MAX_INIT_KEEP)):
        assert int(re.search(r'#define %s (\d+)' % name, src).group(1)) == value


def test_init_poses_is_declared_and_bound():
    m = re.search(r'\bint\s+se3tn_init_poses\s*\(([^)]*)\)\s*;', _header())
    assert m
    params = [' '.join(p.split()) for p in m.group(1).split(',')]
    assert params[-5:] == ['const se3tn_init_opts* opts', 'double* poses_out', 'int32_t* out_rows', 'const se3tn_init_arrays* arrays',
                           'void* stream']
    res, args = L.SIGNATURES['se3tn_init_poses']
    assert res is L._i and len(args) == len(params)
    for p, a in zip(params, args):
        assert (a is L._i) == (p.split()[0] == 'int' and '*' not in p), p


def test_init_spec_defaults_and_fields():
    E = importlib.import_module(PKG + '.engine').Engine
    o = E.init_spec()
    assert (o.viewpoints, o.inplane, o.keep, o.tau_mm, o.min_pixels, o.reserved) == (300, 24, 8, 20, 100, 0)
    assert o.icp and (o.icp.contents.iterations, o.icp.contents.tau_mm, o.icp.contents.min_inliers) == (5, 20, 100)
    o = E.init_spec(dict(viewpoints=12, inplane=4, keep=3, icp=None))
    assert (o.viewpoints, o.inplane, o.keep) == (12, 4, 3) and not o.icp
    assert not E.init_spec(dict(icp=0)).icp
    o = E.init_spec(dict(icp=dict(iterations=2, tau_mm=15)))
    assert (o.icp.contents.iterations, o.icp.contents.tau_mm) == (2, 15)


@pytest.mark.parametrize('bad', [dict(viewpoints=0), dict(viewpoints=4097), dict(inplane=0), dict(inplane=361), dict(keep=0),
                                 dict(keep=33), dict(tau_mm=0), dict(tau_mm=1001), dict(min_pixels=0), dict(min_pixels=176 * 176 + 1),
                                 dict(viewpoints=4096, inplane=17), dict(viewpoints=2, inplane=2, keep=5), dict(viewpoints=1.5),
                                 dict(keep=True), dict(icp=17), dict(icp=dict(iterations=1, bogus=1)), dict(bogus=1), 'all'])
def test_init_spec_refuses(bad):
    E = importlib.import_module(PKG + '.engine').Engine
    with pytest.raises(ValueError):
        E.init_spec(bad)


def test_grid_rotations_are_distinct_orthonormal_and_look_along_their_viewpoint():
    for V, R in ((12, 4), (300, 24), (1, 1), (7, 360)):
        G = init_ref.grid(V, R, np.array([0.01, -0.02, 0.8]))
        Rs = G[:, :3, :3]
        assert np.abs(np.einsum('nij,nkj->nik', Rs, Rs) - np.eye(3)).max() < 1e-14
        assert np.abs(np.linalg.det(Rs) - 1).max() < 1e-14
        assert len({tuple(np.round(r.ravel(), 9)) for r in Rs}) == V * R
        for c in range(0, V * R, max(1, V * R // 97)):
            d = init_ref.viewpoint(c // R, V)
            assert np.abs(Rs[c] @ d - [0, 0, -1]).max() < 1e-14
        assert np.all(G[:, :3, 3] == [0.01, -0.02, 0.8])


def test_mask_statistics_on_a_hand_made_frame():
    K = np.array([[500.0, 0, 10], [0, 400.0, 5], [0, 0, 1]])
    seg = np.zeros((6, 8), np.uint8)
    depth = np.zeros((6, 8), np.uint16)
    seg[1, 2] = seg[1, 3] = seg[4, 6] = seg[5, 0] = 7
    seg[0, 0] = 3
    depth[1, 2], depth[1, 3], depth[4, 6], depth[0, 0] = 900, 700, 800, 100     # (5, 0) has no depth
    stats, t0 = init_ref.mask_stats(depth, seg, 7, 3, K)
    # mask 4, depth 3, u 2+3+6+0, v 1+1+4+5, lower median of (700, 800, 900) = 800
    assert stats.tolist() == [0, 4, 3, 11, 11, 800]
    assert np.array_equal(t0, [0.8 * ((11 / 4 - 10) / 500.0), 0.8 * ((11 / 4 - 5) / 400.0), 0.8])
    depth[4, 6] = 0
    assert init_ref.mask_stats(depth, seg, 7, 3, K)[0].tolist() == [2, 4, 2, 11, 11, 700]     # lower median of two: the smaller
    assert init_ref.mask_stats(depth, seg, 9, 3, K)[0][0] == 1
    assert init_ref.mask_stats(depth, seg, 9, 3, K)[1].tolist() == [0.0, 0.0, 1.0]


def test_score_and_delta_on_hand_made_crops():
    Rd = np.zeros((4, 4), np.uint16); O = np.zeros((4, 4), np.uint16); M = np.zeros((4, 4), bool)
    Rd[0, :3] = 500; O[0, :3] = (510, 515, 600); M[0, :2] = True; M[1, 0] = True; O[1, 0] = 400
    # model 3, maskc 3, overlap 2, pairs 2, S = 10 + 15 = 25, delta = (50 + 2) // 4 = 13, inliers |O - 513| <= 3: both
    assert init_ref.score(Rd, O, M, 3) == [3, 3, 2, 2, 2, 13]
    assert init_ref.score(Rd, O, M, 3, fixed_delta=True) == [3, 3, 2, 2, 0, 0]
    O[0, :2] = (490, 489)                                                # S = -21: delta = (-42 + 2) // 4 = -10 (floor)
    assert init_ref.score(Rd, O, M, 1)[5] == -10
    O[0, :2] = (490, 491)                                                # S = -19: (-38 + 2) // 4 = -9
    assert init_ref.score(Rd, O, M, 1)[5] == -9
    assert init_ref.score(np.zeros((4, 4), np.uint16), O, M, 1) == [0, 3, 0, 0, 0, 0]


def test_rank_rules():
    row = lambda cand, model, maskc, overlap, inlier: np.array([0, cand, model, maskc, overlap, 0, inlier, 0])
    a = row(5, 10, 10, 10, 5)          # 5 / 10
    b = row(3, 20, 20, 10, 9)          # 9 / 30
    assert init_ref.ranks_above(a, b) and not init_ref.ranks_above(b, a)
    c = row(9, 10, 10, 8, 5)           # 5 / 12
    d = row(2, 12, 12, 12, 6)          # 6 / 12
    assert init_ref.ranks_above(d, c)
    e = row(4, 10, 10, 10, 5)          # equal to a, lower candidate
    assert init_ref.ranks_above(e, a)
    f = row(8, 20, 20, 20, 10)         # 10 / 20 = a's score, higher overlap
    assert init_ref.ranks_above(f, a) and init_ref.ranks_above(f, e)
    z = row(0, 0, 0, 0, 0)             # union 0 scores 0
    assert init_ref.ranks_above(a, z) and init_ref.rank_order([z, a, e, f]) == [3, 2, 1, 0]


def test_shift_moves_along_the_ray():
    P = np.eye(4); P[:3, 3] = (0.1, -0.05, 0.8)
    Q = init_ref.shift(P, 40)
    assert np.allclose(Q[:3, 3], P[:3, 3] * (0.84 / 0.8), rtol=0, atol=1e-15) and np.array_equal(Q[:3, :3], P[:3, :3])
