"""Re-initialisation of lost tracks without a GPU: se3tn_reinit_opts in include/se3tn.h against _lib, the entry points'
bindings, Engine.reinit_spec's and the Tracker's option parsing, and oracle/reinit_ref.py's loss, accept and event rules at
their edges."""
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
import reinit_ref as R  # noqa: E402

L = importlib.import_module(PKG + '._lib')
E = importlib.import_module(PKG + '.engine').Engine
P = importlib.import_module(PKG + '.predict')


def _header():
    return open(os.path.join(ROOT, 'include', 'se3tn.h')).read()


def test_reinit_opts_match_the_header():
    m = re.search(r'struct\s+se3tn_reinit_opts\s*\{([^}]*)\}', re.sub(r'/\*.*?\*/', '', _header(), flags=re.S))
    assert ' '.join(m.group(1).split()) == 'int32_t below_permille, after; int32_t reserved[2];'
    assert L.ReinitOpts._fields_ == [('below_permille', C.c_int32), ('after', C.c_int32), ('reserved', C.c_int32 * 2)]
    assert C.sizeof(L.ReinitOpts) == 16
    for name, v in (('NONE', 0), ('BELOW', 1), ('RESTARTED', 2), ('NO_START', 3), ('REJECTED', 4)):
        assert re.search(r'#define SE3TN_REINIT_%s %d\b' % (name, v), _header())
        assert getattr(L, 'REINIT_' + name) == getattr(R, name) == v
    # the existing structs keep their sizes
    assert C.sizeof(L.TrackOpts) == 48 and C.sizeof(L.TrackArrays) == 7 * C.sizeof(C.c_void_p)


def test_bindings():
    sig = L.SIGNATURES
    assert len(sig['se3tn_lost_tracks'][1]) == 8
    assert len(sig['se3tn_fit_poses'][1]) == 16
    assert len(sig['se3tn_accept_starts'][1]) == 13


def test_reinit_spec():
    assert (E.reinit_spec().below_permille, E.reinit_spec().after) == (500, 3)
    assert E.reinit_spec(0.001, 1000).below_permille == 1 and E.reinit_spec(1, 1).below_permille == 1000
    assert E.reinit_spec(0.123, 2).below_permille == 123 and E.reinit_spec(np.float32(0.25), 2).below_permille == 250
    for below in (0, -0.5, 1.001, 0.1234, 0.0005, float('nan'), float('inf'), True, '0.5', None):
        with pytest.raises(ValueError, match='below'):
            E.reinit_spec(below, 3)
    for after in (0, 1001, 2.0, True, None):
        with pytest.raises(ValueError, match='after'):
            E.reinit_spec(0.5, after)


def test_reinit_options():
    assert P.reinit_options(None) is None
    assert P.reinit_options({}) == {'below': 0.5, 'after': 3, 'init': None}
    spec = P.reinit_options({'below': 0.3, 'after': 2, 'init': {'keep': 4}})
    assert spec == {'below': 0.3, 'after': 2, 'init': {'keep': 4}}
    for bad, msg in (([0.5], 'dict'), ({'below': 0.5, 'tau': 3}, 'unknown'), ({'below': 2}, 'below'), ({'after': 0}, 'after'),
                     ({'init': {'keep': 0}}, 'keep'), ({'init': {'views': 3}}, 'unknown')):
        with pytest.raises(ValueError, match=msg):
            P.reinit_options(bad)


def _rows(model, inlier, residual=0):
    return np.array([[model, inlier, inlier, 0, 0, residual]], np.int32)


def test_below_at_its_edges():
    assert not R.below(_rows(1000, 500), 500)[0]            # 1000 inlier == permille model: not below
    assert R.below(_rows(1000, 499), 500)[0]
    assert R.below(_rows(0, 0), 1)[0]                       # model = 0 is below at any threshold
    assert not R.below(_rows(7, 7), 1000)[0] and R.below(_rows(7, 6), 1000)[0]
    big = np.array([[2**31 - 1, 2**30, 2**30, 0, 0, 0]], np.int32)   # the products need int64
    assert R.below(big, 1000)[0] and not R.below(big, 500)[0]


def test_streak_lost_and_reset():
    rows = np.concatenate([_rows(100, 10), _rows(100, 90), _rows(0, 0)])
    streak = np.zeros(3, np.int32)
    for step in range(1, 4):
        streak, event, lost = R.lost_tracks(rows, streak, 500, 3)
        assert list(event) == [1, 0, 1] and list(streak) == [step, 0, step]
        assert list(lost) == ([0, 2] if step == 3 else [])
    # an attempt resets the streak whatever its outcome: a track is retried at most once every `after` frames
    starts, dummy = np.zeros((2, 16)), np.zeros((3, 16))
    init_rows = np.array([[0] + [0] * 7, [1] + [0] * 7], np.int32)
    start_fit = np.concatenate([_rows(100, 5), _rows(100, 100)])
    _, _, streak, event = R.accept_starts([0, 2], starts, init_rows, start_fit, dummy, rows, streak, event)
    assert list(streak) == [0, 0, 0] and list(event) == [R.REJECTED, 0, R.NO_START]
    for step in (1, 2):
        streak, event, lost = R.lost_tracks(rows, streak, 500, 3)
        assert list(streak) == [step, 0, step] and len(lost) == 0


def test_accept_rule():
    tracked = np.concatenate([_rows(100, 50, 500), _rows(100, 50, 500), _rows(100, 50, 500), _rows(100, 50, 500), _rows(9, 9)])
    poses = np.arange(5 * 16, dtype=np.float64).reshape(5, 16)
    starts = -np.arange(4 * 16, dtype=np.float64).reshape(4, 16) - 1
    start_fit = np.concatenate([_rows(100, 50, 500),            # ties the tracked row: rejected
                                _rows(200, 100, 1001),          # the same fraction, a higher mean residual: rejected
                                _rows(200, 100, 998),           # the same fraction, a lower mean residual: restarted
                                _rows(100, 51, 10**6)])         # a higher fraction, whatever the residual: restarted
    init_rows = np.zeros((4, 8), np.int32)
    streak, event = np.full(5, 3, np.int32), np.ones(5, np.int32)
    out_p, out_r, out_s, out_e = R.accept_starts([0, 1, 2, 3], starts, init_rows, start_fit, poses, tracked, streak, event)
    assert list(out_e) == [R.REJECTED, R.REJECTED, R.RESTARTED, R.RESTARTED, 1]
    assert np.array_equal(out_p[[0, 1, 4]], poses[[0, 1, 4]]) and np.array_equal(out_p[2:4], starts[2:4])
    assert np.array_equal(out_r[2:4], start_fit[2:4]) and np.array_equal(out_r[[0, 1, 4]], tracked[[0, 1, 4]])
    assert list(out_s) == [0, 0, 0, 0, 3]                     # track 4 was not in the list: untouched
    row = lambda *a: _rows(*a)[0]
    assert not R.better(row(0, 0), row(0, 0)) and R.better(row(1, 0), row(0, 0))
    assert R.better(row(10, 1, 5), row(10, 0)) and not R.better(row(10, 0), row(10, 1, 5))
    init_rows[3, 0] = 2                                       # no start: nothing changes but the event and the streak
    out_p, out_r, out_s, out_e = R.accept_starts([3], starts[3:], init_rows[3:], start_fit[3:], poses, tracked, streak, event)
    assert out_e[3] == R.NO_START and out_s[3] == 0 and np.array_equal(out_p, poses) and np.array_equal(out_r, tracked)

