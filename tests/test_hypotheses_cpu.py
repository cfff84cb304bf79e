"""CPU: the hypothesis oracle (oracle/hypotheses_ref.py) -- its Philox stream, the distribution of its draws, the composition of
the starts and the selection rule -- and the C ABI of multi-hypothesis tracking in include/se3tn.h against _lib."""
import ctypes as C, importlib, math, os, re

import numpy as np
import pytest
from scipy.stats import truncnorm

import augment_ref as A
import hypotheses_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = 'iros20-6d-pose-tracking_b200'
CTYPES = {'int32_t': C.c_int32, 'int64_t': C.c_int64, 'double': C.c_double}


def test_philox_stream_is_augment_refs():
    for seed, key, h, slot in ((0, 0, 0, 0), (7, 123456789012, 3, 66), (2 ** 64 - 1, -5, 31, 129), (42, 2 ** 40 + 3, 1, 2)):
        k = key & (2 ** 64 - 1)
        assert R.words(seed, key, h, slot) == A.philox((k & A.MASK32, k >> 32, h, slot), (seed & A.MASK32, seed >> 32))
    # hypothesis index 0 is augment_ref's scalar stream: the same uniform from the same words
    for pair, slot in ((0, 0), (99, 5), (2 ** 33 + 1, 17)):
        w = R.words(11, pair, 0, slot)
        assert R.u53(w[0], w[1]) == A.philox_uniform(11, pair, slot)


def test_draws_follow_the_references_distribution():
    N, max_t, max_r = 100000, 0.02, 15.0
    mt = np.empty(N)
    dirs = np.empty((N, 3))
    for k in range(N):
        mt[k], tries = R.magnitude(5, k, 1, R.SLOT_MAG_T, max_t)
        assert 1 <= tries <= R.MAX_TRIES
        w = R.words(5, k, 1, R.SLOT_DIR_T)
        dirs[k] = R.direction(R.u53(w[0], w[1]), R.u53(w[2], w[3]))
    assert np.all(np.abs(mt) <= max_t)
    ref = truncnorm(-1.0, 1.0, loc=0.0, scale=max_t)
    sd = math.sqrt(ref.var() / N)
    assert abs(mt.mean() - ref.mean()) < 5 * sd
    assert abs(mt.var() / ref.var() - 1.0) < 0.02
    np.testing.assert_allclose(np.linalg.norm(dirs, axis=1), 1.0, atol=1e-12)
    assert np.all(np.abs(dirs.mean(axis=0)) < 5 / math.sqrt(3 * N))
    mr = np.array([R.magnitude(5, k, 2, R.SLOT_MAG_R, max_r)[0] for k in range(2000)])
    assert np.all(np.abs(mr) <= max_r) and mr.std() > 0.3 * max_r


def test_starts_compose_p_with_the_inverse_perturbation():
    rng = np.random.default_rng(3)
    P = np.tile(np.eye(4), (3, 1, 1))
    P[:, :3, 3] = rng.uniform(-0.2, 0.2, (3, 3)) + [0, 0, 0.8]
    P[1, :3, :3] = R.cv2.Rodrigues(np.array([0.3, -0.2, 0.5]))[0]
    keys = np.array([0, 2 ** 35 + 1, -7], dtype=np.int64)
    starts, dr = R.expand(P, keys, 5, seed=9, max_t=0.03, max_r=20.0)
    assert np.array_equal(starts[:, 0], P) and not dr[:, 0].any()
    for i in range(3):
        for h in range(1, 5):
            D = R.delta(dr[i, h])
            np.testing.assert_allclose(starts[i, h].dot(D), P[i], atol=1e-14)
            assert np.linalg.norm(D[:3, 3]) <= 0.03 + 1e-15
            ang = math.degrees(math.acos(np.clip((np.trace(D[:3, :3]) - 1) / 2, -1, 1)))
            assert ang <= 20.0 + 1e-9 and abs(ang - abs(dr[i, h, 5])) < 1e-9
            assert tuple(dr[i, h]) == R.draws(9, int(keys[i]), h, 0.03, 20.0)


def _row(model, inlier, residual, observed=None):
    return [model, inlier if observed is None else observed, inlier, 0, 0, residual]


def test_selection_rule():
    rows = np.array([
        [_row(100, 50, 500), _row(100, 50, 500), _row(200, 100, 1000)],   # equal fractions and mean residuals: the lowest h
        [_row(100, 50, 500), _row(100, 60, 900), _row(100, 60, 600)],     # the higher fraction, then the lower mean residual
        [_row(0, 0, 0), _row(100, 0, 0), _row(0, 0, 0)],                  # model = 0 ranks last
        [_row(100, 0, 0), _row(50, 0, 0), _row(10, 10, 90)],              # inlier = 0 ranks below any inlier
        [_row(100, 0, 0, 0), _row(120, 0, 0, 0), _row(80, 0, 0, 0)],      # no depth anywhere: hypothesis 0
        [_row(100, 40, 400), _row(30976, 30976, 30976000 - 1), _row(30976, 30976, 30976000)],
    ], dtype=np.int32)
    assert R.choose(rows).tolist() == [0, 2, 1, 2, 0, 1]
    # counts of a full 176 x 176 window: the cross products need 64 bits, and a near tie must still resolve
    a, b = _row(30976, 30975, 30975 * 1000), _row(30975, 30974, 30974 * 1000 - 1)
    assert R.better(b, a) == (30974 * 30976 > 30975 * 30975)
    assert 30975 * 1000 * 30976 > 2 ** 31


def _header():
    return re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', 'se3tn.h')).read(), flags=re.S)


def test_hypothesis_opts_match_the_header():
    m = re.search(r'\bstruct\s+se3tn_hypothesis_opts\s*\{([^}]*)\}', _header())
    assert m, 'struct se3tn_hypothesis_opts is not defined'
    fields = []
    for decl in filter(None, (d.strip() for d in m.group(1).split(';'))):
        typ, names = decl.split(None, 1)
        fields += [(name.strip(), CTYPES[typ]) for name in names.split(',')]
    L = importlib.import_module(PKG + '._lib')
    assert L.HypothesisOpts._fields_ == fields and C.sizeof(L.HypothesisOpts) == 32
    assert int(re.search(r'SE3TN_MAX_HYPOTHESES\s+(\d+)', _header()).group(1)) == L.MAX_HYPOTHESES == 32
    assert int(re.search(r'SE3TN_HYP_DRAWS\s+(\d+)', _header()).group(1)) == L.HYP_DRAWS == 8


def test_hypothesis_calls_match_the_header():
    src = _header()
    L = importlib.import_module(PKG + '._lib')
    params = [' '.join(p.split()) for p in re.search(r'\bint\s+se3tn_draw_hypotheses\s*\(([^)]*)\)\s*;', src).group(1).split(',')]
    assert params[-4:] == ['const se3tn_hypothesis_opts* hyp', 'double* out_poses', 'double* out_draws', 'void* stream']
    res, args = L.SIGNATURES['se3tn_draw_hypotheses']
    assert res is L._i and len(args) == len(params)


def test_hypothesis_spec_refusals():
    E = importlib.import_module(PKG + '.engine').Engine
    ok = E.hypothesis_spec(4, 2 ** 64 - 1, 0.02, 15)
    assert (ok.hypotheses, ok.seed, ok.max_translation, ok.max_rotation_deg) == (4, -1, 0.02, 15.0)
    for bad in ((0, 0, 0.02, 15), (33, 0, 0.02, 15), (True, 0, 0.02, 15), (2.0, 0, 0.02, 15), (4, 0.5, 0.02, 15),
                (4, 0, 0.0, 15), (4, 0, 1.5, 15), (4, 0, float('nan'), 15), (4, 0, float('inf'), 15),
                (4, 0, 0.02, 0), (4, 0, 0.02, 181), (4, 0, 0.02, float('nan'))):
        with pytest.raises(ValueError):
            E.hypothesis_spec(*bad)


def _pr():
    return importlib.import_module(PKG + '.predict')


BASE = ['--train_data_path', 'x', '--model_path', 'x', '--ckpt_dir', 'x', '--mean_std_path', 'x', '--outdir', 'x']


@pytest.mark.parametrize('mode', ['ycbv', 'ycbineoat', 'ycbv_per_class'])
def test_cli_refuses_hypotheses_in_single_sequence_modes(mode):
    with pytest.raises(SystemExit, match='--hypotheses 4 needs'):
        _pr().main(['--mode', mode] + BASE + ['--hypotheses', '4'])


@pytest.mark.parametrize('S', ['0', '33'])
def test_cli_refuses_hypotheses_out_of_range(S):
    with pytest.raises(SystemExit, match='--hypotheses %s' % S):
        _pr().main(['--mode', 'ycbineoat_all', '--YCBInEOAT_dir', 'x'] + BASE + ['--hypotheses', S])


def test_cli_passes_hypotheses_and_seed(monkeypatch, tmp_path):
    pr, got = _pr(), {}
    monkeypatch.setattr(pr, 'getResultsYcbInEOAT', lambda d, config, outdir, **kw: got.update(kw) or {})
    base = ['--mode', 'ycbineoat_all', '--YCBInEOAT_dir', 'x'] + BASE[:-1] + [str(tmp_path)]
    pr.main(base + ['--hypotheses', '4', '--seed', '9'])
    assert got['hypotheses'] == 4 and got['seed'] == 9
    got.clear()
    pr.main(base)
    assert 'hypotheses' not in got and 'seed' not in got             # a run without the flag makes the same call as before
    rec = {}
    monkeypatch.setattr(pr, 'recoverYcbKeyframes', lambda *a, **kw: rec.update(kw) or (_ for _ in ()).throw(SystemExit('stop')))
    monkeypatch.setattr(pr, 'ycb_class_names', lambda d: ['a', 'b'])
    monkeypatch.setattr(pr, 'recover_front', lambda *a, **kw: None)
    monkeypatch.setattr(pr, 'checkpoint_configs', lambda c: [c])
    monkeypatch.setattr(pr, 'pair_mesh_base', lambda *a: 100)
    with pytest.raises(SystemExit, match='stop'):
        pr.main(['--mode', 'ycbv_recover', '--ycb_dir', 'y', '--class_ids', '1'] + BASE + ['--hypotheses', '4', '--seed', '5'])
    assert rec['hypotheses'] == 4 and rec['seed'] == 5


def test_driver_hypothesis_keys_and_groups():
    pr = _pr()
    assert pr.hypothesis_key(1, 2, 3) == (1 << 40) + (2 << 16) + 3
    for bad in ((1 << 23, 0, 0), (0, 1 << 24, 0), (0, 0, 1 << 16), (-1, 0, 0)):
        with pytest.raises(ValueError):
            pr.hypothesis_key(*bad)
    T = lambda t, r: type('T', (), {'dataset_info': {'max_translation': t, 'max_rotation': r}})()
    trk = {1: T(0.02, 15), 2: T(0.02, 15), 3: T(0.03, 5)}
    opts = pr.step_options(hypotheses=4, seed=3)
    assert (opts.hypotheses, opts.seed) == (4, 3)
    assert pr.hypothesis_groups(trk, [1, 2], opts) == [(None, (0.02, 15.0))]
    g = pr.hypothesis_groups(trk, [1, 3, 2], opts)
    assert [x[1] for x in g] == [(0.02, 15.0), (0.03, 5.0)] and g[0][0].tolist() == [0, 2] and g[1][0].tolist() == [1]
    assert pr.hypothesis_spread({}, pr.step_options(seed=3)) is None          # S = 1 reads no spread
    assert pr.hypothesis_spread({'max_translation': 0.02, 'max_rotation': 15}, opts, 'class 1') == (0.02, 15.0)
    for info in ({}, {'max_translation': 0.02}, {'max_translation': 1.5, 'max_rotation': 15}, {'max_translation': 0.02, 'max_rotation': 0}):
        with pytest.raises(ValueError, match='class 2: dataset_info max_translation / max_rotation'):
            pr.hypothesis_spread(info, opts, 'class 2')
    for bad in (dict(hypotheses=33), dict(hypotheses=0), dict(hypotheses=True), dict(hypotheses=2.0), dict(seed=0.5), dict(seed=True)):
        with pytest.raises(ValueError, match='hypotheses|seed'):
            pr.step_options(**bad)
