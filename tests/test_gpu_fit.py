"""The fit check of a tracking step (se3tn_track_opts.fit_tau_mm, Engine.track_render(fit=), Tracker(fit=), the drivers' fit=): every row
equals oracle/fit_ref.py on the model rendered at the step's new poses and the observed depth crop_bbox cuts at their windows, in
every precision, render mode, batch shape, round count and route; the step's other outputs keep their bits; the graph key,
launch count and refusals follow include/se3tn.h; and the rows mean what their names say on hand-made frames."""
import ctypes as C
import importlib
import os
import sys
import numpy as np
import pytest
import torch
from test_gpu_precision_sweep import eoat, ycbv, pr      # the synthetic layouts of the driver tests  # noqa: F401
from test_gpu_refine import _raw_track_batch, _raw_track_host, _raw_track_render, _tracker

pytestmark = pytest.mark.gpu
PKG = 'iros20-6d-pose-tracking_b200'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import fit_ref  # noqa: E402

TN, RN = 0.03, 5 * np.pi / 180
HW = (480, 640)
SETS = (0, 5)                                   # two weight sets under sparse ids
ZERO = 9                                        # a weight set whose head outputs 0: the pose update is the identity
K = importlib.import_module(PKG + '.synth').CAMERA_K
TAU = 15


@pytest.fixture(scope='module')
def eng(pkg, synth):
    e = pkg.Engine(max_batch=64)
    mean, std = synth.default_mean_std()
    for j, wid in enumerate(SETS):
        e.load_state_dict(synth.make_state_dict(j), wid)
        e.set_mesh(synth.mesh(2 - j, seed=j), wid)
        e.set_stats(mean + 1.5 * j, std * (1 + 0.25 * j), wid)
    sd = synth.make_state_dict(2)
    for k in ('trans_out.0.weight', 'trans_out.0.bias', 'rot_out.0.weight', 'rot_out.0.bias'):
        sd[k] = torch.zeros_like(sd[k])
    e.load_state_dict(sd, ZERO)
    e.set_mesh(synth.mesh(2, seed=7), ZERO)
    e.set_stats(mean, std, ZERO)
    c = Case(e, synth, 6, seed=3)
    e.calibrate_fp8_tracks(c.R, c.D, K, c.P, c.ow, weight_ids=c.wid, render=dict(mode='vispy', image_hw=None, mesh_ids=c.wd))
    yield e
    e.close()


@pytest.fixture(scope='module', autouse=True)
def keep_utils_engine():
    U = importlib.import_module(PKG + '.Utils')
    saved = U._engine
    yield
    U.set_engine(saved)


def _dev(e, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(e.device)


class Case:
    def __init__(self, e, synth, n, seed):
        self.n = n
        self.rgb, self.depth = synth.raw_frame(seed)
        self.depth[100:140, 200:260] = 0                           # holes for the fill to close
        self.poses = synth.raw_poses(n, seed=seed)
        self.poses[0, :3, 3] = (0.3, -0.19, 0.5)                   # a window over the frame's edge
        self.R, self.D, self.P = _dev(e, self.rgb), _dev(e, self.depth), _dev(e, self.poses)
        self.ow = torch.full((n,), 200.0, dtype=torch.float64, device=e.device)
        self.wid = None if n == 1 else np.array([SETS[i % 2] for i in range(n)], dtype=np.int32)
        self.wd = None if self.wid is None else _dev(e, self.wid)


def _step(e, c, k, prec, mode, fill, fit=TAU, **kw):
    n = c.n
    outs = dict(out_poses=torch.empty_like(c.P), out_trans=torch.full((n, 3), float('nan'), device=e.device),
                out_rot=torch.full((n, 3), float('nan'), device=e.device))
    outs.update(kw)
    return e.track_render(c.R, c.D, K, c.P, c.ow, TN, RN, weight_ids_host=c.wid, weight_ids_dev=c.wd, precision=prec, mode=mode,
                          image_hw=HW if mode == 'pyrender' else None, fill_depth=fill, iterations=k, fit=fit, **outs)


def _oracle(e, poses, ow, wd, mode, depth, tau):
    """fit_ref on R = Engine.render at `poses` and O = Engine.crop_bbox of `depth` at compute_bbox(poses)."""
    _, R = e.render(K, poses, ow, wd, mode=mode, image_hw=HW if mode == 'pyrender' else None)
    rgb = torch.zeros(depth.shape + (3,), dtype=torch.uint8, device=e.device)
    _, O = e.crop_bbox(rgb, depth, e.compute_bbox(poses, K, ow))
    torch.cuda.synchronize()
    return fit_ref.fit_rows(R.cpu().numpy(), O.cpu().numpy(), tau)


@pytest.mark.parametrize('fill', [False, True], ids=['raw', 'fill'])
@pytest.mark.parametrize('mode', ['vispy', 'pyrender'])
@pytest.mark.parametrize('prec', ['bf16x3', 'fp8', 'fp32'])
def test_rows_equal_the_oracle(synth, eng, prec, mode, fill):
    for n in (1, 3, 64):
        c = Case(eng, synth, n, seed=n + 7)
        depth = eng.fill_depth(c.D) if fill else c.D
        for k in (1, 3):
            P, tr, ro, rows = _step(eng, c, k, prec, mode, fill)
            want = _oracle(eng, P, c.ow, c.wd, mode, depth, TAU)
            got = rows.cpu().numpy()
            assert np.array_equal(got, want), (n, k)
            assert (got[:, 1] == got[:, 2] + got[:, 3] + got[:, 4]).all()
            assert got[:, 0].sum() > 0 or (n == 1 and mode == 'pyrender')   # track 0's window lies over the camera image's edge
            if n <= 3:                                              # the host route: same poses, same rows
                hp, htr, hro, hrows = eng.track_render_host(c.rgb, c.depth, K, c.poses, c.ow.cpu().numpy(), TN, RN, weight_ids=c.wid,
                                                            precision=prec, mode=mode, image_hw=HW if mode == 'pyrender' else None,
                                                            fill_depth=fill, iterations=k, want_residuals=True, fit=TAU)
                assert np.array_equal(hp, P.cpu().numpy()) and np.array_equal(hrows, got), (n, k)


@pytest.mark.parametrize('prec', ['bf16x3', 'fp8', 'fp32'])
def test_outputs_keep_their_bits(synth, eng, prec):
    for n in (1, 64):
        c = Case(eng, synth, n, seed=20 + n)
        for mode in ('vispy', 'pyrender'):
            for k in (1, 3):
                rounds = [torch.full((k, n, 4, 4), float('nan'), dtype=torch.float64, device=eng.device) for _ in range(2)]
                off = _step(eng, c, k, prec, mode, True, fit=None, out_rounds=rounds[0])
                on = _step(eng, c, k, prec, mode, True, out_rounds=rounds[1])
                assert all(torch.equal(a, b) for a, b in zip(off, on[:3])), (n, mode, k)
                assert torch.equal(rounds[0], rounds[1])


def test_graph_replay_launch_count_and_tau(synth, eng):
    c = Case(eng, synth, 5, seed=41)
    outs = dict(out_poses=torch.empty_like(c.P), out_trans=torch.empty(5, 3, device=eng.device), out_rot=torch.empty(5, 3, device=eng.device))
    _step(eng, c, 2, 'bf16x3', 'vispy', False, fit=None, **outs)
    plain = eng.last_launch_count()
    seen = {}
    for rep in range(3):
        for tau in (5, 50, None, 5):
            out = _step(eng, c, 2, 'bf16x3', 'vispy', False, fit=tau, **outs)
            assert eng.last_step_was_graph()
            assert eng.last_launch_count() == plain + (3 if tau else 0)
            if tau:
                got = out[3].cpu().numpy()
                assert np.array_equal(got, seen.setdefault(tau, got))      # a replay of tau's own graph
    assert np.array_equal(seen[5], _oracle(eng, out[0], c.ow, c.wd, 'vispy', c.D, 5))
    assert not np.array_equal(seen[5], seen[50])
    _step(eng, c, 2, 'fp32', 'vispy', False)
    assert not eng.last_step_was_graph() and eng.last_launch_count() > 3


def _zero_case(e, synth, poses):
    n = len(poses)
    P = _dev(e, poses)
    ow = torch.full((n,), 200.0, dtype=torch.float64, device=e.device)
    ids = np.full(n, ZERO, np.int32)
    return P, ow, ids, _dev(e, ids)


def _zero_step(e, frame_depth, P, ow, ids, wd):
    rgb = np.zeros(HW + (3,), np.uint8)
    return e.track_render_host(rgb, np.ascontiguousarray(frame_depth, dtype=np.uint16), K, P.cpu().numpy(), ow.cpu().numpy(), TN, RN,
                               weight_ids=ids, fit=TAU)


def test_meaning_with_a_zero_head(synth, eng):
    poses = synth.raw_poses(3, seed=60)
    poses[:, :3, 3] = [(0.02, -0.01, 0.55), (-0.03, 0.02, 0.6), (0.0, 0.0, 0.5)]
    P, ow, ids, wd = _zero_case(eng, synth, poses)
    out, rows = _zero_step(eng, np.zeros(HW), P, ow, ids, wd)
    assert np.array_equal(out, poses)                               # the identity update
    assert (rows[:, 0] > 1000).all() and (rows[:, 1] == 0).all()
    _, R = eng.render(K, P, ow, wd)
    R = R.cpu().numpy().astype(np.int64)
    near, far = 100, 60000
    assert R[R > 0].min() > near + TAU and R.max() + TAU < far
    _, rows = _zero_step(eng, np.full(HW, near), P, ow, ids, wd)
    assert (rows[:, 3] == rows[:, 0]).all() and (rows[:, 1] == rows[:, 0]).all()
    _, rows = _zero_step(eng, np.full(HW, far), P, ow, ids, wd)
    assert (rows[:, 4] == rows[:, 0]).all()
    gone = poses.copy(); gone[:, 0, 3] = 5.0                        # every window far right of the image
    G = _zero_case(eng, synth, gone)
    _, rows = _zero_step(eng, np.full(HW, 800), *G)
    assert (rows[:, 1] == 0).all()
    bb = eng.compute_bbox(P, K, ow).cpu().numpy()
    for i in range(3):                                              # R written where crop_bbox samples track i's window
        top, left = bb[i, :, 0].min(), bb[i, :, 1].min()
        ch, cw = bb[i, :, 0].max() - top, bb[i, :, 1].max() - left
        assert ch >= 176 and cw >= 176 and top >= 0 and left >= 0 and top + ch <= HW[0] and left + cw <= HW[1]
        sx = np.minimum(np.floor(np.arange(176) * (1.0 / (176.0 / cw))).astype(np.int64), cw - 1)
        sy = np.minimum(np.floor(np.arange(176) * (1.0 / (176.0 / ch))).astype(np.int64), ch - 1)
        frame = np.zeros(HW, np.uint16)
        frame[np.ix_(top + sy, left + sx)] = R[i]
        one = tuple(x[i:i + 1] for x in (P, ow)) + (ids[i:i + 1], wd[i:i + 1])
        _, rows = _zero_step(eng, frame, *one)
        assert rows[0, 2] == rows[0, 0] and rows[0, 5] == 0 and rows[0, 1] == rows[0, 0]


def _raw_track_render_host(e, c, out, opts, out_fit):
    Kh = np.ascontiguousarray([K[0, 0], K[1, 1], K[0, 2], K[1, 2]])
    h = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
    arrays = importlib.import_module(PKG + '._lib').TrackArrays(out_fit=None if out_fit is None else out_fit.ctypes.data)
    return e.lib.se3tn_track_render_host(e._ctx, h(c.rgb), h(c.depth), HW[0], HW[1], h(Kh), h(c.poses), h(np.full(c.n, 200.0)), 0, 0, 0,
                                         h(c.wid), c.n, TN, RN, 2, h(out[0]), h(out[1]), h(out[2]), C.byref(opts),
                                         C.byref(arrays), C.c_void_p(0))


def test_refusals(synth, eng):
    L = importlib.import_module(PKG + '._lib')
    c = Case(eng, synth, 4, seed=45)
    ra, da = eng.render(K, c.P, c.ow, c.wd)
    dev_out = lambda: (torch.full((4, 4, 4), float('nan'), dtype=torch.float64, device=eng.device),
                       torch.full((4, 3), float('nan'), device=eng.device), torch.full((4, 3), float('nan'), device=eng.device))
    host_out = lambda: (np.full((4, 4, 4), np.nan), np.full((4, 3), np.nan, np.float32), np.full((4, 3), np.nan, np.float32))
    refused = lambda rc, field: rc == L.ERR_INVALID and field in eng.lib.se3tn_last_error(eng._ctx)
    out = dev_out()
    assert _raw_track_batch(eng, c, ra, da, out, L.TrackOpts(iterations=1, fit_tau_mm=0)) == L.OK     # off: track_batch runs
    torch.cuda.synchronize()
    assert torch.isfinite(out[0]).all()
    launches = eng.last_launch_count()
    for bad in (1001, -5, 12):              # out of range for every call; on at all for the two calls that take input A
        opts = L.TrackOpts(iterations=1, fit_tau_mm=bad)
        out, hout, rout, rhout, rows = dev_out(), host_out(), dev_out(), host_out(), np.full((4, L.FIT_COLS), -1, np.int32)
        assert refused(_raw_track_batch(eng, c, ra, da, out, opts), b'fit_tau_mm'), bad
        assert refused(_raw_track_host(eng, c, ra.cpu().numpy(), da.cpu().numpy(), hout, opts), b'fit_tau_mm'), bad
        if bad != 12:
            assert refused(_raw_track_render(eng, c, c.P, rout, opts), b'fit_tau_mm'), bad
            assert refused(_raw_track_render_host(eng, c, rhout, opts, rows), b'fit_tau_mm'), bad
        torch.cuda.synchronize()
        assert all(torch.isnan(x).all() for x in out + rout) and all(np.isnan(x).all() for x in hout + rhout), bad
        assert (rows == -1).all(), bad
    # the host route's rows: out_fit is required while the check is on, and must be NULL while it is off
    hout, rows = host_out(), np.full((4, L.FIT_COLS), -1, np.int32)
    assert refused(_raw_track_render_host(eng, c, hout, L.TrackOpts(iterations=1, fit_tau_mm=12), None), b'out_fit')
    assert refused(_raw_track_render_host(eng, c, hout, L.TrackOpts(iterations=1, fit_tau_mm=0), rows), b'out_fit')
    assert all(np.isnan(x).all() for x in hout) and (rows == -1).all()
    assert eng.last_launch_count() == launches
    for bad in (0, 1001, 2.0, True, '10'):
        with pytest.raises(ValueError, match='fit'):
            eng.track_render(c.R, c.D, K, c.P, c.ow, TN, RN, fit=bad)
    with pytest.raises(ValueError, match='out_fit'):
        eng.track_render(c.R, c.D, K, c.P, c.ow, TN, RN, fit=10, out_fit=torch.empty(4, 5, dtype=torch.int32, device=eng.device))
    eng.track_render(c.R, c.D, K, c.P, c.ow, TN, RN, fit=10)          # leaves nothing on the context for the next track_batch
    eng.track_batch(c.R, c.D, K, c.P, c.ow, ra, da, TN, RN)


def test_tracker(pkg, synth, tmp_path):
    plain, fit = _tracker(pkg, synth, tmp_path), _tracker(pkg, synth, tmp_path, fit=True)
    pr_ = importlib.import_module(PKG + '.predict')
    try:
        assert fit.fit == pr_.FIT_TAU_DEFAULT and plain.fit is None
        rgb, depth = synth.raw_frame(50)
        poses = synth.raw_poses(3, seed=51)
        got = fit.on_track_batch(poses, rgb, depth)                                       # host route
        assert np.array_equal(got, plain.on_track_batch(poses, rgb, depth)) and plain.last_fit is None
        host_rows = fit.last_fit
        assert isinstance(host_rows, np.ndarray) and host_rows.shape == (3, 6) and host_rows.dtype == np.int32
        dev = fit.on_track_batch(torch.from_numpy(poses).cuda(), torch.from_numpy(rgb).cuda(), torch.from_numpy(depth).cuda())
        assert np.array_equal(dev.cpu().numpy(), got) and torch.is_tensor(fit.last_fit)
        assert np.array_equal(fit.last_fit.cpu().numpy(), host_rows)
        one = fit.on_track(poses[0], rgb, depth)
        assert one.shape == (4, 4) and fit.last_fit.shape == (1, 6) and fit.last_fit[0, 0] > 0
        f = pr_.fit_fractions(host_rows)
        assert np.allclose(f['inlier'], host_rows[:, 2] / host_rows[:, 0])
        rgbA, depthA = plain.render_window(poses[0])
        with pytest.raises(ValueError, match='input A was passed in'):
            fit.on_track(poses[0], rgb, depth, rgbA=rgbA, depthA=depthA)
        with pytest.raises(ValueError, match='input A was passed in'):
            fit.on_track_batch(poses[:1], rgb, depth, rgbA[None], depthA[None])
        with pytest.raises(ValueError, match='fit'):
            _tracker(pkg, synth, tmp_path, fit=0)
    finally:
        plain.engine.close(); fit.engine.close()


def _poses_tree(root):
    out = {}
    for d, _, fs in os.walk(root):
        for f in fs:
            if f != 'fit.npy':
                with open(os.path.join(d, f), 'rb') as x:
                    out[os.path.relpath(os.path.join(d, f), root)] = x.read()
    return out


def _fits(root):
    return {os.path.relpath(d, root): np.load(os.path.join(d, 'fit.npy')) for d, _, fs in os.walk(root) if 'fit.npy' in fs}


def _recording(pr):
    """Every Engine.track_render call with a fit check -> (its poses after the step, its fit rows), in call order."""
    E = pr.Engine
    orig = E.track_render
    got = []

    def rec(self, *a, **kw):
        res = orig(self, *a, **kw)
        if kw.get('fit'):
            got.append(res[3].cpu().numpy().copy())
        return res
    return E, orig, rec, got


def test_ycbineoat_fit(pr, eoat, capsys, monkeypatch):
    tmp, tpl = eoat
    data, ycb = str(tmp / 'data'), str(tmp / 'ycb')
    E, orig, rec, got = _recording(pr)
    monkeypatch.setattr(E, 'track_render', rec)
    run = lambda out, **kw: pr.getResultsYcbInEOAT(data, tpl, str(tmp / 'fit' / out), ycb_dir=ycb, max_frames=5, **kw)
    plain = run('plain')
    assert not got
    on = run('on', fit=TAU)
    assert all(np.array_equal(plain[v], on[v]) for v in plain)
    assert _poses_tree(str(tmp / 'fit' / 'plain')) == _poses_tree(str(tmp / 'fit' / 'on'))
    fits = _fits(str(tmp / 'fit' / 'on'))
    videos = sorted(pr.ycbineoat_videos(data))
    assert sorted(fits) == sorted(v for v, _ in videos)
    steps = iter(got)
    for v, _ in videos:                                             # videos in run order, one n = 1 step per frame
        want = np.stack([next(steps)[0] for _ in range(len(on[v]))])
        assert fits[v].dtype == np.int32 and np.array_equal(fits[v], want)
    assert not os.path.exists(str(tmp / 'fit' / 'on' / 'fit.npy'))
    pr.main(['--mode', 'ycbineoat_all', '--YCBInEOAT_dir', data, '--ycb_dir', ycb, '--outdir', str(tmp / 'fit' / 'cli'),
             '--max_frames', '5', '--fit', str(TAU), '--score'] + sum([['--' + k, v] for k, v in tpl.items()], []))
    assert 'fit check' in capsys.readouterr().out
    assert _poses_tree(str(tmp / 'fit' / 'cli')) == _poses_tree(str(tmp / 'fit' / 'plain'))


def test_ycbv_fit_and_score(pr, ycbv, capsys):
    tmp, tpl = ycbv
    ycb = str(tmp / 'ycb')
    run = lambda out, **kw: pr.getResultsYcbAll(ycb, [2, 5, 7], tpl, str(tmp / 'fit' / out), **kw)
    run('plain')
    run('on', fit=TAU)
    assert _poses_tree(str(tmp / 'fit' / 'plain')) == _poses_tree(str(tmp / 'fit' / 'on'))
    fits = _fits(str(tmp / 'fit' / 'on'))
    assert fits and all((f[0] == -1).all() and (f[1:, 0] > 0).all() for f in fits.values())
    for rel, f in fits.items():                                     # one row per pose file
        assert len([x for x in os.listdir(os.path.join(str(tmp / 'fit' / 'on'), rel)) if x.endswith('.txt')]) == len(f)
    sweep = run('sweep', fit=TAU, precision=['bf16x3', 'fp8'])
    for m in ('bf16x3', 'fp8'):
        run(m, fit=TAU, precision=m)
        a, b = _fits(str(tmp / 'fit' / m)), _fits(str(tmp / 'fit' / 'sweep' / m))
        assert sorted(a) == sorted(b) and all(np.array_equal(a[k], b[k]) for k in a)
    assert sweep
    r = pr.score_fit(str(tmp / 'fit' / 'on'), ycb, class_ids=[2, 5, 7])
    assert r['frames'] > 0 and 0 <= r['lost'] <= 1
    with pytest.raises(SystemExit, match='--fit'):
        pr.main(['--mode', 'ycbv', '--ycb_dir', ycb, '--outdir', str(tmp / 'x'), '--fit', '10', '--seq_id', '48']
                + sum([['--' + k, v] for k, v in tpl.items()], []))
