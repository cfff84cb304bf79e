"""Refinement rounds inside one tracking step (se3tn_track_opts.iterations, Engine.track_render(iterations=k), Tracker(iterations=k),
the one-pass drivers' iterations=): a k-round step must give the bits of k chained single-round steps on the same device frame,
whatever the render mode, depth fill, precision, batch size or mix of weight sets; the host call those of the device call; and the
graph key, launch count and refusals must follow include/se3tn.h."""
import ctypes as C
import importlib
import os
import numpy as np
import pytest
import torch
from test_gpu_precision_sweep import eoat, ycbv, pr      # the synthetic layouts of the driver tests  # noqa: F401

pytestmark = pytest.mark.gpu
PKG = 'iros20-6d-pose-tracking_b200'
TN, RN = 0.03, 5 * np.pi / 180
HW = (480, 640)
SETS = (0, 5)                                   # two weight sets under sparse ids
K = importlib.import_module(PKG + '.synth').CAMERA_K


def _make_engine(pkg, synth, max_batch=64):
    e = pkg.Engine(max_batch=max_batch)
    mean, std = synth.default_mean_std()
    for j, wid in enumerate(SETS):
        e.load_state_dict(synth.make_state_dict(j), wid)
        e.set_mesh(synth.mesh(2 - j, seed=j), wid)
        e.set_stats(mean + 1.5 * j, std * (1 + 0.25 * j), wid)
    return e


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


@pytest.fixture(scope='module')
def eng(pkg, synth):
    e = _make_engine(pkg, synth)
    c = Case(e, synth, 6, seed=3)                                  # every set calibrated for 'fp8' on round-0 inputs
    e.calibrate_fp8_tracks(c.R, c.D, K, c.P, c.ow, weight_ids=c.wid, render=dict(mode='vispy', image_hw=None, mesh_ids=c.wd))
    assert all(e.fp8_scales(w) is not None for w in SETS)
    yield e
    e.close()


@pytest.fixture(scope='module', autouse=True)
def keep_utils_engine():
    U = importlib.import_module(PKG + '.Utils')
    saved = U._engine
    yield
    U.set_engine(saved)


def _step(e, c, P, k, prec, mode, fill, out_poses=None):
    n = c.n
    outs = dict(out_poses=torch.empty_like(P) if out_poses is None else out_poses,
                out_trans=torch.full((n, 3), float('nan'), device=e.device), out_rot=torch.full((n, 3), float('nan'), device=e.device))
    return e.track_render(c.R, c.D, K, P, c.ow, TN, RN, weight_ids_host=c.wid, weight_ids_dev=c.wd, precision=prec, mode=mode,
                          image_hw=HW if mode == 'pyrender' else None, fill_depth=fill, iterations=k, **outs)


def _chained(e, c, k, prec, mode, fill):
    P = c.P.clone()
    for _ in range(k):
        P, tr, ro = _step(e, c, P, 1, prec, mode, fill)
    return P, tr, ro


def _same(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize('fill', [False, True], ids=['raw', 'fill'])
@pytest.mark.parametrize('mode', ['vispy', 'pyrender'])
@pytest.mark.parametrize('prec', ['bf16x3', 'bf16', 'fp8', 'fp32'])
def test_k_rounds_equal_k_chained_steps(synth, eng, prec, mode, fill):
    for n in (1, 5, 64):
        c = Case(eng, synth, n, seed=n)
        for k in (2, 3):
            want = _chained(eng, c, k, prec, mode, fill)
            got = _step(eng, c, c.P, k, prec, mode, fill)
            assert _same(got, want), (prec, mode, fill, n, k)
            P = c.P.clone()                                         # in place: poses_out == poses_in
            inplace = _step(eng, c, P, k, prec, mode, fill, out_poses=P)
            assert _same(inplace, want), (prec, mode, fill, n, k, 'in place')
            assert torch.isfinite(got[0]).all() and not torch.equal(got[0], c.P)


@pytest.mark.parametrize('mode', ['vispy', 'pyrender'])
@pytest.mark.parametrize('fill', [False, True], ids=['raw', 'fill'])
def test_host_call_equals_device_call(synth, eng, mode, fill):
    for n in (1, 5):
        c = Case(eng, synth, n, seed=20 + n)
        want = [x.cpu().numpy() for x in _step(eng, c, c.P, 3, 'bf16x3', mode, fill)]
        for rep in range(2):                                        # the second call replays the step's graph
            got = eng.track_render_host(c.rgb, c.depth, K, c.poses, np.full(n, 200.0), TN, RN, weight_ids=c.wid, mode=mode,
                                        image_hw=HW if mode == 'pyrender' else None, want_residuals=True, fill_depth=fill, iterations=3)
            assert all(np.array_equal(g, w) for g, w in zip(got, want)), (mode, fill, n, rep)
        assert eng.last_step_was_graph()


def test_graph_replay_and_launch_count(pkg, synth, eng):
    c = Case(eng, synth, 5, seed=41)
    P = c.P.clone()
    _step(eng, c, P, 1, 'bf16x3', 'vispy', False, out_poses=P)
    per_round = eng.last_launch_count()
    _step(eng, c, P, 1, 'bf16x3', 'vispy', True, out_poses=P)
    fill = eng.last_launch_count() - per_round
    assert fill == 8                                                # the bilateral fill (include/se3tn.h)
    for k in (2, 3, 8):
        for f in (False, True):
            for rep in range(2):
                _step(eng, c, P, k, 'bf16x3', 'vispy', f, out_poses=P)
                assert eng.last_launch_count() == (fill if f else 0) + k * per_round, (k, f)
                if rep:
                    assert eng.last_step_was_graph(), (k, f)
    _step(eng, c, P, 3, 'fp32', 'vispy', False, out_poses=P)
    assert not eng.last_step_was_graph()


def test_k_back_to_one_is_a_context_that_never_set_it(pkg, synth, eng):
    fresh = _make_engine(pkg, synth)
    try:
        c = Case(eng, synth, 5, seed=43)
        _step(eng, c, c.P, 3, 'bf16x3', 'vispy', False)
        got = _step(eng, c, c.P, 1, 'bf16x3', 'vispy', False)
        launches = eng.last_launch_count()
        cf = Case(fresh, synth, 5, seed=43)
        want = fresh.track_render(cf.R, cf.D, K, cf.P, cf.ow, TN, RN, weight_ids_host=cf.wid, weight_ids_dev=cf.wd)
        assert all(torch.equal(a.cpu(), b.cpu()) for a, b in zip(got, want))
        assert launches == fresh.last_launch_count()
    finally:
        fresh.close()


def _byref(opts):
    return None if opts is None else C.byref(opts)


def _raw_track_batch(e, c, ra, da, out, opts=None):
    Kh = np.ascontiguousarray([K[0, 0], K[1, 1], K[0, 2], K[1, 2]])
    p = lambda t: C.c_void_p(t.data_ptr())
    return e.lib.se3tn_track_batch(e._ctx, p(c.R), p(c.D), HW[0], HW[1], Kh.ctypes.data_as(C.c_void_p), p(c.P), p(c.ow), p(ra), p(da),
                                   c.wid.ctypes.data_as(C.c_void_p), p(c.wd), c.n, TN, RN, 2, p(out[1]), p(out[2]), p(out[0]),
                                   _byref(opts), C.c_void_p(torch.cuda.current_stream().cuda_stream))


def _raw_track_host(e, c, ra, da, out, opts=None):
    Kh = np.ascontiguousarray([K[0, 0], K[1, 1], K[0, 2], K[1, 2]])
    h = lambda a: a.ctypes.data_as(C.c_void_p)
    return e.lib.se3tn_track_host(e._ctx, h(c.rgb), h(c.depth), HW[0], HW[1], h(Kh), h(c.poses), h(np.full(c.n, 200.0)), h(ra), h(da),
                                  h(c.wid), c.n, TN, RN, 2, h(out[0]), h(out[1]), h(out[2]), _byref(opts), C.c_void_p(0))


def _raw_track_render(e, c, P, out, opts=None, rounds=None):
    Kh = np.ascontiguousarray([K[0, 0], K[1, 1], K[0, 2], K[1, 2]])
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    arrays = importlib.import_module(PKG + '._lib').TrackArrays(round_poses=None if rounds is None else rounds.data_ptr())
    return e.lib.se3tn_track_render(e._ctx, p(c.R), p(c.D), HW[0], HW[1], Kh.ctypes.data_as(C.c_void_p), p(P), p(c.ow), 0, 0, 0,
                                    c.wid.ctypes.data_as(C.c_void_p), p(c.wd), c.n, TN, RN, 2, p(out[1]), p(out[2]), p(out[0]),
                                    _byref(opts), C.byref(arrays),
                                    C.c_void_p(torch.cuda.current_stream().cuda_stream))


def test_refusals(synth, eng):
    L = importlib.import_module(PKG + '._lib')
    c = Case(eng, synth, 4, seed=45)
    ra, da = eng.render(K, c.P, c.ow, c.wd)
    dev_out = lambda: (torch.full((4, 4, 4), float('nan'), dtype=torch.float64, device=eng.device),
                       torch.full((4, 3), float('nan'), device=eng.device), torch.full((4, 3), float('nan'), device=eng.device))
    host_out = lambda: (np.full((4, 4, 4), np.nan), np.full((4, 3), np.nan, np.float32), np.full((4, 3), np.nan, np.float32))
    refused = lambda rc, field: rc == L.ERR_INVALID and field in eng.lib.se3tn_last_error(eng._ctx)
    out = dev_out()
    assert _raw_track_batch(eng, c, ra, da, out, L.TrackOpts(iterations=1)) == L.OK     # k = 1: track_batch runs
    torch.cuda.synchronize()
    assert torch.isfinite(out[0]).all()
    launches = eng.last_launch_count()
    for bad in (0, 9, -1, 2, 3):              # out of range for every call; k > 1 for the two calls that take input A
        opts = L.TrackOpts(iterations=bad)
        out, hout, rout = dev_out(), host_out(), dev_out()
        assert refused(_raw_track_batch(eng, c, ra, da, out, opts), b'iterations'), bad
        assert refused(_raw_track_host(eng, c, ra.cpu().numpy(), da.cpu().numpy(), hout, opts), b'iterations'), bad
        if bad not in (2, 3):
            assert refused(_raw_track_render(eng, c, c.P, rout, opts), b'iterations'), bad
        torch.cuda.synchronize()
        assert all(torch.isnan(x).all() for x in out + rout) and all(np.isnan(x).all() for x in hout), bad
    # round_poses must not overlap the poses a later round reads: over poses_out, then over poses_in
    rounds = torch.full((3, 4, 4, 4), float('nan'), dtype=torch.float64, device=eng.device)
    out = dev_out()
    assert refused(_raw_track_render(eng, c, c.P, (rounds[2],) + out[1:], L.TrackOpts(iterations=3), rounds), b'round_poses')
    rounds[0].copy_(c.P)
    assert refused(_raw_track_render(eng, c, rounds[0], out, L.TrackOpts(iterations=3), rounds), b'round_poses')
    torch.cuda.synchronize()
    assert all(torch.isnan(x).all() for x in out) and torch.isnan(rounds[1:]).all()
    assert eng.last_launch_count() == launches
    for bad in (0, 9, 2.0, True):
        with pytest.raises(ValueError, match='iterations'):
            eng.track_render(c.R, c.D, K, c.P, c.ow, TN, RN, iterations=bad)
    # a track_render call with k = 3 leaves nothing on the context that the Engine's own track_batch would have to undo
    eng.track_render(c.R, c.D, K, c.P, c.ow, TN, RN, iterations=3)
    eng.track_batch(c.R, c.D, K, c.P, c.ow, ra, da, TN, RN)


def _tracker(pkg, synth, tmp_path, **kw):
    mio = importlib.import_module(PKG + '.mesh_io')
    path = str(tmp_path / 'model.ply')
    mio.save_ply_mesh(path, synth.mesh(2, seed=4))
    info = {'resolution': 176, 'object_width': 200.0, 'boundingbox': 10,
            'camera': {'focalX': K[0, 0], 'focalY': K[1, 1], 'centerX': K[0, 2], 'centerY': K[1, 2], 'height': 480, 'width': 640}}
    mean, std = synth.default_mean_std()
    return pkg.Tracker(info, mean, std, {'state_dict': synth.make_state_dict(0)}, model_path=path, renderer='cuda', max_batch=4, **kw)


@pytest.mark.parametrize('prec', ['bf16x3', 'fp8'])
def test_tracker(pkg, synth, tmp_path, prec):
    one, three = _tracker(pkg, synth, tmp_path, precision=prec), _tracker(pkg, synth, tmp_path, precision=prec, iterations=3)
    try:
        rgb, depth = synth.raw_frame(50)
        pose = synth.raw_poses(1, seed=50)[0]
        want = pose
        for _ in range(3):
            want = one.on_track(want, rgb, depth)
        assert np.array_equal(three.on_track(pose, rgb, depth), want)
        if prec == 'fp8':                                           # calibrated on the frame's round-0 inputs, as with k = 1
            assert np.array_equal(three.engine.fp8_scales(0), one.engine.fp8_scales(0))
        poses = synth.raw_poses(3, seed=51)
        chained = poses
        for _ in range(3):
            chained = one.on_track_batch(chained, rgb, depth)
        assert np.array_equal(three.on_track_batch(poses, rgb, depth), chained)          # host route
        got = three.on_track_batch(torch.from_numpy(poses).cuda(), torch.from_numpy(rgb).cuda(), torch.from_numpy(depth).cuda())
        assert np.array_equal(got.cpu().numpy(), chained)                                 # device route
        rgbA, depthA = one.render_window(pose)
        with pytest.raises(ValueError, match='input A was passed in'):
            three.on_track(pose, rgb, depth, rgbA=rgbA, depthA=depthA)
        with pytest.raises(ValueError, match='input A was passed in'):
            three.on_track_batch(poses[:1], rgb, depth, rgbA[None], depthA[None])
    finally:
        one.engine.close(); three.engine.close()


def test_tracker_needs_the_cuda_renderer(pkg, synth):
    info = {'resolution': 176, 'object_width': 200.0, 'boundingbox': 10,
            'camera': {'focalX': K[0, 0], 'focalY': K[1, 1], 'centerX': K[0, 2], 'centerY': K[1, 2], 'height': 480, 'width': 640}}
    mean, std = synth.default_mean_std()
    with pytest.raises(ValueError, match='CUDA renderer'):
        pkg.Tracker(info, mean, std, {'state_dict': synth.make_state_dict(0)}, max_batch=1, iterations=2)


def _tree(root):
    out = {}
    for d, _, fs in os.walk(root):
        for f in fs:
            with open(os.path.join(d, f), 'rb') as x:
                out[os.path.relpath(os.path.join(d, f), root)] = x.read()
    return out


def test_ycbineoat_sweep_of_counts(pr, eoat):
    tmp, tpl = eoat
    data, ycb = str(tmp / 'data'), str(tmp / 'ycb')
    run = lambda out, **kw: pr.getResultsYcbInEOAT(data, tpl, str(tmp / 'refine' / out), ycb_dir=ycb, **kw)
    plain = run('plain')
    sweep = run('sweep', iterations=[1, 2])
    assert sorted(sweep) == [1, 2] and sorted(os.listdir(tmp / 'refine' / 'sweep')) == ['iter1', 'iter2']
    for k in (1, 2):
        single = run('k%d' % k, iterations=k)
        assert all(np.array_equal(single[v], sweep[k][v]) for v in single)
        assert _tree(str(tmp / 'refine' / ('k%d' % k))) == _tree(str(tmp / 'refine' / 'sweep' / ('iter%d' % k)))
    assert _tree(str(tmp / 'refine' / 'k1')) == _tree(str(tmp / 'refine' / 'plain'))
    assert all(np.array_equal(plain[v], sweep[1][v]) for v in plain)
    assert any(not np.array_equal(sweep[1][v], sweep[2][v]) for v in plain)
    both = run('both', iterations=[2, 1], precision=['fp8', 'bf16x3'])
    assert list(both) == [2, 1] and all(list(both[k]) == ['fp8', 'bf16x3'] for k in both)
    for k in (1, 2):
        for m in ('fp8', 'bf16x3'):
            single = run('k%d_%s' % (k, m), iterations=k, precision=m)
            assert all(np.array_equal(single[v], both[k][m][v]) for v in single)
            assert _tree(str(tmp / 'refine' / ('k%d_%s' % (k, m)))) == _tree(str(tmp / 'refine' / 'both' / ('iter%d' % k) / m))


def test_ycbv_sweep_of_counts_and_score(pr, ycbv, capsys):
    tmp, tpl = ycbv
    ycb = str(tmp / 'ycb')
    run = lambda out, **kw: pr.getResultsYcbAll(ycb, [2, 5, 7], tpl, str(tmp / 'refine' / out), **kw)
    sweep = run('sweep', iterations=[1, 2])
    for k in (1, 2):
        run('k%d' % k, iterations=k)
        assert _tree(str(tmp / 'refine' / ('k%d' % k))) == _tree(str(tmp / 'refine' / 'sweep' / ('iter%d' % k)))
    run('plain')
    assert _tree(str(tmp / 'refine' / 'k1')) == _tree(str(tmp / 'refine' / 'plain'))
    ref, rows = pr.score_iterations(sweep, str(tmp / 'refine' / 'sweep'), ycb, tpl)
    assert ref == 'iter1' and list(rows) == ['iter1', 'iter2']
    assert rows['iter1']['add_max'] == 0 and rows['iter2']['add_max'] > 0
    assert 'variant iter2' in capsys.readouterr().out
