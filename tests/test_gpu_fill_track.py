"""Raw sensor depth in, hole-filled inside the tracking step (se3tn_track_opts' fill, Engine track calls' fill_depth=,
Tracker(fill_depth=)): every step must give the same bits as Engine.fill_depth on the whole frame followed by the same entry
point with the fill off, whatever the graph cache, the upload window or a Tracker sharing the Engine did before."""
import ctypes as C
import importlib
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
TN, RN = 0.03, 5 * np.pi / 180
K = importlib.import_module('iros20-6d-pose-tracking_b200.synth').CAMERA_K
ENTRIES = ('track_batch', 'track_render', 'track_host', 'track_render_host')
BRANCHES = [dict(extrapolate=True), dict(blur_type='gaussian', max_depth=1.8), dict(extrapolate=True, blur_type='gaussian')]


def _make_engine(pkg, synth, max_batch=64):
    e = pkg.Engine(max_batch=max_batch)
    mean, std = synth.default_mean_std()
    e.load_state_dict(synth.make_state_dict(0), 0)
    e.set_stats(mean, std, 0)
    e.set_mesh(synth.mesh(2, seed=0), 0)
    return e


@pytest.fixture(scope='module')
def eng(pkg, synth):
    e = _make_engine(pkg, synth)
    yield e
    e.close()


@pytest.fixture(scope='module', autouse=True)
def keep_utils_engine():
    """Every Tracker points Utils' shared engine at its own, and these tests close theirs: restore the one set before."""
    U = importlib.import_module('iros20-6d-pose-tracking_b200.Utils')
    saved = U._engine
    yield
    U.set_engine(saved)


def _centre(p):
    return int(round(K[1, 1] * p[1, 3] / p[2, 3] + K[1, 2])), int(round(K[0, 0] * p[0, 3] / p[2, 3] + K[0, 2]))


def _raw(synth, seed, poses, far=True):
    """synth.raw_frame plus holes inside the first tracks' crop windows: a small one the diamond dilation closes and a large one
    that is still empty after the 7x7 fill.  far=False drops the depths beyond 2 m, whose filled metres are negative."""
    rgb, depth = synth.raw_frame(seed)
    for p in poses[:4]:
        v, u = _centre(p)
        depth[max(v - 6, 0):max(v - 2, 0), max(u - 6, 0):max(u - 2, 0)] = 0
        depth[max(v, 0):max(v + 24, 0), max(u, 0):max(u + 24, 0)] = 0
    if not far:
        depth[depth > 2000] = 0
    return rgb, depth


def _dev(e, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(e.device)


class Case:
    def __init__(self, e, synth, n, seed, poses=None, far=True):
        self.poses = synth.raw_poses(n, seed=seed) if poses is None else poses
        self.rgb, self.depth = _raw(synth, seed, self.poses, far)
        self.n = n
        self.R, self.D, self.P = _dev(e, self.rgb), _dev(e, self.depth), _dev(e, self.poses)
        self.ow = torch.full((n,), 200.0, dtype=torch.float64, device=e.device)
        self.ra, self.da = e.render(K, self.P, self.ow)             # input A of the entry points that take it


def _run(e, entry, c, depth, fill=None, precision='bf16x3', outs=None):
    """One call of `entry` on case c with the given depth frame (CUDA tensor for the device entry points, numpy for the host
    ones) -> (poses, trans, rot) as numpy."""
    if entry == 'track_batch':
        r = e.track_batch(c.R, depth, K, c.P, c.ow, c.ra, c.da, TN, RN, precision=precision, fill_depth=fill, **(outs or {}))
    elif entry == 'track_render':
        r = e.track_render(c.R, depth, K, c.P, c.ow, TN, RN, precision=precision, fill_depth=fill, **(outs or {}))
    elif entry == 'track_host':
        return e.track_host(c.rgb, depth, K, c.poses, np.full(c.n, 200.0), c.ra.cpu().numpy(), c.da.cpu().numpy(), TN, RN,
                            precision=precision, want_residuals=True, fill_depth=fill)
    else:
        return e.track_render_host(c.rgb, depth, K, c.poses, np.full(c.n, 200.0), TN, RN, precision=precision, want_residuals=True,
                                   fill_depth=fill)
    return tuple(x.cpu().numpy() for x in r)


def _filled(e, D, fill=None):
    kw = {} if fill in (None, True) else fill
    return e.fill_depth(D, **kw)


def _frame(entry, c, D):
    """The depth frame in the form `entry` takes."""
    return D.cpu().numpy() if entry.endswith('host') else D


def _equal(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize('entry', ENTRIES)
def test_same_bits_as_fill_then_track(synth, eng, entry):
    for n in (1, 64):
        c = Case(eng, synth, n, seed=n)
        want = _run(eng, entry, c, _frame(entry, c, _filled(eng, c.D)))
        plain = eng.last_launch_count()
        for rep in range(2):                                      # the second call replays the step's graph
            got = _run(eng, entry, c, _frame(entry, c, c.D), fill=True)
            assert _equal(got, want), (entry, n, rep)
            assert eng.last_step_was_graph() and eng.last_launch_count() == plain + 8, (entry, n)
        assert np.isfinite(got[0]).all()


@pytest.mark.parametrize('fill', BRANCHES, ids=['extrapolate', 'gaussian', 'extrapolate+gaussian'])
def test_other_branches(synth, eng, fill):
    c = Case(eng, synth, 5, seed=31)
    want = _run(eng, 'track_render', c, _filled(eng, c.D, fill))
    plain = eng.last_launch_count()
    got = _run(eng, 'track_render', c, c.D, fill=fill)
    assert _equal(got, want), fill
    extra = (6 if fill.get('blur_type') == 'gaussian' else 8) + (3 if fill.get('extrapolate') else 0)
    assert eng.last_launch_count() == plain + extra


def test_fp32_and_profiled_steps(synth, eng):
    """SE3TN_PREC_FP32 and an enabled profiler run plain stream launches, no graph."""
    c = Case(eng, synth, 5, seed=37)
    F = _filled(eng, c.D)
    want = _run(eng, 'track_batch', c, F, precision='fp32')
    assert _equal(_run(eng, 'track_batch', c, c.D, fill=True, precision='fp32'), want)
    assert not eng.last_step_was_graph()
    want = _run(eng, 'track_render', c, F)
    eng.set_profiling(True)
    try:
        got = _run(eng, 'track_render', c, c.D, fill=True)
        assert not eng.last_step_was_graph()
        assert eng.get_profile()[17] > 0                          # K0 ran and was timed
    finally:
        eng.set_profiling(False)
    assert _equal(got, want)


def _tracker(pkg, synth, tmp_path, engine=None, **kw):
    mio = importlib.import_module('iros20-6d-pose-tracking_b200.mesh_io')
    path = str(tmp_path / 'model.ply')
    mio.save_ply_mesh(path, synth.mesh(2, seed=4))
    info = {'resolution': 176, 'object_width': 200.0, 'boundingbox': 10,
            'camera': {'focalX': K[0, 0], 'focalY': K[1, 1], 'centerX': K[0, 2], 'centerY': K[1, 2], 'height': 480, 'width': 640}}
    mean, std = synth.default_mean_std()
    trk = pkg.Tracker(info, mean, std, {'state_dict': synth.make_state_dict(0)}, model_path=path, max_batch=8, engine=engine, **kw)
    assert type(trk.renderer).__name__ == 'CudaRenderer'
    return trk


def test_whole_frame_is_filled(pkg, synth, eng, tmp_path):
    """One small crop window; a large patch at 60 m far outside it survives the hole filling and the median, so it sets the
    minimum of the median-filtered (inverted) image.  That stretches the bilateral's range table from about 1.5 m to about 60 m
    and changes the filled depth inside the window.  The host entry points and both of the Tracker's routes must fill the
    whole depth frame, over two frames that differ only outside the window."""
    p = np.eye(4); p[:3, 3] = (0.0, 0.0, 1.5)                      # a 142-pixel window around the image centre
    c = Case(eng, synth, 1, seed=41, poses=p[None])
    far = c.depth.copy(); far[400:470, 10:80] = 60000
    frames = [far, c.depth]                                       # equal inside the window
    top, left = 241 - 80, 313 - 80
    filled = [_filled(eng, _dev(eng, f)).cpu().numpy() for f in frames]
    assert np.array_equal(frames[0][top:top + 160, left:left + 160], frames[1][top:top + 160, left:left + 160])
    assert not np.array_equal(filled[0][top:top + 160, left:left + 160], filled[1][top:top + 160, left:left + 160])
    for entry in ('track_host', 'track_render_host'):
        for f, fl in zip(frames, filled):
            want = _run(eng, entry, c, fl)
            got = _run(eng, entry, c, f, fill=True)
            assert _equal(got, want), entry
    # Tracker.on_track_batch on numpy frames (the host route) and on CUDA tensors (the device route)
    trk = _tracker(pkg, synth, tmp_path, fill_depth=True)
    try:
        plain = _tracker(pkg, synth, tmp_path, engine=trk.engine)
        T = lambda a: _dev(trk.engine, a)
        for f, fl in zip(frames, filled):
            assert np.array_equal(trk.on_track_batch(p[None], c.rgb, f), plain.on_track_batch(p[None], c.rgb, fl))
            got = trk.on_track_batch(T(p[None]), T(c.rgb), T(f))
            assert got.is_cuda and torch.equal(got, plain.on_track_batch(T(p[None]), T(c.rgb), T(fl)))
    finally:
        trk.engine.close()


def test_graph_replay_and_new_frame_values(synth, eng):
    c = Case(eng, synth, 5, seed=43)
    outs = dict(out_poses=torch.empty_like(c.P), out_trans=torch.empty(5, 3, device=eng.device), out_rot=torch.empty(5, 3, device=eng.device))
    for _ in range(2):
        _run(eng, 'track_render', c, c.D, fill=True, outs=outs)
    assert eng.last_step_was_graph()
    _, new = _raw(synth, 44, c.poses)
    c.D.copy_(_dev(eng, new))                                      # the same buffer with a new frame: the replayed graph fills it
    got = _run(eng, 'track_render', c, c.D, fill=True, outs=outs)
    assert eng.last_step_was_graph()
    assert _equal(got, _run(eng, 'track_render', c, _filled(eng, c.D)))


def test_larger_plain_fill_between_filled_steps(pkg, synth):
    """se3tn_fill_depth on a larger frame replaces the fill block that captured steps hold: they are dropped and captured again."""
    e = _make_engine(pkg, synth, max_batch=8)
    try:
        c = Case(e, synth, 5, seed=47)
        want = _run(e, 'track_render', c, _filled(e, c.D))
        for _ in range(2):
            assert _equal(_run(e, 'track_render', c, c.D, fill=True), want)
        assert e.last_step_was_graph()
        _, big = synth.raw_frame(seed=48, h=960, w=1280)
        e.fill_depth(_dev(e, big))
        for _ in range(2):
            assert _equal(_run(e, 'track_render', c, c.D, fill=True), want)
            assert e.last_step_was_graph()
    finally:
        e.close()


def test_trackers_sharing_an_engine(pkg, synth, tmp_path):
    """A Tracker that fills and one that does not, on one Engine (and so the same host-call buffers and device frames),
    interleaved: each gives what it gives alone."""
    trk = _tracker(pkg, synth, tmp_path)
    try:
        fil = _tracker(pkg, synth, tmp_path, engine=trk.engine, fill_depth=True)
        e = trk.engine
        poses = synth.raw_poses(3, seed=51)
        frames = [_raw(synth, 52 + f, poses) for f in range(3)]
        T = lambda a: _dev(e, a)
        alone = [(trk.on_track(poses[0], r, d), trk.on_track_batch(poses, r, d), trk.on_track_batch(T(poses), T(r), T(d)).cpu().numpy())
                 for r, d in frames]
        for (r, d), want in zip(frames, alone):
            fd = _filled(e, T(d)).cpu().numpy()
            assert np.array_equal(fil.on_track(poses[0], r, d), trk.on_track(poses[0], r, fd))
            assert np.array_equal(trk.on_track(poses[0], r, d), want[0])
            assert np.array_equal(fil.on_track_batch(poses, r, d), trk.on_track_batch(poses, r, fd))
            assert np.array_equal(trk.on_track_batch(poses, r, d), want[1])
            R, D = T(r), T(d)                                      # one set of device buffers for both
            got = fil.on_track_batch(T(poses), R, D).cpu().numpy()
            assert np.array_equal(trk.on_track_batch(T(poses), R, D).cpu().numpy(), want[2])
            assert np.array_equal(got, trk.on_track_batch(T(poses), R, T(fd)).cpu().numpy())
    finally:
        trk.engine.close()


def test_raw_depth_is_not_written(synth, eng):
    c = Case(eng, synth, 5, seed=53)
    keep_t, keep_a = c.D.clone(), c.depth.copy()
    for entry in ENTRIES:
        _run(eng, entry, c, c.depth if entry.endswith('host') else c.D, fill=True)
        torch.cuda.synchronize()
        assert torch.equal(c.D, keep_t) and np.array_equal(c.depth, keep_a), entry


def _raw_track_batch(e, c, outs, opts=None):
    K4 = e._k4(K)
    vp = lambda t: C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)
    return e.lib.se3tn_track_batch(e._ctx, vp(c.R), vp(c.D), 480, 640, K4.ctypes.data_as(C.c_void_p), vp(c.P), vp(c.ow), vp(c.ra), vp(c.da),
                                   C.c_void_p(0), C.c_void_p(0), c.n, TN, RN, 2, vp(outs[1]), vp(outs[2]), vp(outs[0]),
                                   None if opts is None else C.byref(opts), C.c_void_p(torch.cuda.current_stream(e.device).cuda_stream))


def test_errors_and_fill_off(pkg, synth, eng):
    lib = pkg.engine._lib
    c = Case(eng, synth, 5, seed=59)
    want_fill = _run(eng, 'track_batch', c, _filled(eng, c.D))
    nan_outs = lambda: [torch.full((5, 4, 4), float('nan'), dtype=torch.float64, device=eng.device),
                        torch.full((5, 3), float('nan'), device=eng.device), torch.full((5, 3), float('nan'), device=eng.device)]
    bad = [{'blur_type': 'box'}, {'max_depth': 0}, {'max_depth': -1}, {'max_depth': float('nan')}, {'max_dpth': 2.0}, 'yes']
    for b in bad:                                                  # rejected in Python before anything is queued
        o = nan_outs()
        before = eng.last_launch_count()
        for entry in ENTRIES:
            with pytest.raises(ValueError):
                _run(eng, entry, c, _frame(entry, c, c.D), fill=b, outs=dict(out_poses=o[0], out_trans=o[1], out_rot=o[2]))
        torch.cuda.synchronize()
        assert eng.last_launch_count() == before and all(torch.isnan(x).all() for x in o), b
        with pytest.raises(ValueError):
            pkg.Tracker({}, None, None, None, fill_depth=b)
    # ... and in C, where a rejected call launches nothing, writes nothing and names the field
    before = eng.last_launch_count()
    for (max_depth, extrapolate, blur), field in (((2.0, 0, 7), b'fill_blur'), ((0.0, 0, 0), b'fill_max_depth'),
                                                  ((-1.0, 0, 0), b'fill_max_depth'), ((float('nan'), 0, 0), b'fill_max_depth'),
                                                  ((float('inf'), 0, 1), b'fill_max_depth'), ((1e300, 1, 0), b'fill_max_depth')):
        o = nan_outs()
        opts = lib.TrackOpts(fill_depth=1, fill_max_depth=max_depth, fill_extrapolate=extrapolate, fill_blur=blur, iterations=1)
        assert _raw_track_batch(eng, c, o, opts) == lib.ERR_INVALID, (max_depth, extrapolate, blur)
        assert field in eng.lib.se3tn_last_error(eng._ctx)
        torch.cuda.synchronize()
        assert all(torch.isnan(x).all() for x in o)
    assert eng.last_launch_count() == before
    o = nan_outs()
    assert _raw_track_batch(eng, c, o, lib.TrackOpts(fill_depth=1, fill_max_depth=2.0, iterations=1)) == lib.OK
    assert _equal([x.cpu().numpy() for x in o], want_fill)
    # fill off: the same bits and launches as a fresh context's step without options
    fresh = _make_engine(pkg, synth)
    try:
        cf = Case(fresh, synth, 5, seed=59)
        o = nan_outs()
        assert _raw_track_batch(fresh, cf, o) == lib.OK
        want, launches = [x.cpu().numpy() for x in o], fresh.last_launch_count()
    finally:
        fresh.close()
    assert _equal(_run(eng, 'track_batch', c, c.D), want)
    assert eng.last_launch_count() == launches == 11             # K0 + 8 resident convs + trunk + head/K6
    assert _equal(_run(eng, 'track_batch', c, c.D, fill=False), want)


@pytest.mark.parametrize('render_in_step', [True, False])
def test_tracker_drop_in_for_the_ros_node(pkg, synth, tmp_path, render_in_step):
    """Tracker(fill_depth=True).on_track(p, rgb, raw) is the reference ROS node's
    on_track(p, rgb, (fill_depth(raw / 1e3) * 1000).astype(uint16)), bit for bit, over a closed 20-frame sequence.  The frames
    have no depth beyond max_depth: numpy's conversion of the negative metres those give to uint16 is undefined."""
    U = importlib.import_module('iros20-6d-pose-tracking_b200.Utils')
    fil = _tracker(pkg, synth, tmp_path, fill_depth=True)
    ros = _tracker(pkg, synth, tmp_path)
    try:
        pa = np.eye(4); pa[:3, 3] = (0.02, -0.01, 1.0)
        pb = pa.copy()
        for f in range(20):
            rgb, raw = _raw(synth, 200 + f, pa[None], far=False)
            U.set_engine(ros.engine)
            depth = (U.fill_depth(raw / 1e3) * 1000).astype(np.uint16)
            if render_in_step:
                a, b = fil.on_track(pa, rgb, raw), ros.on_track(pb, rgb, depth)
            else:
                ra, da = fil.render_window(pa)
                a = fil.on_track(pa, rgb, raw, rgbA=ra, depthA=da)
                b = ros.on_track(pb, rgb, depth, rgbA=ra, depthA=da)
            assert np.isfinite(a).all() and np.array_equal(a, b), f
            pa, pb = a, b
    finally:
        fil.engine.close()
        ros.engine.close()
