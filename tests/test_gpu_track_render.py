"""Tracking from the previous poses and the frame alone: se3tn_track_render / se3tn_track_render_host render input A inside
the step (render -> K0 -> conv stack -> head + K6) and must give the same bits as the two-call path (se3tn_render_ex, then
se3tn_track_batch) on the same inputs, and the reference's pose within POSE_ATOL when the oracle renders input A."""
import ctypes as C
import importlib
import numpy as np
import pytest
import torch
import se3_oracle as O

pytestmark = pytest.mark.gpu
POSE_ATOL = 1e-4
TN, RN = 0.03, 5 * np.pi / 180
HW = (480, 640)
PRECS = ('bf16x3', 'tf32', 'bf16', 'fp32')
K = importlib.import_module('iros20-6d-pose-tracking_b200.synth').CAMERA_K


@pytest.fixture(scope='module')
def models(synth):
    return {0: synth.mesh(2, seed=0), 1: synth.mesh(1, seed=1)}


def _make_engine(pkg, synth, models):
    e = pkg.Engine(max_batch=64)
    mean, std = synth.default_mean_std()
    for wid in (0, 1):
        e.load_state_dict(synth.make_state_dict(wid), wid)
        e.set_mesh(models[wid], wid)
    e.set_stats(mean, std, 0)
    e.set_stats(mean + 1.5, std * 1.25, 1)
    return e


@pytest.fixture(scope='module')
def eng(pkg, synth, models):
    e = _make_engine(pkg, synth, models)
    yield e
    e.close()


def _dev(eng, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(eng.device)


def _ids(n):
    """Interleaved weight / mesh ids; a single track uses the NULL-ids path (set 0, mesh 0)."""
    return None if n == 1 else (np.arange(n) % 2).astype(np.int32)


def _case(eng, synth, n, seed, edge=True):
    rgb, depth = synth.raw_frame(seed)
    poses = synth.raw_poses(n, seed=seed)
    if edge:
        poses[0, :3, 3] = (0.32, -0.2, 0.5)                       # the first window hangs over the frame's edge
    return rgb, depth, poses, _dev(eng, rgb), _dev(eng, depth), _dev(eng, poses), torch.full((n,), 200.0, dtype=torch.float64, device=eng.device)


def _two_call(eng, R, D, P, ow, wid, prec, mode, **outs):
    """What a caller did before: render input A into its own tensors, then track_batch on them."""
    ids = _dev(eng, wid) if wid is not None else None
    ra, da = eng.render(K, P, ow, ids, mode=mode, image_hw=HW if mode == 'pyrender' else None)
    return eng.track_batch(R, D, K, P, ow, ra, da, TN, RN, weight_ids_host=wid, weight_ids_dev=ids, precision=prec, **outs)


def _fused(eng, R, D, P, ow, wid, prec, mode, **outs):
    ids = _dev(eng, wid) if wid is not None else None
    return eng.track_render(R, D, K, P, ow, TN, RN, weight_ids_host=wid, weight_ids_dev=ids, precision=prec, mode=mode,
                            image_hw=HW if mode == 'pyrender' else None, **outs)


def _equal(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize('mode', ['vispy', 'pyrender'])
@pytest.mark.parametrize('prec', PRECS)
def test_same_bits_as_render_then_track_batch(synth, eng, mode, prec):
    for n in (1, 5, 64):
        rgb, depth, poses, R, D, P, ow = _case(eng, synth, n, seed=n)
        wid = _ids(n)
        want = _two_call(eng, R, D, P, ow, wid, prec, mode)
        got = _fused(eng, R, D, P, ow, wid, prec, mode)
        assert _equal(got, want), (mode, prec, n)
        assert torch.isfinite(got[0]).all()


@pytest.mark.parametrize('mode', ['vispy', 'pyrender'])
def test_host_call_equals_device_call(synth, eng, mode):
    hw = HW if mode == 'pyrender' else None
    for n in (1, 5):
        rgb, depth, poses, R, D, P, ow = _case(eng, synth, n, seed=40 + n)
        if n > 1:
            poses[1, :3, 3] = (2.0, 2.0, 0.5)                     # this window misses the frame entirely
            P = _dev(eng, poses)
        ow_h = np.full(n, 200.0); ow_h[-1] = 150.0
        ow = _dev(eng, ow_h)
        wid = _ids(n)
        want = [x.cpu().numpy() for x in _fused(eng, R, D, P, ow, wid, 'bf16x3', mode)]
        for rep in range(2):                                      # the second call replays the step's graph
            got = eng.track_render_host(rgb, depth, K, poses, ow_h, TN, RN, weight_ids=wid, mode=mode, image_hw=hw, want_residuals=True)
            assert all(np.array_equal(g, w) for g, w in zip(got, want)), (mode, n, rep)
        assert eng.last_step_was_graph()


@pytest.mark.parametrize('mode', ['vispy', 'pyrender'])
def test_matches_oracle_fed_with_the_oracle_render(synth, eng, models, mode):
    n = 3
    rgb, depth, poses, R, D, P, ow = _case(eng, synth, n, seed=7, edge=False)     # the oracle's crop_bbox needs windows that overlap the frame
    wid = np.array([0, 1, 0], dtype=np.int32)
    got = eng.track_render_host(rgb, depth, K, poses, np.full(n, 200.0), TN, RN, weight_ids=wid, mode=mode,
                                image_hw=HW if mode == 'pyrender' else None)
    mean, std = synth.default_mean_std()
    stats = {0: (mean, std), 1: (mean + 1.5, std * 1.25)}
    for i in range(n):
        k = int(wid[i])
        ra, da = (O.render_window(poses[i], K, 200.0, models[k]) if mode == 'vispy'
                  else O.render_window_pyrender(poses[i], K, 200.0, models[k], *HW))
        ref = O.on_track(synth.make_state_dict(k), poses[i], rgb, depth, ra, da, K, 200.0, *stats[k], TN, RN)
        assert np.abs(got[i] - ref).max() < POSE_ATOL, (mode, i)


def test_graph_replay_and_new_pose_values(pkg, synth, eng, models, monkeypatch):
    n = 5
    rgb, depth, poses, R, D, P, ow = _case(eng, synth, n, seed=11)
    wid = _ids(n)
    outs = dict(out_poses=torch.empty_like(P), out_trans=torch.empty(n, 3, device=eng.device), out_rot=torch.empty(n, 3, device=eng.device))
    _two_call(eng, R, D, P, ow, wid, 'bf16x3', 'vispy', **outs)
    batch_launches = eng.last_launch_count()
    for _ in range(2):
        _fused(eng, R, D, P, ow, wid, 'bf16x3', 'vispy', **outs)
    assert eng.last_step_was_graph() and eng.last_launch_count() == batch_launches + 2
    # the same buffers with new pose values: the replayed graph reads them
    new = synth.raw_poses(n, seed=12)
    P.copy_(_dev(eng, new))
    got = [x.clone() for x in _fused(eng, R, D, P, ow, wid, 'bf16x3', 'vispy', **outs)]
    assert eng.last_step_was_graph()
    monkeypatch.setenv('SE3TN_GRAPH', '0')
    plain = _make_engine(pkg, synth, models)
    try:
        want = _fused(plain, _dev(plain, rgb), _dev(plain, depth), _dev(plain, new), ow.clone(), wid, 'bf16x3', 'vispy')
        assert not plain.last_step_was_graph()
        assert _equal(got, want)
    finally:
        plain.close()


def test_set_mesh_redraws_captured_steps(synth, eng, models):
    n = 5
    rgb, depth, poses, R, D, P, ow = _case(eng, synth, n, seed=13)
    wid = _ids(n)
    outs = dict(out_poses=torch.empty_like(P), out_trans=torch.empty(n, 3, device=eng.device), out_rot=torch.empty(n, 3, device=eng.device))
    for _ in range(2):
        old = [x.clone() for x in _fused(eng, R, D, P, ow, wid, 'bf16x3', 'vispy', **outs)]
    assert eng.last_step_was_graph()
    bigger = synth.mesh(3, seed=5)                                # 4x the faces of model 0: a larger projected-vertex workspace
    assert len(bigger['pos']) > max(len(m['pos']) for m in models.values())
    try:
        eng.set_mesh(bigger, 0)
        got = [x.clone() for x in _fused(eng, R, D, P, ow, wid, 'bf16x3', 'vispy', **outs)]
        want = _two_call(eng, R, D, P, ow, wid, 'bf16x3', 'vispy')
        assert _equal(got, want)
        assert not torch.equal(got[0], old[0])
    finally:
        eng.set_mesh(models[0], 0)


def test_closed_loop_poses_out_to_poses_in(synth, eng):
    n = 5
    rgb, depth, poses, R, D, P, ow = _case(eng, synth, n, seed=17)
    wid = _ids(n)
    ids = _dev(eng, wid)
    bufs = [P.clone(), torch.empty_like(P)]
    tr, ro = torch.empty(n, 3, device=eng.device), torch.empty(n, 3, device=eng.device)
    ref = P.clone()
    for f in range(5):
        frgb, fdepth = synth.raw_frame(seed=60 + f)
        R.copy_(_dev(eng, frgb)); D.copy_(_dev(eng, fdepth))
        eng.track_render(R, D, K, bufs[0], ow, TN, RN, weight_ids_host=wid, weight_ids_dev=ids, out_poses=bufs[1], out_trans=tr, out_rot=ro)
        ra, da = eng.render(K, ref, ow, ids)
        ref, _, _ = eng.track_batch(R, D, K, ref, ow, ra, da, TN, RN, weight_ids_host=wid, weight_ids_dev=ids)
        assert torch.equal(bufs[1], ref), f
        bufs.reverse()


def _raw_track_render(eng, R, D, P, ow, mode, rh, rw, wid, n, outs):
    wh = np.ascontiguousarray(wid, dtype=np.int32) if wid is not None else None
    wd = _dev(eng, wh) if wh is not None else None
    K4 = eng._k4(K)
    vp = lambda t: C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)
    return eng.lib.se3tn_track_render(eng._ctx, vp(R), vp(D), R.shape[0], R.shape[1], K4.ctypes.data_as(C.c_void_p), vp(P), vp(ow), mode, rh, rw,
                                      wh.ctypes.data_as(C.c_void_p) if wh is not None else C.c_void_p(0), vp(wd), n, TN, RN, 2,
                                      vp(outs[1]), vp(outs[2]), vp(outs[0]), None, None,
                                      C.c_void_p(torch.cuda.current_stream(eng.device).cuda_stream))


def test_errors_launch_nothing_and_leave_the_context_usable(pkg, synth, eng):
    lib = pkg.engine._lib
    n = 5
    rgb, depth, poses, R, D, P, ow = _case(eng, synth, n, seed=19)
    wid = _ids(n)
    want = [x.clone() for x in _two_call(eng, R, D, P, ow, wid, 'bf16x3', 'vispy')]
    mean, std = synth.default_mean_std()
    eng.load_state_dict(synth.make_state_dict(2), 2); eng.set_mesh(synth.mesh(0, seed=2), 2)        # id 2: no statistics
    eng.set_mesh(synth.mesh(0, seed=3), 3)                                                          # id 3: a model only
    eng.load_state_dict(synth.make_state_dict(4), 4); eng.set_stats(mean, std, 4)                   # id 4: no model
    big = 65
    Pb, owb = P[:1].expand(big, 4, 4).contiguous(), torch.full((big,), 200.0, dtype=torch.float64, device=eng.device)
    cases = [('no statistics', lambda o: _raw_track_render(eng, R, D, P, ow, 0, 0, 0, [0, 1, 2, 0, 1], n, o), lib.ERR_STATE),
             ('no weights', lambda o: _raw_track_render(eng, R, D, P, ow, 0, 0, 0, [0, 3, 0, 1, 0], n, o), lib.ERR_STATE),
             ('no mesh', lambda o: _raw_track_render(eng, R, D, P, ow, 0, 0, 0, [0, 1, 0, 1, 4], n, o), lib.ERR_STATE),
             ('n > max_batch', lambda o: _raw_track_render(eng, R, D, Pb, owb, 0, 0, 0, None, big, o), lib.ERR_INVALID),
             ('unknown mode', lambda o: _raw_track_render(eng, R, D, P, ow, 7, *HW, wid, n, o), lib.ERR_INVALID),
             ('render_H', lambda o: _raw_track_render(eng, R, D, P, ow, 1, 0, 640, wid, n, o), lib.ERR_INVALID),
             ('render_W', lambda o: _raw_track_render(eng, R, D, P, ow, 1, 480, 70000, wid, n, o), lib.ERR_INVALID)]
    for name, call, code in cases:
        m = big if name == 'n > max_batch' else n
        outs = [torch.full((m, 4, 4), float('nan'), dtype=torch.float64, device=eng.device),
                torch.full((m, 3), float('nan'), device=eng.device), torch.full((m, 3), float('nan'), device=eng.device)]
        before = eng.last_launch_count()
        assert call(outs) == code, name
        torch.cuda.synchronize()
        assert eng.last_launch_count() == before and all(torch.isnan(o).all() for o in outs), name
        if name == 'no mesh':
            assert b'4' in eng.lib.se3tn_last_error(eng._ctx)
        got = _fused(eng, R, D, P, ow, wid, 'bf16x3', 'vispy')                # the next valid call is correct
        assert _equal(got, want), name
    # the same checks through the host entry point and the Python layer
    with pytest.raises(pkg.engine._lib.Se3tnError) as e:
        eng.track_render_host(rgb, depth, K, poses, np.full(n, 200.0), TN, RN, weight_ids=np.array([0, 1, 4, 0, 1], np.int32))
    assert e.value.code == lib.ERR_STATE
    with pytest.raises(pkg.engine._lib.Se3tnError) as e:
        eng.track_render_host(rgb, depth, K, np.tile(poses[:1], (big, 1, 1)), np.full(big, 200.0), TN, RN)
    assert e.value.code == lib.ERR_INVALID
    with pytest.raises(pkg.engine._lib.Se3tnError) as e:
        eng.track_render_host(rgb, depth, K, poses, np.full(n, 200.0), TN, RN, mode='pyrender', image_hw=(480, 0))
    assert e.value.code == lib.ERR_INVALID
    with pytest.raises(ValueError):
        eng.track_render(R, D, K, P, ow, TN, RN, mode='opengl')
    got = eng.track_render_host(rgb, depth, K, poses, np.full(n, 200.0), TN, RN, weight_ids=wid)
    assert np.array_equal(got, want[0].cpu().numpy())


def _tracker(pkg, synth, tmp_path, pyrender):
    mio = importlib.import_module('iros20-6d-pose-tracking_b200.mesh_io')
    mesh = synth.mesh(2, seed=4)
    info = {'resolution': 176, 'object_width': 200.0, 'boundingbox': 10,
            'camera': {'focalX': K[0, 0], 'focalY': K[1, 1], 'centerX': K[0, 2], 'centerY': K[1, 2], 'height': HW[0], 'width': HW[1]}}
    if pyrender:
        path = str(tmp_path / 'model.obj')
        with open(path, 'w') as f:
            for v, c in zip(mesh['pos'], mesh['col']):
                f.write('v %.9g %.9g %.9g %.9g %.9g %.9g\n' % (*v, *(c / 255.0)))
            for t in mesh['faces']:
                f.write('f %d %d %d\n' % tuple(t + 1))
        info['renderer'] = 'pyrenderer'
    else:
        path = str(tmp_path / 'model.ply')
        mio.save_ply_mesh(path, mesh)
    mean, std = synth.default_mean_std()
    trk = pkg.Tracker(info, mean, std, {'state_dict': synth.make_state_dict(0)}, model_path=path, max_batch=8)
    assert type(trk.renderer).__name__ == 'CudaRenderer' and trk.renderer.mode == ('pyrender' if pyrender else 'vispy')
    return trk


@pytest.mark.parametrize('pyrender', [False, True])
def test_tracker_renders_inside_the_step(pkg, synth, tmp_path, monkeypatch, pyrender):
    trk = _tracker(pkg, synth, tmp_path, pyrender)
    try:
        rgb, depth = synth.raw_frame(seed=23)
        poses = synth.raw_poses(3, seed=23)
        # the old sequence: render_window, then on_track with input A
        ras, das = zip(*[trk.render_window(p) for p in poses])
        want1 = trk.on_track(poses[0], rgb, depth, rgbA=ras[0], depthA=das[0])
        wantn = trk.on_track_batch(poses, rgb, depth, np.stack(ras), np.stack(das))
        dev = trk.engine.device
        T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        wantt = trk.on_track_batch(T(poses), T(rgb), T(depth), T(np.stack(ras)), T(np.stack(das)))

        def no_render(*a, **k):
            raise AssertionError('tracking must not call Engine.render')
        monkeypatch.setattr(pkg.Engine, 'render', no_render)
        for _ in range(2):
            assert np.array_equal(trk.on_track(poses[0], rgb, depth), want1)
        assert np.array_equal(trk.on_track_batch(poses, rgb, depth), wantn)
        got = trk.on_track_batch(T(poses), T(rgb), T(depth))
        assert got.is_cuda and torch.equal(got, wantt)
        assert trk.frame_cnt == 3
    finally:
        trk.engine.close()


def test_tracker_keeps_user_built_renderers(pkg, synth):
    """A CudaRenderer built by the caller renders on its own engine with its own camera, model and width.  Where the tracking
    step cannot draw the same (another engine or K, another mesh id, another width), the Tracker renders input A first, as
    before: on_track equals render_window + on_track with input A, on_track_batch equals render_batch + on_track_batch."""
    cr = importlib.import_module('iros20-6d-pose-tracking_b200.cuda_renderer')
    mean, std = synth.default_mean_std()
    info = {'resolution': 176, 'object_width': 200.0, 'boundingbox': 10,
            'camera': {'focalX': K[0, 0], 'focalY': K[1, 1], 'centerX': K[0, 2], 'centerY': K[1, 2], 'height': HW[0], 'width': HW[1]}}
    mesh = synth.mesh(2, seed=4)
    rgb, depth = synth.raw_frame(seed=29)
    poses = synth.raw_poses(3, seed=29)
    own = pkg.Engine(max_batch=8)                                 # the renderer's engine
    eng = pkg.Engine(max_batch=8)                                 # the Tracker's engine
    try:
        cases = {'second engine, float32 K': (own, dict(K=K.astype(np.float32))),
                 'mesh_id 3': (eng, dict(mesh_id=3)),
                 'width 180': (eng, dict(object_width=180.0))}
        for name, (e, kw) in cases.items():
            args = dict(K=K, object_width=200.0)
            args.update(kw)
            r = cr.CudaRenderer(mesh, args.pop('K'), e, args.pop('object_width'), **args)
            trk = pkg.Tracker(info, mean, std, {'state_dict': synth.make_state_dict(0)}, model_path=None, engine=eng, renderer=r)
            ra, da = r.render_window(poses[0])
            assert np.array_equal(trk.on_track(poses[0], rgb, depth), trk.on_track(poses[0], rgb, depth, rgbA=ra, depthA=da)), name
            P = torch.from_numpy(poses).to(eng.device)
            ras, das = r.render_batch(P, torch.full((3,), 200.0, dtype=torch.float64, device=eng.device))
            want = trk.on_track_batch(poses, rgb, depth, ras.cpu().numpy(), das.cpu().numpy())
            assert np.array_equal(trk.on_track_batch(poses, rgb, depth), want), name
    finally:
        own.close()
        eng.close()
