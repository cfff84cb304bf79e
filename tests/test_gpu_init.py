"""Start poses from a mask and the depth frame (se3tn_init_poses, Engine.init_poses, Tracker.initialize): the mask statistics,
every candidate row, the kept candidates, the ICP-refined poses and the final choice equal oracle/init_ref.py's; a frame drawn
at a grid candidate's rotation returns it; on the synthetic scene the start lands near the pose that drew it; calls are
bit-reproducible and leave tracking steps as they were; failed objects and refusals follow include/se3tn.h."""
import ctypes as C
import importlib
import os
import sys
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
PKG = 'iros20-6d-pose-tracking_b200'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import init_ref  # noqa: E402
import se3_oracle as so  # noqa: E402

L = importlib.import_module(PKG + '._lib')
synth_mod = importlib.import_module(PKG + '.synth')
K = synth_mod.CAMERA_K
HW = (480, 640)
WIDTH = 200.0
SMALL = dict(viewpoints=12, inplane=4, keep=3, tau_mm=20, min_pixels=100)
ICP = (2, 20, 100)                               # iterations, tau, min_inliers of the small case
# labelled_scene(seed=1), 8 objects, the defaults: on one H100 the median ADD-S of the returned starts was 0.69 mm (6 of 8 below
# 0.75 mm, two at 8.0 and 10.6 mm); the bound leaves headroom over that median
ADDS_BOUND_MM = 1.5


def _small_mesh(synth):
    m = dict(synth.mesh())
    m['pos'] = (m['pos'] * np.float32(0.7)).astype(np.float32)
    return m


@pytest.fixture(scope='module')
def scene(synth):
    mesh, gts, starts, D, seg = init_ref.labelled_scene(synth, 3, seed=0)
    return dict(mesh=mesh, gts=gts, D=D, seg=seg)


@pytest.fixture(scope='module')
def eng(pkg, synth):
    e = pkg.Engine(max_batch=20)                 # 48 candidates: chunks of 20, 20, 8; 3 objects: 144 rows in 8 chunks
    e.set_mesh(synth.mesh(), 0)
    e.set_mesh(_small_mesh(synth), 3)
    yield e
    e.close()


def _dev(e, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(e.device)


def _outs(e, n, spec, icp):
    VR, Kk = spec['viewpoints'] * spec['inplane'], spec['keep']
    f = lambda *s: torch.full(s, float('nan'), dtype=torch.float64, device=e.device)
    i = lambda *s: torch.full(s, -7, dtype=torch.int32, device=e.device)
    out = dict(stats=torch.full((n, 6), -7, dtype=torch.int64, device=e.device), t0=f(n, 3), cand_rows=i(n, VR, 8),
               kept_rows=i(n, Kk, 8), kept_poses=f(n, Kk, 4, 4))
    if icp:
        out.update(icp_poses=f(n, Kk, 4, 4), icp_rows=i(n, Kk, 8), icp_stats=f(n, Kk, 4))
    return out


def _call(e, sc, n, mode='vispy', icp=ICP, spec=SMALL, depth=None, seg=None, out=None):
    labels = [1, 2, 3][:n]
    ids = np.array([0, 3, 0][:n], np.int32)
    init = dict(spec, icp=None if icp is None else dict(iterations=icp[0], tau_mm=icp[1], min_inliers=icp[2]))
    out = _outs(e, n, spec, icp is not None) if out is None else out
    D = _dev(e, sc['D'] if depth is None else depth)
    S = _dev(e, sc['seg'] if seg is None else seg)
    ow = torch.full((n,), WIDTH, dtype=torch.float64, device=e.device)
    P, R = e.init_poses(D, S, K, labels, ow, weight_ids=ids, mode=mode, image_hw=HW if mode == 'pyrender' else None, init=init, out=out)
    torch.cuda.synchronize()
    return P.cpu().numpy(), R.cpu().numpy(), {k: v.cpu().numpy() for k, v in out.items()}, ids


@pytest.mark.parametrize('mode', ['vispy', 'pyrender'])
@pytest.mark.parametrize('n', [1, 3])
def test_every_stage_equals_the_oracle(eng, scene, synth, mode, n):
    P, R, o, ids = _call(eng, scene, n, mode)
    meshes = {0: scene['mesh'], 3: _small_mesh(synth)}
    V, Rr, Kk = SMALL['viewpoints'], SMALL['inplane'], SMALL['keep']
    H, W = HW if mode == 'pyrender' else (None, None)
    for i in range(n):
        ref = init_ref.init_object(scene['D'], scene['seg'], K, i + 1, WIDTH, meshes[int(ids[i])], V, Rr, Kk, SMALL['tau_mm'],
                                   SMALL['min_pixels'], icp=ICP, mode=mode, H=H, W=W, grid_poses=None)
        assert np.array_equal(o['stats'][i], ref['stats'])
        assert np.abs(o['t0'][i] - ref['t0']).max() <= 1e-12
        assert np.array_equal(o['cand_rows'][i], ref['rows'])
        assert np.array_equal(o['kept_rows'][i], ref['kept_rows'])
        assert np.abs(o['kept_poses'][i] - ref['kept_poses']).max() <= 1e-12
        # ICP from the device's kept poses, as test_gpu_icp checks the tracking step's
        ip = np.stack([init_ref.icp_ref.icp(Pk, K, WIDTH, meshes[int(ids[i])], scene['D'], ICP[1], ICP[2], ICP[0], mode, H, W)[0][-1]
                       for Pk in o['kept_poses'][i]])
        assert np.abs(o['icp_poses'][i] - ip).max() <= 1e-9
        rows = np.stack([init_ref.row(ref['stats'][0], c, init_ref.score_pose(Pk, K, WIDTH, meshes[int(ids[i])], scene['D'], scene['seg'],
                                                                             i + 1, SMALL['tau_mm'], mode, H, W, fixed_delta=True))
                         for c, Pk in zip(o['kept_rows'][i][:, 1], o['icp_poses'][i])])
        assert np.array_equal(o['icp_rows'][i], rows)
        best = init_ref.rank_order(rows)[0]
        assert np.array_equal(R[i], rows[best]) and np.array_equal(P[i], o['icp_poses'][i][best])


def test_without_icp_returns_the_top_grid_candidate(eng, scene):
    P, R, o, _ = _call(eng, scene, 3, icp=None)
    for i in range(3):
        assert np.array_equal(R[i], o['kept_rows'][i][0]) and np.array_equal(P[i], o['kept_poses'][i][0])
        order = init_ref.rank_order(o['cand_rows'][i])
        assert [int(c) for c in o['kept_rows'][i][:, 1]] == order[:SMALL['keep']]


def test_a_frame_drawn_at_a_grid_rotation_returns_it(eng, synth):
    # the frame is drawn at candidate c's rotation and a translation of its own; the call's grid sits at the t0 the mask gives
    # and moves along the ray by delta, so this checks that the rotation is recovered (or a view of equal score within 1 mm)
    mesh = synth.mesh()
    spec = dict(SMALL, keep=1)
    for c in (5, 22, 41):
        D = np.zeros(HW, np.uint16)
        P = np.eye(4)
        P[:3, :3] = init_ref.grid_rotation(c, spec['viewpoints'], spec['inplane'])
        P[:3, 3] = (0.02, -0.01, 0.7)
        D = init_ref.full_depth(P, K, mesh, *HW)
        seg = (D > 0).astype(np.uint8)
        Pd, R, o, _ = _call(eng, dict(D=D, seg=seg), 1, icp=None, spec=spec)
        got = int(R[0][1])
        if got != c:                                 # a symmetric view with an equal score
            rows = o['cand_rows'][0]
            x, y = rows[got], rows[c]
            assert int(x[6]) * max(int(y[2]) + y[3] - y[4], 1) == int(y[6]) * max(int(x[2]) + x[3] - x[4], 1)
            pts = mesh['pos'].astype(np.float64)
            G = init_ref.grid(spec['viewpoints'], spec['inplane'], o['t0'][0])
            assert so.adi(G[got], G[c], pts) < 1e-3


def test_synthetic_scene_accuracy(eng, pkg, synth):
    e = pkg.Engine(max_batch=64)
    try:
        e.set_mesh(synth.mesh(), 0)
        mesh, gts, _, D, seg = init_ref.labelled_scene(synth, 8, seed=1)
        n = 8
        ow = torch.full((n,), WIDTH, dtype=torch.float64, device=e.device)
        P, R = e.init_poses(_dev(e, D), _dev(e, seg), K, list(range(1, n + 1)), ow, init=None)
        P = P.cpu().numpy()
        pts = mesh['pos'].astype(np.float64)
        adds = [so.adi(P[i], gts[i], pts) * 1000 for i in range(n)]
        print('init ADD-S mm', np.round(adds, 2), 'rows', R.cpu().numpy())
        assert np.median(adds) < ADDS_BOUND_MM
    finally:
        e.close()


def test_two_calls_are_bit_identical(eng, scene):
    a = _call(eng, scene, 3)
    b = _call(eng, scene, 3)
    assert np.array_equal(a[0], b[0], equal_nan=True) and np.array_equal(a[1], b[1])
    for k in a[2]:
        assert np.array_equal(a[2][k], b[2][k], equal_nan=True), k


def test_tracking_step_is_unchanged_by_an_init_call(eng, scene, synth):
    mean, std = synth.default_mean_std()
    eng.load_state_dict(synth.make_state_dict(0), 0)
    eng.set_stats(mean, std, 0)
    rgb = _dev(eng, synth.raw_frame(3)[0])
    D = _dev(eng, scene['D'])
    poses = _dev(eng, scene['gts'])
    ow = torch.full((3,), WIDTH, dtype=torch.float64, device=eng.device)

    def step():
        r = eng.track_render(rgb, D, K, poses, ow, 0.03, 5 * np.pi / 180, fit=15, icp=2)
        torch.cuda.synchronize()
        return [t.cpu().numpy() for t in r]
    before = step()
    _call(eng, scene, 3)
    after = step()
    for x, y in zip(before, after):
        assert np.array_equal(x, y)


def test_failed_objects_get_their_status_and_nan(eng, scene):
    seg = scene['seg'].copy()
    D = scene['D'].copy()
    D[seg == 2] = 0                                  # object 2: a mask without depth
    seg[seg == 3] = 0                                # object 3: no mask
    P, R, o, _ = _call(eng, scene, 3, depth=D, seg=seg)
    assert R[0][0] == 0 and np.isfinite(P[0]).all()
    assert R[1][0] == 2 and np.isnan(P[1]).all() and o['stats'][1][0] == 2
    assert R[2][0] == 1 and np.isnan(P[2]).all() and o['stats'][2][0] == 1


def _raw(e, D, S, opts, labels, ids_h, ids_d, n, poses, rows, arrays=None, ow=None):
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    Kh = np.ascontiguousarray([K[0, 0], K[1, 1], K[0, 2], K[1, 2]])
    lab = np.ascontiguousarray(labels, np.int32)
    ow = torch.full((max(n, 1),), WIDTH, dtype=torch.float64, device=e.device) if ow is None else ow
    return e.lib.se3tn_init_poses(e._ctx, p(D), p(S), HW[0], HW[1], Kh.ctypes.data_as(C.c_void_p), lab.ctypes.data_as(C.c_void_p), p(ow),
                                  L.RENDER_VISPY, 0, 0, None if ids_h is None else ids_h.ctypes.data_as(C.c_void_p), p(ids_d), n,
                                  None if opts is None else C.byref(opts), p(poses), p(rows),
                                  None if arrays is None else C.byref(arrays), C.c_void_p(torch.cuda.current_stream().cuda_stream))


def test_refusals_queue_nothing(eng, scene):
    D, S = _dev(eng, scene['D']), _dev(eng, scene['seg'])
    n = 2
    poses = torch.full((n, 4, 4), float('nan'), dtype=torch.float64, device=eng.device)
    rows = torch.full((n, 8), -7, dtype=torch.int32, device=eng.device)
    good = lambda **kw: L.InitOpts(**dict(dict(viewpoints=4, inplane=2, keep=2, tau_mm=20, min_pixels=10), **kw))
    assert _raw(eng, D, S, good(), [1, 2], None, None, n, poses, rows) == L.OK
    torch.cuda.synchronize()
    assert (rows[:, 0] == 0).all()
    poses.fill_(float('nan')); rows.fill_(-7)
    torch.cuda.synchronize()
    bad_icp = L.IcpOpts(iterations=0, tau_mm=20, min_inliers=100)
    cases = [(good(viewpoints=0), 'viewpoints'), (good(viewpoints=4097), 'viewpoints'), (good(inplane=361), 'inplane'),
             (good(viewpoints=4096, inplane=17), 'inplane = '), (good(keep=0), 'keep'), (good(keep=9), 'keep'),
             (good(keep=11, viewpoints=20), 'max_batch'), (good(tau_mm=0), 'tau_mm'), (good(min_pixels=0), 'min_pixels'),
             (good(reserved=1), 'reserved'), (good(icp=C.pointer(bad_icp)), 'icp->iterations'), (None, 'opts is NULL')]
    for opts, what in cases:
        rc = _raw(eng, D, S, opts, [1, 2], None, None, n, poses, rows)
        assert rc == L.ERR_INVALID and what in L.load().se3tn_last_error(eng._ctx).decode(), what
    assert _raw(eng, D, S, good(), [0, 2], None, None, n, poses, rows) == L.ERR_INVALID          # label out of range
    assert _raw(eng, D, S, good(), [1, 256], None, None, n, poses, rows) == L.ERR_INVALID
    ids = np.array([0, 7], np.int32)                 # id 7 has no mesh
    assert _raw(eng, D, S, good(), [1, 2], ids, _dev(eng, ids), n, poses, rows) == L.ERR_STATE
    assert _raw(eng, D, S, good(), [1, 2], ids, None, n, poses, rows) == L.ERR_INVALID            # host ids without device ids
    arr = L.InitArrays(icp_poses=torch.empty(n, 2, 16, dtype=torch.float64, device=eng.device).data_ptr())
    assert _raw(eng, D, S, good(), [1, 2], None, None, n, poses, rows, arr) == L.ERR_INVALID       # ICP output without icp
    arr = L.InitArrays(t0=poses.data_ptr())
    assert _raw(eng, D, S, good(), [1, 2], None, None, n, poses, rows, arr) == L.ERR_INVALID       # two outputs overlap
    arr = L.InitArrays(cand_rows=S.data_ptr())
    assert _raw(eng, D, S, good(), [1, 2], None, None, n, poses, rows, arr) == L.ERR_INVALID       # an output over an input
    torch.cuda.synchronize()
    assert torch.isnan(poses).all() and (rows == -7).all()


def test_tracker_initialize_equals_the_engine_call(pkg, synth, scene):
    info = {'resolution': 176, 'boundingbox': 10, 'object_width': WIDTH,
            'camera': {'focalX': K[0, 0], 'focalY': K[1, 1], 'centerX': K[0, 2], 'centerY': K[1, 2], 'height': HW[0], 'width': HW[1]}}
    mean, std = synth.default_mean_std()
    trk = pkg.Tracker(info, mean, std, {'state_dict': synth.make_state_dict(0)}, model_path=None, max_batch=8)
    trk.renderer = importlib.import_module(PKG + '.cuda_renderer').CudaRenderer(synth.mesh(), K, trk.engine, WIDTH)
    start = trk.initialize(scene['D'], scene['seg'] == 2, label=5, viewpoints=12, inplane=4, keep=3)
    e = trk.engine
    ow = torch.full((1,), WIDTH, dtype=torch.float64, device=e.device)
    seg = np.where(scene['seg'] == 2, 5, 0).astype(np.uint8)
    P, R = e.init_poses(_dev(e, scene['D']), _dev(e, seg), K, [5], ow, init=dict(viewpoints=12, inplane=4, keep=3))
    assert np.array_equal(start, P[0].cpu().numpy()) and np.array_equal(trk.last_init, R[0].cpu().numpy())
    rgb = synth.raw_frame(3)[0]
    pose = trk.on_track(start, rgb, scene['D'])
    assert pose.shape == (4, 4) and np.isfinite(pose).all()
    with pytest.raises(ValueError, match='mask is empty'):
        trk.initialize(scene['D'], np.zeros(HW, bool))
    with pytest.raises(ValueError, match='labels 0..255'):
        trk.initialize(scene['D'], scene['seg'].astype(np.int32) * 200, label=2)


def test_tracker_initialize_scores_the_filled_depth(pkg, synth, scene):
    info = {'resolution': 176, 'boundingbox': 10, 'object_width': WIDTH,
            'camera': {'focalX': K[0, 0], 'focalY': K[1, 1], 'centerX': K[0, 2], 'centerY': K[1, 2], 'height': HW[0], 'width': HW[1]}}
    mean, std = synth.default_mean_std()
    fill = dict(max_depth=2.0, blur_type='gaussian')
    trk = pkg.Tracker(info, mean, std, {'state_dict': synth.make_state_dict(0)}, model_path=None, max_batch=8, fill_depth=fill)
    trk.renderer = importlib.import_module(PKG + '.cuda_renderer').CudaRenderer(synth.mesh(), K, trk.engine, WIDTH)
    raw = scene['D'].copy()
    raw[::7, ::5] = 0                                # holes the fill closes
    spec = dict(viewpoints=12, inplane=4, keep=3)
    start = trk.initialize(raw, scene['seg'], label=1, **spec)
    e = trk.engine
    filled = e.fill_depth(_dev(e, raw), 2.0, blur_type='gaussian')
    ow = torch.full((1,), WIDTH, dtype=torch.float64, device=e.device)
    P, R = e.init_poses(filled, _dev(e, scene['seg']), K, [1], ow, init=spec)
    assert np.array_equal(start, P[0].cpu().numpy()) and np.array_equal(trk.last_init, R[0].cpu().numpy())
    P_raw, _ = e.init_poses(_dev(e, raw), _dev(e, scene['seg']), K, [1], ow, init=spec)
    assert not np.array_equal(P_raw.cpu().numpy(), P.cpu().numpy())    # the raw frame scores differently
