"""Re-initialisation of lost tracks (se3tn_lost_tracks, se3tn_fit_poses, se3tn_accept_starts, Engine.reinit, Tracker(reinit=)):
the loss and accept rules equal oracle/reinit_ref.py bit for bit; fit_poses gives exactly the fit rows of a tracking step at
that step's poses; refusals follow include/se3tn.h; and a Tracker restarts an object that jumped, with the pose a lone
init_poses call gives, while the other object's poses keep the bits of a Tracker without re-initialisation."""
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
import reinit_ref as R  # noqa: E402

L = importlib.import_module(PKG + '._lib')
synth_mod = importlib.import_module(PKG + '.synth')
K = synth_mod.CAMERA_K
HW = (480, 640)
TN, RN = 0.03, 5 * np.pi / 180
SETS = (0, 5)
TAU = 15
MAX_BATCH = 64
WIDTH = 200.0
# the jump case below, at the init defaults: on one H100 80GB HBM3 (700 W limit) the restarted object's ADD-S was 1.63 mm; the
# bound leaves headroom over it
ADDS_BOUND_MM = 5.0


@pytest.fixture(scope='module')
def eng(pkg, synth):
    e = pkg.Engine(max_batch=MAX_BATCH)
    mean, std = synth.default_mean_std()
    for j, wid in enumerate(SETS):
        e.load_state_dict(synth.make_state_dict(j), wid)
        e.set_mesh(synth.mesh(2 - j, seed=j), wid)
        e.set_stats(mean + 1.5 * j, std * (1 + 0.25 * j), wid)
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


# ---------------------------------------------------------------------------------------------------- 1. the loss rule
@pytest.mark.parametrize('n', [1, MAX_BATCH])
def test_lost_tracks_equal_the_oracle(eng, n):
    rng = np.random.default_rng(n)
    streak_ref = np.zeros(n, np.int32)
    streak = torch.zeros(n, dtype=torch.int32, device=eng.device)
    seen_lost = 0
    for step in range(12):
        model = rng.choice([0, 1, 100, 30976], size=n)
        inlier = (rng.uniform(size=n) * (model + 1)).astype(np.int64).clip(0, model)
        if step % 4 == 3:
            inlier = model * 3 // 10                        # exactly at 300 permille: not below there
        rows = np.zeros((n, 6), np.int32)
        rows[:, 0], rows[:, 1], rows[:, 2] = model, model, inlier
        streak_ref, event_ref, lost_ref = R.lost_tracks(rows, streak_ref, 300, 2)
        out_lost = torch.full((n + 1,), -9, dtype=torch.int32, device=eng.device)
        event, lost = eng.lost_tracks(_dev(eng, rows), streak, 0.3, 2, out_lost=out_lost)
        torch.cuda.synchronize()
        assert eng.last_launch_count() == 1
        lost = lost.cpu().numpy()
        assert np.array_equal(streak.cpu().numpy(), streak_ref) and np.array_equal(event.cpu().numpy(), event_ref)
        assert lost[0] == len(lost_ref) and np.array_equal(lost[1:1 + lost[0]], lost_ref)
        assert (lost[1 + lost[0]:] == -9).all()               # entries past the count are not written
        seen_lost += len(lost_ref)
    assert seen_lost > 0


def test_lost_tracks_over_several_scan_tiles(pkg):
    # lost_kernel scans 1024 tracks per tile: 1100 tracks carry the count of the first tile into the second
    n = 1100
    e = pkg.Engine(max_batch=n)
    try:
        rng = np.random.default_rng(7)
        streak_ref = np.zeros(n, np.int32)
        streak = torch.zeros(n, dtype=torch.int32, device=e.device)
        for step in range(4):
            model = rng.choice([0, 50, 100], size=n)
            inlier = (rng.uniform(size=n) * (model + 1)).astype(np.int64).clip(0, model)
            rows = np.zeros((n, 6), np.int32)
            rows[:, 0], rows[:, 2] = model, inlier
            streak_ref, event_ref, lost_ref = R.lost_tracks(rows, streak_ref, 500, 2)
            event, lost = e.lost_tracks(_dev(e, rows), streak, 0.5, 2)
            lost = lost.cpu().numpy()
            assert np.array_equal(streak.cpu().numpy(), streak_ref) and np.array_equal(event.cpu().numpy(), event_ref)
            assert lost[0] == len(lost_ref) and np.array_equal(lost[1:1 + lost[0]], lost_ref)
            assert step == 0 or ((lost_ref < 1024).any() and (lost_ref >= 1024).any())
    finally:
        e.close()


def test_lost_tracks_refusals(eng):
    n = 4
    rows = torch.zeros(n, 6, dtype=torch.int32, device=eng.device)
    streak, event = torch.zeros(n, dtype=torch.int32, device=eng.device), torch.zeros(n, dtype=torch.int32, device=eng.device)
    lost = torch.zeros(n + 1, dtype=torch.int32, device=eng.device)
    call = lambda o, n=n, s=streak, ev=event: eng.lib.se3tn_lost_tracks(eng._ctx, C.c_void_p(rows.data_ptr()), n, C.byref(o),
                                                                     C.c_void_p(s.data_ptr()), C.c_void_p(ev.data_ptr()),
                                                                     C.c_void_p(lost.data_ptr()), C.c_void_p(0))
    for opts, what in ((L.ReinitOpts(0, 3), 'below_permille'), (L.ReinitOpts(1001, 3), 'below_permille'), (L.ReinitOpts(500, 0), 'after'),
                       (L.ReinitOpts(500, 1001), 'after'), (L.ReinitOpts(500, 3, (C.c_int32 * 2)(0, 1)), 'reserved')):
        assert call(opts) == L.ERR_INVALID and what in eng.lib.se3tn_last_error(eng._ctx).decode()
    assert call(L.ReinitOpts(500, 3), n=MAX_BATCH + 1) == L.ERR_INVALID
    assert call(L.ReinitOpts(500, 3), ev=streak) == L.ERR_INVALID and 'overlap' in eng.lib.se3tn_last_error(eng._ctx).decode()
    torch.cuda.synchronize()
    assert (streak == 0).all() and (event == 0).all()       # nothing was queued


# ---------------------------------------------------------------------------------------------------- 2. the fit at given poses
def _frame(synth, seed):
    rgb, depth = synth.raw_frame(seed)
    return rgb, depth


@pytest.mark.parametrize('mode', ['vispy', 'pyrender'])
@pytest.mark.parametrize('fill', [False, True])
def test_fit_poses_equal_the_step_rows(synth, eng, mode, fill):
    n = 6
    rgb, depth = _frame(synth, 11)
    poses = synth.raw_poses(n, seed=12)
    wid = np.array([SETS[i % 2] for i in range(n)], np.int32)
    ow = torch.full((n,), WIDTH, dtype=torch.float64, device=eng.device)
    image_hw = HW if mode == 'pyrender' else None
    P, _, _, rows = eng.track_render(_dev(eng, rgb), _dev(eng, depth), K, _dev(eng, poses), ow, TN, RN, weight_ids_host=wid,
                                     weight_ids_dev=_dev(eng, wid), mode=mode, image_hw=image_hw, fit=TAU,
                                     fill_depth=True if fill else None)
    frame = eng.fill_depth(_dev(eng, depth), 2.0) if fill else _dev(eng, depth)
    got = eng.fit_poses(frame, K, P, ow, TAU, weight_ids=wid, mode=mode, image_hw=image_hw)
    torch.cuda.synchronize()
    assert eng.last_launch_count() == 3
    assert np.array_equal(got.cpu().numpy(), rows.cpu().numpy())
    assert (rows.cpu().numpy()[:, 0] > 0).all() and (rows.cpu().numpy()[:, 2] > 0).any()


def test_fit_poses_leave_captured_steps_alone(synth, eng):
    n = 3
    rgb, depth = _frame(synth, 21)
    poses = _dev(eng, synth.raw_poses(n, seed=22))
    ow = torch.full((n,), WIDTH, dtype=torch.float64, device=eng.device)
    args = (_dev(eng, rgb), _dev(eng, depth), K, poses, ow, TN, RN)
    a = [t.clone() for t in eng.track_render(*args, fit=TAU)]
    fit_block = eng._fit_rows_view()[:n].clone()
    other = eng.fit_poses(_dev(eng, np.full(HW, 700, np.uint16)), K, synth_pose_far(n, eng), ow, 5)
    assert torch.equal(eng._fit_rows_view()[:n], fit_block)   # se3tn_fit_rows' buffer is not written
    b = eng.track_render(*args, fit=TAU)
    assert eng.last_step_was_graph()
    torch.cuda.synchronize()
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    # a pose with a non-finite entry draws nothing: its row is all 0
    bad = poses.clone()
    bad[1, 0, 3] = float('nan')
    rows = eng.fit_poses(args[1], K, bad, ow, TAU).cpu().numpy()
    assert (rows[1] == 0).all() and rows[0, 0] > 0 and other.shape == (n, 6)


def synth_pose_far(n, e):
    P = torch.eye(4, dtype=torch.float64, device=e.device).repeat(n, 1, 1)
    P[:, 2, 3] = 0.7
    return P.contiguous()


def test_fit_poses_refusals(synth, eng):
    n = 2
    depth = _dev(eng, np.zeros(HW, np.uint16))
    poses = synth_pose_far(n, eng)
    ow = torch.full((n,), WIDTH, dtype=torch.float64, device=eng.device)
    with pytest.raises(ValueError):
        eng.fit_poses(depth, K, poses, ow, 0)
    with pytest.raises(L.Se3tnError, match='has no mesh') as ei:
        eng.fit_poses(depth, K, poses, ow, TAU, weight_ids=[0, 7])
    assert ei.value.code == L.ERR_STATE
    with pytest.raises(L.Se3tnError, match='overlap'):
        eng.fit_poses(depth, K, poses, ow, TAU, out=poses.view(torch.int32).view(-1)[:n * 6].view(n, 6))


# ---------------------------------------------------------------------------------------------------- 3. the accept rule
def test_accept_starts_equal_the_oracle(eng):
    n = 7
    rng = np.random.default_rng(5)
    poses = rng.normal(size=(n, 4, 4))
    rows = np.array([[100, 80, 50, 10, 20, 500]] * n, np.int32)
    rows[6] = 0
    lost = np.array([1, 2, 3, 4, 6], np.int32)
    starts = rng.normal(size=(len(lost), 4, 4))
    init_rows = np.zeros((len(lost), 8), np.int32)
    init_rows[3, 0] = 1                                       # track 4: no start
    init_rows[:, 2:] = 77                                     # the rest of the init row is not read
    start_fit = np.array([[100, 90, 50, 0, 40, 500],           # a tie with the tracked row: rejected
                          [200, 200, 101, 0, 99, 1],           # a higher fraction: restarted
                          [200, 200, 100, 0, 100, 999],        # the same fraction, a lower mean residual: restarted
                          [400, 400, 400, 0, 0, 0],            # would win, but init failed
                          [1, 0, 0, 0, 1, 0]], np.int32)       # model > 0 ranks above model = 0: restarted
    streak = np.array([5, 2, 2, 2, 2, 5, 2], np.int32)
    event = np.array([0, 1, 1, 1, 1, 0, 1], np.int32)
    ref = R.accept_starts(lost, starts.reshape(-1, 16), init_rows, start_fit, poses.reshape(n, 16), rows, streak, event)
    d = [_dev(eng, a) for a in (poses, rows, streak, event)]
    eng.accept_starts(lost, _dev(eng, starts), _dev(eng, init_rows), _dev(eng, start_fit), *d)
    torch.cuda.synchronize()
    assert eng.last_launch_count() == 1
    got = [t.cpu().numpy() for t in d]
    assert list(got[3]) == [0, R.REJECTED, R.RESTARTED, R.RESTARTED, R.NO_START, 0, R.RESTARTED]
    assert np.array_equal(got[0].reshape(n, 16), ref[0])      # bit for bit: restarted poses are the starts' bits
    for g, r in zip(got[1:], ref[1:]):
        assert np.array_equal(g, r)
    assert np.array_equal(got[0][[0, 5]], poses[[0, 5]]) and list(got[2]) == [5, 0, 0, 0, 0, 5, 0]


def test_accept_starts_refusals(eng):
    n = 4
    z = lambda *s, dt=torch.int32: torch.zeros(*s, dtype=dt, device=eng.device)
    poses, rows, streak, event = z(n, 4, 4, dt=torch.float64), z(n, 6), z(n), z(n)
    starts, init_rows, start_fit = z(2, 4, 4, dt=torch.float64), z(2, 8), z(2, 6)
    for lost, msg in (([1, 1], 'repeats'), ([0, 4], 'not in'), ([-1, 2], 'not in')):
        with pytest.raises(L.Se3tnError, match=msg):
            eng.accept_starts(lost, starts, init_rows, start_fit, poses, rows, streak, event)
    with pytest.raises(L.Se3tnError, match='overlap'):
        eng.accept_starts([0, 1], starts, init_rows, start_fit, poses, rows, streak, streak)
    torch.cuda.synchronize()
    assert (poses == 0).all() and (rows == 0).all() and (streak == 0).all() and (event == 0).all()


# ---------------------------------------------------------------------------------------------------- 4. the Tracker
def _zero_head_tracker(pkg, synth, tmp_path, reinit, max_batch=2):
    path = str(tmp_path / 'model.ply')
    importlib.import_module(PKG + '.mesh_io').save_ply_mesh(path, synth.mesh())     # the model labelled_scene draws
    info = {'resolution': 176, 'boundingbox': 10, 'object_width': WIDTH,
            'camera': {'focalX': K[0, 0], 'focalY': K[1, 1], 'centerX': K[0, 2], 'centerY': K[1, 2], 'height': HW[0], 'width': HW[1]}}
    mean, std = synth.default_mean_std()
    sd = synth.make_state_dict(2)
    for k in ('trans_out.0.weight', 'trans_out.0.bias', 'rot_out.0.weight', 'rot_out.0.bias'):
        sd[k] = torch.zeros_like(sd[k])                       # the pose update is the identity: poses move only when restarted
    return pkg.Tracker(info, mean, std, {'state_dict': sd}, model_path=path, renderer='cuda', max_batch=max_batch, reinit=reinit)


def _adds_mm(mesh, P, G):
    pts = mesh['pos'].astype(np.float64)
    a = pts @ P[:3, :3].T + P[:3, 3]
    b = pts @ G[:3, :3].T + G[:3, 3]
    d = np.sqrt(((a[:, None, :] - b[None, :, :]) ** 2).sum(-1)).min(axis=1)
    return 1000 * d.mean()


def _scene(mesh, poses):
    """The pyrender-mode depth of the objects at `poses` and their label image (object k is k + 1), nearest surface per pixel."""
    D, S = np.zeros(HW, np.uint16), np.zeros(HW, np.uint8)
    for k, P in enumerate(poses):
        d = init_ref.full_depth(P, K, mesh, *HW)
        win = (d > 0) & ((D == 0) | (d < D))
        D, S = np.where(win, d, D), np.where(win, np.uint8(k + 1), S)
    return D, S


@pytest.fixture(scope='module')
def jump(synth):
    """Two objects, both wholly inside the frame; object 1 jumps to a new pose at frame JUMP_AT.  -> (mesh, gts before, gts after,
    frames [(depth, seg)])."""
    mesh, gts, _, _, _ = init_ref.labelled_scene(synth, 2, seed=0)
    gts[0, :3, 3], gts[1, :3, 3] = (-0.12, 0.08, 0.8), (0.0, -0.08, 0.82)
    moved = gts.copy()
    turn = init_ref.icp_ref.exp_so3(np.array([0.3, 0.8, 0.52]) / np.linalg.norm([0.3, 0.8, 0.52]) * np.radians(50))
    moved[1, :3, :3] = turn @ gts[1, :3, :3]
    moved[1, :3, 3] = (0.14, 0.04, 0.86)
    return mesh, gts, moved, [_scene(mesh, gts)] * JUMP_AT + [_scene(mesh, moved)] * (FRAMES - JUMP_AT)


JUMP_AT, FRAMES, AFTER = 2, 5, 2


@pytest.mark.parametrize('route', ['host', 'device'])
def test_tracker_restarts_the_object_that_jumped(pkg, synth, jump, route, tmp_path):
    mesh, gts, moved, frames = jump
    trk = _zero_head_tracker(pkg, synth, tmp_path, dict(below=0.5, after=AFTER))
    plain = _zero_head_tracker(pkg, synth, tmp_path, None)
    assert trk.engine.max_batch == 2 * 8 and trk.fit == importlib.import_module(PKG + '.predict').FIT_TAU_DEFAULT
    rgb = np.zeros(HW + (3,), np.uint8)
    as_in = (lambda a: a) if route == 'host' else (lambda a: _dev(trk.engine, a))
    poses, poses_plain = gts.copy(), gts.copy()
    events = []
    for f, (D, S) in enumerate(frames):
        out = trk.on_track_batch(as_in(poses), rgb, D, seg=S, labels=[1, 2])
        poses = out if route == 'host' else out.cpu().numpy()
        ev = trk.last_reinit if route == 'host' else trk.last_reinit.cpu().numpy()
        events.append(list(ev))
        poses_plain = plain.on_track_batch(poses_plain, rgb, D)
        assert np.array_equal(poses[0], poses_plain[0])       # the other object keeps the bits of a Tracker without reinit
        if f == JUMP_AT + AFTER - 1:
            e = trk.engine
            ow = torch.full((1,), WIDTH, dtype=torch.float64, device=e.device)
            start, _ = e.init_poses(_dev(e, D), _dev(e, S), K, [2], ow)
            assert np.array_equal(poses[1], start[0].cpu().numpy())     # the lone init call's start, bit for bit
        if f < JUMP_AT + AFTER - 1:
            assert np.array_equal(poses[1], gts[1])
    assert events[:JUMP_AT] == [[0, 0]] * JUMP_AT
    assert events[JUMP_AT:JUMP_AT + AFTER] == [[0, 1]] * (AFTER - 1) + [[0, R.RESTARTED]]
    adds = _adds_mm(mesh, poses[1], moved[1])
    print('restarted object ADD-S %.3f mm' % adds)
    assert adds < ADDS_BOUND_MM
    trk.reset_reinit()
    assert trk._streak is None


def test_tracker_without_a_mask_does_not_restart(pkg, synth, jump, tmp_path):
    _, gts, _, frames = jump
    trk = _zero_head_tracker(pkg, synth, tmp_path, dict(below=0.5, after=1))
    rgb = np.zeros(HW + (3,), np.uint8)
    D, _ = frames[-1]
    out = trk.on_track_batch(gts.copy(), rgb, D)
    assert list(trk.last_reinit) == [0, 1] and np.array_equal(out, gts)
    pose = trk.on_track(gts[1], rgb, D)                       # one track: a new n starts the streaks again
    assert list(trk.last_reinit) == [1] and np.array_equal(pose, gts[1])


def test_tracker_refuses_masks_and_engines_it_cannot_use(pkg, synth, jump, tmp_path):
    _, gts, _, frames = jump
    trk = _zero_head_tracker(pkg, synth, tmp_path, dict(below=0.5, after=1))
    rgb = np.zeros(HW + (3,), np.uint8)
    D, S = frames[-1]
    with pytest.raises(ValueError, match='bool mask or a uint8 label image'):
        trk.on_track(gts[1], rgb, D, mask=S.astype(np.int64) * 300, label=2)
    with pytest.raises(ValueError, match='uint8 label image'):
        trk.on_track_batch(gts.copy(), rgb, D, seg=S.astype(np.int32), labels=[1, 2])
    pose = trk.on_track(gts[1], rgb, D, mask=S == 2)              # a bool mask: the object's pixels under label 1
    assert trk.last_reinit[0] == R.RESTARTED and np.isfinite(pose).all()
    pose = trk.on_track(gts[1], rgb, D, mask=S, label=2)          # a uint8 label image, then its int32 copy: the same restart
    assert trk.last_reinit[0] == R.RESTARTED
    assert np.array_equal(trk.on_track(gts[1], rgb, D, mask=S.astype(np.int32), label=2), pose) and trk.last_reinit[0] == R.RESTARTED
    # a shared Engine must hold n x init keep tracks: refused before the step, so the streaks do not move
    small = pkg.Engine(max_batch=8)
    try:
        with pytest.raises(ValueError, match='max_batch'):
            _zero_head_tracker_on(pkg, synth, tmp_path, small, dict(below=0.5, after=1, init={'keep': 9}))
        t2 = _zero_head_tracker_on(pkg, synth, tmp_path, small, dict(below=0.5, after=1))
        with pytest.raises(ValueError, match='exceed the engine'):
            t2.on_track_batch(gts.copy(), rgb, D, seg=S, labels=[1, 2])
        assert t2._streak is None
    finally:
        small.close()


def _zero_head_tracker_on(pkg, synth, tmp_path, engine, reinit):
    path = str(tmp_path / 'model.ply')
    importlib.import_module(PKG + '.mesh_io').save_ply_mesh(path, synth.mesh())
    info = {'resolution': 176, 'boundingbox': 10, 'object_width': WIDTH,
            'camera': {'focalX': K[0, 0], 'focalY': K[1, 1], 'centerX': K[0, 2], 'centerY': K[1, 2], 'height': HW[0], 'width': HW[1]}}
    mean, std = synth.default_mean_std()
    return pkg.Tracker(info, mean, std, {'state_dict': synth.make_state_dict(2)}, model_path=path, renderer='cuda', engine=engine,
                       reinit=reinit)
