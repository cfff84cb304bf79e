"""The depth refinement of a tracking step (se3tn_track_opts.icp, Engine.track_render(icp=), Tracker(icp=)): ICP off is
se3tn_track_render bit for bit; every iteration's pose equals oracle/icp_ref.py's from the same start and the inlier counts are
exact; with a zero head, ICP alone carries perturbed starts back to the poses that drew a synthetic frame; degenerate tracks
keep their poses; graph replay, launch counts and refusals follow include/se3tn.h; the Tracker's two routes agree."""
import ctypes as C
import importlib
import os
import sys
import numpy as np
import pytest
import torch
from test_icp_cpu import ADD_BOUND_MM, ROT_BOUND_DEG, errors, synthetic_scene

pytestmark = pytest.mark.gpu
PKG = 'iros20-6d-pose-tracking_b200'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import icp_ref  # noqa: E402

TN, RN = 0.03, 5 * np.pi / 180
HW = (480, 640)
NET, ZERO = 0, 9                                # a random network and one whose head outputs 0 (the pose update is the identity)
K = importlib.import_module(PKG + '.synth').CAMERA_K
WIDTH = 200.0


@pytest.fixture(scope='module')
def eng(pkg, synth):
    e = pkg.Engine(max_batch=64)
    mean, std = synth.default_mean_std()
    zero = synth.make_state_dict(2)
    for k in ('trans_out.0.weight', 'trans_out.0.bias', 'rot_out.0.weight', 'rot_out.0.bias'):
        zero[k] = torch.zeros_like(zero[k])
    for wid, sd in ((NET, synth.make_state_dict(0)), (ZERO, zero)):
        e.load_state_dict(sd, wid)
        e.set_mesh(synth.mesh(), wid)
        e.set_stats(mean, std, wid)
    yield e
    e.close()


@pytest.fixture(scope='module', autouse=True)
def keep_utils_engine():
    U = importlib.import_module(PKG + '.Utils')
    saved = U._engine
    yield
    U.set_engine(saved)


@pytest.fixture(scope='module')
def scene(synth):
    mesh, gts, starts, D = synthetic_scene(synth, 8, seed=0)
    return dict(mesh=mesh, gts=gts, starts=starts, D=D, rgb=synth.raw_frame(3)[0])


def _dev(e, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(e.device)


class Case:
    """n tracks of the scene (the 8 starts repeated), ids alternating NET / ZERO unless all `ids`."""
    def __init__(self, e, sc, n, ids=None, depth=None):
        self.n = n
        self.poses = np.ascontiguousarray(np.concatenate([sc['starts']] * ((n + 7) // 8))[:n])
        self.rgb, self.depth = sc['rgb'], sc['D'] if depth is None else depth
        self.R, self.D, self.P = _dev(e, self.rgb), _dev(e, self.depth), _dev(e, self.poses)
        self.ow = torch.full((n,), WIDTH, dtype=torch.float64, device=e.device)
        self.wid = np.array([NET if (ids is None and i % 2 == 0) else (ids if ids is not None else ZERO) for i in range(n)], np.int32)
        self.wd = _dev(e, self.wid)


def _nan(e, *shape, dtype=torch.float64):
    return torch.full(shape, float('nan'), dtype=dtype, device=e.device)


def _step(e, c, icp, prec='bf16x3', mode='vispy', fill=None, k=1, **kw):
    outs = dict(out_poses=_nan(e, c.n, 4, 4), out_trans=_nan(e, c.n, 3, dtype=torch.float32), out_rot=_nan(e, c.n, 3, dtype=torch.float32))
    outs.update(kw)
    return e.track_render(c.R, c.D, K, c.P, c.ow, TN, RN, weight_ids_host=c.wid, weight_ids_dev=c.wd, precision=prec, mode=mode,
                          image_hw=HW if mode == 'pyrender' else None, fill_depth=fill, iterations=k, icp=icp, **outs)


def _raw_icp(e, c, out, opts=None, rounds=None, icp=None, icp_poses=None, out_icp=None):
    """se3tn_track_render with opts->icp = icp (None: NULL) and the step's arrays."""
    L = importlib.import_module(PKG + '._lib')
    Kh = np.ascontiguousarray([K[0, 0], K[1, 1], K[0, 2], K[1, 2]])
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    if opts is not None:
        opts.icp = None if icp is None else C.pointer(icp)
    arrays = L.TrackArrays(*(None if t is None else t.data_ptr() for t in (None, rounds, None, icp_poses, None, None, out_icp)))
    return e.lib.se3tn_track_render(e._ctx, p(c.R), p(c.D), HW[0], HW[1], Kh.ctypes.data_as(C.c_void_p), p(c.P), p(c.ow), 0, 0, 0,
                                    c.wid.ctypes.data_as(C.c_void_p), p(c.wd), c.n, TN, RN, L.PREC_BF16X3, p(out[1]), p(out[2]),
                                    p(out[0]), None if opts is None else C.byref(opts), C.byref(arrays),
                                    C.c_void_p(torch.cuda.current_stream().cuda_stream))


def test_icp_off_is_track_render(eng, scene):
    L = importlib.import_module(PKG + '._lib')
    c = Case(eng, scene, 5)
    res = []
    for explicit in (False, True):                   # opts without the pointer fields set, then opts->icp = NULL
        out = (_nan(eng, 5, 4, 4), _nan(eng, 5, 3, dtype=torch.float32), _nan(eng, 5, 3, dtype=torch.float32))
        rounds = _nan(eng, 2, 5, 4, 4)
        opts = L.TrackOpts(iterations=2, fit_tau_mm=15)
        if explicit:
            assert _raw_icp(eng, c, out, opts, rounds, icp=None) == L.OK and not opts.icp
        else:
            arrays = L.TrackArrays(round_poses=rounds.data_ptr())
            p = lambda t: C.c_void_p(t.data_ptr())
            Kh = np.ascontiguousarray([K[0, 0], K[1, 1], K[0, 2], K[1, 2]])
            assert eng.lib.se3tn_track_render(eng._ctx, p(c.R), p(c.D), HW[0], HW[1], Kh.ctypes.data_as(C.c_void_p), p(c.P), p(c.ow),
                                              0, 0, 0, c.wid.ctypes.data_as(C.c_void_p), p(c.wd), c.n, TN, RN, L.PREC_BF16X3,
                                              p(out[1]), p(out[2]), p(out[0]), C.byref(opts), C.byref(arrays),
                                              C.c_void_p(torch.cuda.current_stream().cuda_stream)) == L.OK
        torch.cuda.synchronize()
        res.append((out, rounds, eng._fit_rows_view()[:5].clone(), eng.last_launch_count(), eng.last_step_was_graph()))
    (a, ra, fa, na, ga), (b, rb, fb, nb, gb) = res
    assert all(torch.equal(x, y) for x, y in zip(a, b)) and torch.equal(ra, rb) and torch.equal(fa, fb)
    assert na == nb and ga and gb


@pytest.mark.parametrize('mode', ['vispy', 'pyrender'])
@pytest.mark.parametrize('fill', [False, True], ids=['raw', 'fill'])
@pytest.mark.parametrize('prec', ['bf16x3', 'fp32'])
def test_iterations_equal_the_oracle(eng, scene, prec, fill, mode):
    M = 2
    for n in ((1, 8, 64) if mode == 'vispy' else (1, 8)):       # the pyrender oracle rasterises the whole frame per track
        c = Case(eng, scene, n)
        rounds, slots = _nan(eng, 1, n, 4, 4), _nan(eng, M, n, 4, 4)
        P, _, _, stats = _step(eng, c, {'iterations': M, 'tau_mm': 20, 'min_inliers': 100}, prec, mode=mode, fill=fill or None,
                               out_rounds=rounds, out_icp_poses=slots)
        depth = eng.fill_depth(c.D) if fill else c.D
        torch.cuda.synchronize()
        depth, pre, slots, stats = depth.cpu().numpy(), rounds[0].cpu().numpy(), slots.cpu().numpy(), stats.cpu().numpy()
        assert np.array_equal(slots[-1], P.cpu().numpy())
        moved = 0
        for i in range(n):
            start = pre[i]
            for m in range(M):
                want, st, terms = icp_ref.iterate(start, K, WIDTH, scene['mesh'], depth, 20, 100, mode, *HW)
                got = slots[m, i]
                if want is start:                                     # a skipped update keeps the pose bit for bit
                    assert np.array_equal(got, start), (n, i, m)
                else:
                    moved += 1
                    assert np.abs(got[:3, 3] - want[:3, 3]).max() <= 1e-9, (n, i, m)
                    assert np.abs(got[:3, :3] - want[:3, :3]).max() <= 1e-9, (n, i, m)
                if m == M - 1:
                    assert stats[i, 0] == st[0] == len(terms['e']), (n, i)
                start = got
        assert moved > 0


@pytest.mark.parametrize('mode', ['vispy', 'pyrender'])
def test_iterations_equal_the_oracle_on_a_dense_model(pkg, synth, scene, mode):
    """test_iterations_equal_the_oracle's check with a level-6 model (81,920 faces): the triangle ids ICP reads come from
    sub-pixel triangles, many per pixel, so they test the rasteriser's choice among them.  2 tracks, 2 iterations."""
    M, n, DENSE = 2, 2, 5
    mesh = synth.mesh(6, seed=6)
    e = pkg.Engine(max_batch=8)
    try:
        mean, std = synth.default_mean_std()
        e.load_state_dict(synth.make_state_dict(0), DENSE); e.set_stats(mean, std, DENSE); e.set_mesh(mesh, DENSE)
        c = Case(e, scene, n, ids=DENSE)
        rounds, slots = _nan(e, 1, n, 4, 4), _nan(e, M, n, 4, 4)
        P, _, _, stats = _step(e, c, {'iterations': M, 'tau_mm': 20, 'min_inliers': 100}, mode=mode, out_rounds=rounds, out_icp_poses=slots)
        torch.cuda.synchronize()
        pre, slots, stats, P = rounds[0].cpu().numpy(), slots.cpu().numpy(), stats.cpu().numpy(), P.cpu().numpy()
    finally:
        e.close()
    assert np.array_equal(slots[-1], P)
    moved = 0
    for i in range(n):
        start = pre[i]
        for m in range(M):
            want, st, terms = icp_ref.iterate(start, K, WIDTH, mesh, scene['D'], 20, 100, mode, *HW)
            got = slots[m, i]
            if want is start:
                assert np.array_equal(got, start), (i, m)
            else:
                moved += 1
                assert np.abs(got[:3, 3] - want[:3, 3]).max() <= 1e-9, (i, m)
                assert np.abs(got[:3, :3] - want[:3, :3]).max() <= 1e-9, (i, m)
            if m == M - 1:
                assert stats[i, 0] == st[0] == len(terms['e']), i
            start = got
    assert moved > 0


@pytest.mark.parametrize('n', [1, 8])
def test_zero_head_converges(synth, eng, scene, n):
    c = Case(eng, scene, n, ids=ZERO)
    first = _step(eng, c, 1, mode='pyrender')[3].cpu().numpy()
    P, _, _, stats = _step(eng, c, 10, mode='pyrender')
    P, stats = P.cpu().numpy(), stats.cpu().numpy()
    for i in range(n):
        add, rot = errors(synth, P[i], scene['gts'][i])
        assert add <= ADD_BOUND_MM and rot <= ROT_BOUND_DEG, (i, add, rot)
        assert stats[i, 2] < first[i, 2] and stats[i, 3] < first[i, 3], (i, first[i], stats[i])
        assert stats[i, 0] >= 100


def test_degenerate_tracks_keep_their_poses(eng, scene):
    c = Case(eng, scene, 8, ids=ZERO)
    plain = _step(eng, c, None)[0]
    for depth, icp in ((np.zeros_like(scene['D']), 3), (scene['D'], {'iterations': 3, 'min_inliers': 176 * 176})):
        z = Case(eng, scene, 8, ids=ZERO, depth=depth)
        P, _, _, stats = _step(eng, z, icp)
        assert torch.equal(P, plain)
        assert (stats[:, 2:] == 0).all()
        if not depth.any():
            assert (stats[:, 0] == 0).all()
    off = Case(eng, scene, 8, ids=ZERO)
    off.poses[3, :3, 3] = (2.0, 0.0, 0.5)                                 # its window lies wholly outside the frame
    off.P = _dev(eng, off.poses)
    plain = _step(eng, off, None)[0]
    P, _, _, stats = _step(eng, off, 3)
    assert torch.equal(P[3], plain[3]) and stats[3].tolist() == [0, 0, 0, 0]
    assert stats[0, 2] > 0                                               # the others move


def test_graph_replay_and_launch_count(eng, scene):
    c = Case(eng, scene, 8)
    outs = dict(out_poses=_nan(eng, 8, 4, 4), out_trans=_nan(eng, 8, 3, dtype=torch.float32), out_rot=_nan(eng, 8, 3, dtype=torch.float32),
                out_icp_poses=_nan(eng, 3, 8, 4, 4))
    _step(eng, c, None, **{k: v for k, v in outs.items() if k != 'out_icp_poses'})
    plain = eng.last_launch_count()
    frames = [scene['D'], np.where(scene['D'] > 0, scene['D'] + 4, 0).astype(np.uint16)]
    seen = []
    for rep in range(2):
        for f in frames:
            c.D.copy_(_dev(eng, f))
            P, _, _, stats = _step(eng, c, 3, **outs)
            assert eng.last_step_was_graph() and eng.last_launch_count() == plain + 4 * 3
            seen.append((P.clone(), stats.clone(), outs['out_icp_poses'].clone()))
    assert not torch.equal(seen[0][0], seen[1][0])                       # a fresh result for each frame
    for a, b in zip(seen[:2], seen[2:]):
        assert all(torch.equal(x, y) for x, y in zip(a, b))
    c.D.copy_(_dev(eng, frames[0]))
    P, _, _, stats = _step(eng, c, 3, prec='fp32', **outs)
    assert not eng.last_step_was_graph() and eng.last_launch_count() > 12


def test_refusals(eng, scene):
    L = importlib.import_module(PKG + '._lib')
    c = Case(eng, scene, 4)
    refused = lambda rc, field: rc == L.ERR_INVALID and field in eng.lib.se3tn_last_error(eng._ctx).decode()
    opts = L.TrackOpts(iterations=2)
    good = dict(iterations=2, tau_mm=20, min_inliers=100, reserved=0)
    hp = lambda a: a.ctypes.data_as(C.c_void_p)
    Kh = np.ascontiguousarray([K[0, 0], K[1, 1], K[0, 2], K[1, 2]])
    for field, bad in (('iterations', 0), ('iterations', 17), ('tau_mm', 0), ('tau_mm', 1001), ('min_inliers', 5),
                       ('min_inliers', 176 * 176 + 1), ('reserved', 1)):
        out = (_nan(eng, 4, 4, 4), _nan(eng, 4, 3, dtype=torch.float32), _nan(eng, 4, 3, dtype=torch.float32))
        slots, st = _nan(eng, 2, 4, 4, 4), _nan(eng, 4, 4)
        icp = L.IcpOpts(**dict(good, **{field: bad}))
        assert refused(_raw_icp(eng, c, out, opts, None, icp, slots, st), 'icp->' + field), (field, bad)
        host_poses, host_icp = np.full((4, 4, 4), np.nan), np.full((4, 4), np.nan)
        opts.icp = C.pointer(icp)
        rc = eng.lib.se3tn_track_render_host(eng._ctx, hp(c.rgb), hp(c.depth), HW[0], HW[1], hp(Kh), hp(c.poses),
                                             hp(np.full(4, WIDTH)), 0, 0, 0, hp(c.wid), 4, TN, RN, L.PREC_BF16X3, hp(host_poses), None,
                                             None, C.byref(opts), C.byref(L.TrackArrays(out_icp=host_icp.ctypes.data)), None)
        assert refused(rc, 'icp->' + field)
        torch.cuda.synchronize()
        assert all(torch.isnan(t).all() for t in out + (slots, st)) and np.isnan(host_poses).all() and np.isnan(host_icp).all()
    icp = L.IcpOpts(**good)
    rounds = _nan(eng, 2, 4, 4, 4)
    big = _nan(eng, 8, 4, 4, 4)                      # big[0] is poses_out
    out = (big[0], _nan(eng, 4, 3, dtype=torch.float32), _nan(eng, 4, 3, dtype=torch.float32))
    for slots, st in ((big[0:2], None),              # icp_poses over poses_out
                      (rounds, None),                # icp_poses over round_poses
                      (big[2:4], big[3, 0]),         # out_icp inside icp_poses
                      (None, rounds[0, 0])):         # out_icp over round_poses
        assert refused(_raw_icp(eng, c, out, opts, rounds, icp, slots, st), 'icp_poses and out_icp must not overlap')
        torch.cuda.synchronize()
        assert torch.isnan(big).all() and torch.isnan(rounds).all()
    assert _raw_icp(eng, c, out, opts, rounds, icp, big[1:3], big[3, 0]) == L.OK     # clear of everything: runs
    torch.cuda.synchronize()
    assert torch.isfinite(big[:3]).all() and torch.isfinite(big[3, 0]).all()


def test_tracker_routes_agree(pkg, synth, eng, scene, tmp_path):
    mio = importlib.import_module(PKG + '.mesh_io')
    path = str(tmp_path / 'model.ply')
    mio.save_ply_mesh(path, scene['mesh'])
    info = {'resolution': 176, 'object_width': WIDTH, 'boundingbox': 10,
            'camera': {'focalX': K[0, 0], 'focalY': K[1, 1], 'centerX': K[0, 2], 'centerY': K[1, 2], 'height': 480, 'width': 640}}
    mean, std = synth.default_mean_std()
    zero = synth.make_state_dict(2)                                   # a zero head: ICP alone moves the tracks
    for k in ('trans_out.0.weight', 'trans_out.0.bias', 'rot_out.0.weight', 'rot_out.0.bias'):
        zero[k] = torch.zeros_like(zero[k])
    make = lambda **kw: pkg.Tracker(info, mean, std, {'state_dict': zero}, model_path=path, renderer='cuda', max_batch=8, **kw)
    with pytest.raises(ValueError, match='hypotheses'):
        make(icp=2, hypotheses=2)
    t = make(icp=3, fit=10)
    poses = np.ascontiguousarray(scene['starts'][:4])
    rgbA, depthA = np.zeros((4, 176, 176, 3), np.uint8), np.zeros((4, 176, 176), np.uint16)
    with pytest.raises(ValueError, match='icp=3 draws every model'):       # input A passed in: ICP cannot redraw the models
        t.on_track_batch(poses, scene['rgb'], scene['D'], rgbA, depthA)
    with pytest.raises(ValueError, match='icp=3 draws every model'):
        t.on_track(poses[0], scene['rgb'], scene['D'], rgbA=rgbA[0], depthA=depthA[0])
    host = t.on_track_batch(poses, scene['rgb'], scene['D'])
    host_icp, host_fit = t.last_icp, t.last_fit
    dev = t.on_track_batch(_dev(t.engine, poses), _dev(t.engine, scene['rgb']), _dev(t.engine, scene['D']))
    torch.cuda.synchronize()
    assert isinstance(host, np.ndarray) and np.array_equal(host, dev.cpu().numpy())
    assert np.array_equal(host_icp, t.last_icp.cpu().numpy()) and np.array_equal(host_fit, t.last_fit.cpu().numpy())
    assert host_icp.shape == (4, 4) and (host_icp[:, 0] > 0).all()
    plain = make()
    assert not np.array_equal(plain.on_track_batch(poses, scene['rgb'], scene['D']), host) and plain.last_icp is None
    one = t.on_track(poses[0], scene['rgb'], scene['D'])
    assert one.shape == (4, 4) and np.isfinite(one).all() and t.last_icp.shape == (1, 4)
