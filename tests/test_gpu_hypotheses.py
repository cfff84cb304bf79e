"""Multi-hypothesis tracking on the device (se3tn_track_opts.hyp, se3tn_draw_hypotheses, Engine.track_hypotheses,
Tracker(hypotheses=)): the starts equal oracle/hypotheses_ref.py, every hypothesis is a plain track_render step over the expanded
starts bit for bit, the choice follows the fit rule, S = 1 is the plain step, a zero head recovers the hypothesis the frame shows,
one graph replays with fresh keys, and the refusals queue nothing."""
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
import hypotheses_ref as HR  # noqa: E402

TN, RN = 0.03, 5 * np.pi / 180
HW = (480, 640)
SETS = (0, 5)
ZERO = 9                                        # a weight set whose head outputs 0: the pose update is the identity
K = importlib.import_module(PKG + '.synth').CAMERA_K
TAU = 15
FIT_TAU = importlib.import_module(PKG + '.predict').FIT_TAU_DEFAULT
MAXB = 64
SPREAD = dict(max_translation=0.02, max_rotation_deg=15.0)


@pytest.fixture(scope='module')
def eng(pkg, synth):
    e = pkg.Engine(max_batch=MAXB)
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


def _addr(t):
    return None if t is None else (t.data_ptr() if torch.is_tensor(t) else t.ctypes.data)


def _raw_render(e, c, opts, arrays, poses_out, P=None, n=None, trans=None):
    """se3tn_track_render on Case c's device frame and tracks with these options and arrays (a TrackArrays, or a raw address),
    past Engine's own checks."""
    E = importlib.import_module(PKG + '.engine')
    n = c.n if n is None else n
    trans = torch.empty(n, 3, device=e.device) if trans is None else trans
    return e.lib.se3tn_track_render(
        e._ctx, E._ptr(c.R), E._ptr(c.D), HW[0], HW[1], E._hptr(E.Engine._k4(K)), E._ptr(c.P if P is None else P), E._ptr(c.ow),
        0, 0, 0, E._hptr(c.wid), E._ptr(c.wd), n, TN, RN, 2, E._ptr(trans), E._ptr(trans.clone()), E._ptr(poses_out),
        C.byref(opts), arrays if isinstance(arrays, C.c_void_p) else C.byref(arrays), E._stream(e.device))


def _raw_render_host(e, c, opts, arrays, poses_out):
    """se3tn_track_render_host on Case c's host frame and tracks with these options and arrays."""
    E = importlib.import_module(PKG + '.engine')
    return e.lib.se3tn_track_render_host(
        e._ctx, E._hptr(c.rgb), E._hptr(c.depth), HW[0], HW[1], E._hptr(E.Engine._k4(K)), E._hptr(c.poses),
        E._hptr(np.full(c.n, 200.0)), 0, 0, 0, E._hptr(c.wid), c.n, TN, RN, 2, E._hptr(poses_out), None, None, C.byref(opts),
        C.byref(arrays), E._stream(e.device))


class Case:
    def __init__(self, e, synth, n, seed):
        self.n = n
        self.rgb, self.depth = synth.raw_frame(seed)
        self.poses = synth.raw_poses(n, seed=seed)
        self.R, self.D, self.P = _dev(e, self.rgb), _dev(e, self.depth), _dev(e, self.poses)
        self.ow = torch.full((n,), 200.0, dtype=torch.float64, device=e.device)
        self.wid = None if n == 1 else np.array([SETS[i % 2] for i in range(n)], dtype=np.int32)
        self.wd = None if self.wid is None else _dev(e, self.wid)
        self.keys = torch.arange(n, dtype=torch.int64, device=e.device) * 7919 + (seed << 40)


def _hyp(e, c, S, k, prec, mode, seed=1, **kw):
    return e.track_hypotheses(c.R, c.D, K, c.P, c.ow, TN, RN, c.keys, S, seed=seed, fit=TAU, weight_ids_host=c.wid,
                              weight_ids_dev=c.wd, precision=prec, mode=mode, image_hw=HW if mode == 'pyrender' else None,
                              iterations=k, **SPREAD, **kw)


def _plain(e, c, starts, S, k, prec, mode):
    """track_render over the n x S expanded starts, ids and widths repeated track-major -> (poses, rows, rounds)."""
    n = c.n
    P = starts.reshape(n * S, 4, 4).contiguous()
    wid = None if c.wid is None else np.repeat(c.wid, S)
    rounds = torch.empty(k, n * S, 4, 4, dtype=torch.float64, device=e.device)
    out = e.track_render(c.R, c.D, K, P, c.ow.repeat_interleave(S), TN, RN, weight_ids_host=wid,
                         weight_ids_dev=None if wid is None else _dev(e, wid), precision=prec, mode=mode,
                         image_hw=HW if mode == 'pyrender' else None, iterations=k, fit=TAU, out_rounds=rounds)
    return out[0], out[3], rounds


@pytest.mark.parametrize('mode', ['vispy', 'pyrender'])
@pytest.mark.parametrize('prec', ['bf16x3', 'fp8', 'fp32'])
def test_one_hypothesis_is_the_plain_step(synth, eng, prec, mode):
    for n in (1, 3, 16):
        c = Case(eng, synth, n, seed=n)
        for k in (1, 3):
            rounds = torch.empty(k, n, 1, 4, 4, dtype=torch.float64, device=eng.device)
            P, choice, rows, R = _hyp(eng, c, 1, k, prec, mode, out_rounds=rounds)
            want_P, want_rows, want_R = _plain(eng, c, c.P[:, None], 1, k, prec, mode)
            assert torch.equal(P, want_P) and torch.equal(rows, want_rows) and torch.equal(R.reshape(k, n, 4, 4), want_R), (n, k)
            assert not choice.any()


def test_expansion_equals_the_oracle(synth, eng):
    n, S, seed = 2, 32, 2 ** 63 + 12345
    c = Case(eng, synth, n, seed=11)
    starts, draws = eng.draw_hypotheses(c.P, c.keys, S, seed=seed, want_draws=True, **SPREAD)
    want, wd = HR.expand(c.poses, c.keys.cpu().numpy(), S, seed, SPREAD['max_translation'], SPREAD['max_rotation_deg'])
    got, gd = starts.cpu().numpy(), draws.cpu().numpy()
    assert np.array_equal(got[:, 0], c.poses) and not gd[:, 0].any()
    assert np.array_equal(gd[..., :4], wd[..., :4]) and np.array_equal(gd[..., 6:], wd[..., 6:])     # uniforms, tries
    # CUDA's log / sqrt / sincospi against libm's: a few ulps of the normal, so a few ulps of max near m = 0 as well
    for col, top in ((4, SPREAD['max_translation']), (5, SPREAD['max_rotation_deg'])):
        assert np.abs(gd[..., col] - wd[..., col]).max() <= 1e-14 * top
    assert np.abs(got - want).max() < 1e-12
    # the draws depend on (seed, key, h) alone: a subset of the tracks, another order, S, n
    sub = eng.draw_hypotheses(c.P[[1, 0]].contiguous(), c.keys[[1, 0]].contiguous(), 4, seed=seed, **SPREAD)
    assert torch.equal(sub, starts[[1, 0], :4])
    other = eng.draw_hypotheses(c.P, c.keys, S, seed=seed + 1, **SPREAD)
    assert not torch.equal(other[:, 1:], starts[:, 1:]) and torch.equal(other[:, 0], starts[:, 0])


@pytest.mark.parametrize('mode', ['vispy', 'pyrender'])
@pytest.mark.parametrize('prec', ['bf16x3', 'fp8', 'fp32'])
def test_every_hypothesis_is_a_plain_step_and_the_fit_chooses(synth, eng, prec, mode):
    for n, S in ((1, 4), (3, 4), (16, 4)):                        # 16 x 4 = max_batch
        c = Case(eng, synth, n, seed=30 + n)
        starts = eng.draw_hypotheses(c.P, c.keys, S, seed=1, **SPREAD)
        for k in (1, 3):
            hp = torch.empty(n, S, 4, 4, dtype=torch.float64, device=eng.device)
            rounds = torch.empty(k, n, S, 4, 4, dtype=torch.float64, device=eng.device)
            P, choice, rows, H, R = _hyp(eng, c, S, k, prec, mode, out_hyp_poses=hp, out_rounds=rounds)
            all_rows = eng._fit_rows_view()[:n * S].clone()
            want_P, want_rows, want_R = _plain(eng, c, starts, S, k, prec, mode)
            assert torch.equal(H.reshape(n * S, 4, 4), want_P) and torch.equal(R.reshape(k, n * S, 4, 4), want_R), (n, k)
            assert torch.equal(all_rows, want_rows), (n, k)
            ch = choice.cpu().numpy()
            assert np.array_equal(ch, HR.choose(want_rows.cpu().numpy().reshape(n, S, 6))), (n, k)
            idx = torch.arange(n, device=eng.device) * S + choice.long()
            assert torch.equal(P, want_P[idx]) and torch.equal(rows, want_rows[idx])
            if n <= 3:                                               # the host route
                hP, hc, hrows = eng.track_hypotheses_host(c.rgb, c.depth, K, c.poses, c.ow.cpu().numpy(), TN, RN, c.keys.cpu().numpy(),
                                                          S, seed=1, fit=TAU, weight_ids=c.wid, precision=prec, mode=mode,
                                                          image_hw=HW if mode == 'pyrender' else None, iterations=k, **SPREAD)
                assert np.array_equal(hP, P.cpu().numpy()) and np.array_equal(hc, ch) and np.array_equal(hrows, rows.cpu().numpy())


def test_a_zero_head_recovers_the_hypothesis_the_frame_shows(synth, eng):
    n, S, hstar = 2, 8, 5
    poses = synth.raw_poses(n, seed=60)
    poses[:, :3, 3] = [(0.02, -0.01, 0.55), (-0.03, 0.02, 0.6)]
    P = _dev(eng, poses)
    ow = torch.full((n,), 200.0, dtype=torch.float64, device=eng.device)
    ids = np.full(n, ZERO, np.int32)
    keys = torch.tensor([101, 202], dtype=torch.int64, device=eng.device)
    starts = eng.draw_hypotheses(P, keys, S, seed=4, **SPREAD)
    frame = np.zeros(HW, np.uint16)
    Hs = starts[:, hstar].contiguous()
    _, R = eng.render(K, Hs, ow, _dev(eng, ids))
    R = R.cpu().numpy()
    bb = eng.compute_bbox(Hs, K, ow).cpu().numpy()
    for i in range(n):                                               # hypothesis h*'s depth where crop_bbox samples its window
        top, left = bb[i, :, 0].min(), bb[i, :, 1].min()
        ch, cw = bb[i, :, 0].max() - top, bb[i, :, 1].max() - left
        assert top >= 0 and left >= 0 and top + ch <= HW[0] and left + cw <= HW[1]
        sx = np.minimum(np.floor(np.arange(176) * (1.0 / (176.0 / cw))).astype(np.int64), cw - 1)
        sy = np.minimum(np.floor(np.arange(176) * (1.0 / (176.0 / ch))).astype(np.int64), ch - 1)
        sub = frame[np.ix_(top + sy, left + sx)]
        frame[np.ix_(top + sy, left + sx)] = np.where(R[i] > 0, R[i], sub)
    rgb = np.zeros(HW + (3,), np.uint8)
    hp = torch.empty(n, S, 4, 4, dtype=torch.float64, device=eng.device)
    out, choice, rows, H = eng.track_hypotheses(_dev(eng, rgb), _dev(eng, frame), K, P, ow, TN, RN, keys, S, seed=4, fit=TAU,
                                                weight_ids_host=ids, out_hyp_poses=hp, **SPREAD)
    all_rows = eng._fit_rows_view()[:n * S].cpu().numpy().reshape(n, S, 6)
    assert torch.equal(H, starts)                                    # the identity update: the rounds leave the starts as drawn
    assert (choice.cpu().numpy() == hstar).all()
    r = rows.cpu().numpy()
    assert (r[:, 2] == r[:, 0]).all() and (r[:, 5] == 0).all() and (r[:, 0] > 1000).all()
    assert (all_rows[:, 0, 2] < r[:, 2]).all()
    assert torch.equal(out, starts[:, hstar])


def test_one_graph_replays_with_fresh_keys(synth, eng):
    n, S, k = 3, 4, 2
    c = Case(eng, synth, n, seed=70)
    outs = dict(out_poses=torch.empty_like(c.P), out_trans=torch.empty(n, 3, device=eng.device), out_rot=torch.empty(n, 3, device=eng.device),
                out_choice=torch.empty(n, dtype=torch.int32, device=eng.device), out_fit=torch.empty(n, 6, dtype=torch.int32, device=eng.device),
                out_hyp_poses=torch.empty(n, S, 4, 4, dtype=torch.float64, device=eng.device))
    seen = []
    for frame in range(3):
        c.keys.copy_(torch.arange(n, device=eng.device) + 1000 * (frame % 2))
        _hyp(eng, c, S, k, 'bf16x3', 'vispy', **outs)
        if frame:
            assert eng.last_step_was_graph()
        seen.append(outs['out_hyp_poses'].clone())
        want = eng.draw_hypotheses(c.P, c.keys, S, seed=1, **SPREAD)
        _plain(eng, c, want, S, k, 'bf16x3', 'vispy')
        plain_launches = eng.last_launch_count()
        _hyp(eng, c, S, k, 'bf16x3', 'vispy', **outs)
        assert eng.last_launch_count() == plain_launches + 2
    assert not torch.equal(seen[0], seen[1]) and torch.equal(seen[0], seen[2])
    # in place: poses_out is poses_in
    P0 = c.P.clone()
    _hyp(eng, c, S, k, 'bf16x3', 'vispy', **dict(outs, out_poses=c.P))
    in_place = c.P.clone()
    c.P.copy_(P0)
    P, *_ = _hyp(eng, c, S, k, 'bf16x3', 'vispy', **outs)
    assert torch.equal(in_place, P)


def test_refusals_queue_nothing(synth, eng, pkg):
    L = importlib.import_module(PKG + '._lib')
    n = 3
    c = Case(eng, synth, n, seed=80)
    outs = dict(out_poses=torch.full_like(c.P, 7.0), out_choice=torch.full((n,), 9, dtype=torch.int32, device=eng.device),
                out_fit=torch.full((n, 6), 9, dtype=torch.int32, device=eng.device))
    snap = {k: v.clone() for k, v in outs.items()}

    def refused(fn, match):
        with pytest.raises(L.Se3tnError, match=match):
            fn()
        torch.cuda.synchronize()
        for key, v in outs.items():
            assert torch.equal(v, snap[key]), key

    def raw(**over):                                     # the C call with one argument changed, past Engine's own checks
        a = dict(S=4, seed=1, max_t=0.02, max_r=15.0, reserved=0, keys=c.keys, tau=TAU, hyp_poses=None, fit=outs['out_fit'],
                 poses_out=outs['out_poses'], n=n, P=c.P)
        a.update(over)
        hyp = L.HypothesisOpts(hypotheses=a['S'], reserved=a['reserved'], seed=a['seed'], max_translation=a['max_t'],
                               max_rotation_deg=a['max_r'])
        arrays = L.TrackArrays(draw_keys=_addr(a['keys']), hyp_poses=_addr(a['hyp_poses']), out_fit=_addr(a['fit']),
                               out_choice=_addr(outs['out_choice']))
        L.check(_raw_render(eng, c, L.TrackOpts(iterations=1, fit_tau_mm=a['tau'], hyp=C.pointer(hyp)), arrays, a['poses_out'],
                            P=a['P'], n=a['n']), eng._ctx)

    refused(lambda: raw(S=0), 'hyp->hypotheses')
    refused(lambda: raw(S=33), 'hyp->hypotheses')
    refused(lambda: raw(reserved=1), 'hyp->reserved')
    refused(lambda: raw(max_t=0.0), 'hyp->max_translation')
    refused(lambda: raw(max_t=float('inf')), 'hyp->max_translation')
    refused(lambda: raw(max_t=1.5), 'hyp->max_translation')
    refused(lambda: raw(max_r=0.0), 'hyp->max_rotation_deg')
    refused(lambda: raw(max_r=200.0), 'hyp->max_rotation_deg')
    refused(lambda: raw(S=32), 'exceeds max_batch')
    refused(lambda: raw(tau=0), 'fit_tau_mm')
    refused(lambda: raw(keys=None), 'draw_keys')
    refused(lambda: raw(fit=outs['out_poses'].view(torch.int32)[:n]), 'overlap')
    refused(lambda: raw(hyp_poses=c.P), 'overlap')
    both = torch.cat([c.P, c.P[:1]])                               # poses_out one track past poses_in in the same buffer
    refused(lambda: raw(P=both[:n], poses_out=both[1:]), 'overlap')
    sd_missing = np.array([0, 5, 77], np.int32)
    with pytest.raises(L.Se3tnError) as e:
        eng.track_hypotheses(c.R, c.D, K, c.P, c.ow, TN, RN, c.keys, 4, fit=TAU, weight_ids_host=sd_missing, **SPREAD, **outs)
    assert e.value.code == L.ERR_STATE
    torch.cuda.synchronize()
    for key, v in outs.items():
        assert torch.equal(v, snap[key]), key


def test_option_and_array_refusals_queue_nothing(synth, eng):
    """ICP inside a hypothesis step, and a se3tn_track_arrays field on a route or in a mode that does not take it (or missing
    where the options need it): SE3TN_ERR_INVALID naming the field, with nothing written to any output."""
    L = importlib.import_module(PKG + '._lib')
    n = 3
    c = Case(eng, synth, n, seed=81)
    dev = dict(poses=torch.full_like(c.P, 7.0), choice=torch.full((n,), 9, dtype=torch.int32, device=eng.device),
               fit=torch.full((n, 6), 9, dtype=torch.int32, device=eng.device), stats=torch.full((n, 4), 9.0, dtype=torch.float64,
               device=eng.device), slots=torch.full((1, n, 4, 4), 9.0, dtype=torch.float64, device=eng.device),
               hyps=torch.full((n, 4, 4, 4), 9.0, dtype=torch.float64, device=eng.device))
    host = dict(poses=np.full((n, 4, 4), 7.0), choice=np.full(n, 9, np.int32), fit=np.full((n, 6), 9, np.int32),
                stats=np.full((n, 4), 9.0), keys=np.arange(n, dtype=np.int64), slots=np.full((1, n, 4, 4), 9.0))
    snap = [v.clone() for v in dev.values()] + [v.copy() for v in host.values()]
    hyp = L.HypothesisOpts(hypotheses=4, seed=1, **SPREAD)
    icp = L.IcpOpts(iterations=1, tau_mm=20, min_inliers=100)
    opts = lambda **kw: L.TrackOpts(iterations=1, fit_tau_mm=TAU, **{k: C.pointer(v) for k, v in kw.items()})
    with_hyp = dict(draw_keys=c.keys, out_fit=dev['fit'], out_choice=dev['choice'])
    host_hyp = dict(draw_keys=host['keys'], out_fit=host['fit'], out_choice=host['choice'])
    arrays = lambda **kw: L.TrackArrays(**{k: _addr(v) for k, v in kw.items()})
    refused = lambda rc, field: rc == L.ERR_INVALID and field in eng.lib.se3tn_last_error(eng._ctx).decode()
    cases = [                                            # (route, options, arrays, the field the error names)
        ('dev', opts(icp=icp, hyp=hyp), arrays(**with_hyp), 'opts->icp and opts->hyp'),
        ('host', opts(icp=icp, hyp=hyp), arrays(**host_hyp), 'opts->icp and opts->hyp'),
        ('dev', opts(hyp=hyp), arrays(**with_hyp, icp_poses=dev['slots']), 'arrays->icp_poses'),
        ('dev', opts(hyp=hyp), arrays(**with_hyp, out_icp=dev['stats']), 'arrays->out_icp'),
        ('dev', opts(hyp=hyp), arrays(draw_keys=c.keys, out_fit=dev['fit']), 'arrays->out_choice'),
        ('dev', opts(hyp=hyp), arrays(draw_keys=c.keys, out_choice=dev['choice']), 'arrays->out_fit'),
        ('dev', opts(), arrays(out_fit=dev['fit']), 'arrays->out_fit'),
        ('dev', opts(), arrays(out_choice=dev['choice']), 'arrays->out_choice'),
        ('dev', opts(), arrays(draw_keys=c.keys), 'arrays->draw_keys'),
        ('dev', opts(), arrays(hyp_poses=dev['hyps']), 'arrays->hyp_poses'),
        ('dev', opts(icp=icp), arrays(out_fit=dev['fit']), 'arrays->out_fit'),
        ('host', opts(hyp=hyp), arrays(**host_hyp, hyp_poses=host['slots']), 'arrays->hyp_poses'),
        ('host', opts(), arrays(out_fit=host['fit'], round_poses=host['slots']), 'arrays->round_poses'),
        ('host', opts(icp=icp), arrays(out_fit=host['fit'], icp_poses=host['slots']), 'arrays->icp_poses'),
        ('host', opts(), arrays(out_fit=host['fit'], out_icp=host['stats']), 'arrays->out_icp'),
        ('host', opts(), arrays(out_fit=host['fit'], out_choice=host['choice']), 'arrays->out_choice'),
        ('host', opts(), arrays(out_fit=host['fit'], draw_keys=host['keys']), 'arrays->draw_keys'),
    ]
    for route, o, a, field in cases:
        rc = _raw_render(eng, c, o, a, dev['poses']) if route == 'dev' else _raw_render_host(eng, c, o, a, host['poses'])
        assert refused(rc, field), (route, field)
    # the struct itself must be host memory: a device address in its place is refused, not read
    assert refused(_raw_render(eng, c, opts(), C.c_void_p(dev['slots'].data_ptr()), dev['poses']), 'arrays points to device memory')
    # input A from the caller: neither batch call takes ICP or hypotheses
    E = importlib.import_module(PKG + '.engine')
    ra = torch.zeros(n, 176, 176, 3, dtype=torch.uint8, device=eng.device)
    da = torch.zeros(n, 176, 176, dtype=torch.uint16, device=eng.device)
    tr = torch.empty(n, 3, device=eng.device)
    for o, field in ((L.TrackOpts(iterations=1, icp=C.pointer(icp)), 'opts->icp'), (L.TrackOpts(iterations=1, hyp=C.pointer(hyp)), 'opts->hyp')):
        rc = eng.lib.se3tn_track_batch(eng._ctx, E._ptr(c.R), E._ptr(c.D), HW[0], HW[1], E._hptr(E.Engine._k4(K)), E._ptr(c.P),
                                       E._ptr(c.ow), E._ptr(ra), E._ptr(da), E._hptr(c.wid), E._ptr(c.wd), n, TN, RN, 2, E._ptr(tr),
                                       E._ptr(tr.clone()), E._ptr(dev['poses']), C.byref(o), E._stream(eng.device))
        assert refused(rc, field)
        rc = eng.lib.se3tn_track_host(eng._ctx, E._hptr(c.rgb), E._hptr(c.depth), HW[0], HW[1], E._hptr(E.Engine._k4(K)),
                                      E._hptr(c.poses), E._hptr(np.full(n, 200.0)), E._hptr(ra.cpu().numpy()), E._hptr(da.cpu().numpy()),
                                      E._hptr(c.wid), n, TN, RN, 2, E._hptr(host['poses']), None, None, C.byref(o), E._stream(eng.device))
        assert refused(rc, field)
    torch.cuda.synchronize()
    for want, got in zip(snap, list(dev.values()) + list(host.values())):
        assert (torch.equal(want, got) if torch.is_tensor(want) else np.array_equal(want, got))


def _tracker(pkg, synth, tmp_path, **kw):
    mio = importlib.import_module(PKG + '.mesh_io')
    path = str(tmp_path / 'model.ply')
    mio.save_ply_mesh(path, synth.mesh(2, seed=4))
    info = {'resolution': 176, 'object_width': 200.0, 'boundingbox': 10, 'max_translation': 0.02, 'max_rotation': 15,
            'camera': {'focalX': K[0, 0], 'focalY': K[1, 1], 'centerX': K[0, 2], 'centerY': K[1, 2], 'height': 480, 'width': 640}}
    mean, std = synth.default_mean_std()
    return pkg.Tracker(info, mean, std, {'state_dict': synth.make_state_dict(0)}, model_path=path, renderer='cuda', max_batch=4, **kw)


def test_tracker(pkg, synth, tmp_path):
    rgb, depth = synth.raw_frame(50)
    poses = synth.raw_poses(3, seed=51)
    plain, one = _tracker(pkg, synth, tmp_path, fit=TAU), _tracker(pkg, synth, tmp_path, fit=TAU, hypotheses=1)
    four = [_tracker(pkg, synth, tmp_path, hypotheses=4, seed=3) for _ in range(2)]
    try:
        assert four[0].engine.max_batch == 16 and four[0].fit == FIT_TAU
        assert np.array_equal(one.on_track_batch(poses, rgb, depth), plain.on_track_batch(poses, rgb, depth))
        assert np.array_equal(one.last_fit, plain.last_fit) and one.last_choice is None
        for frame in range(2):                        # host route, device route: the same keys (seed, call, track)
            host = four[0].on_track_batch(poses, rgb, depth)
            dev = four[1].on_track_batch(torch.from_numpy(poses).cuda(), torch.from_numpy(rgb).cuda(), torch.from_numpy(depth).cuda())
            assert np.array_equal(host, dev.cpu().numpy()), frame
            assert np.array_equal(four[0].last_fit, four[1].last_fit.cpu().numpy())
            assert np.array_equal(four[0].last_choice, four[1].last_choice.cpu().numpy())
            keys = (np.int64(frame) << np.int64(32)) + np.arange(3, dtype=np.int64)
            want, choice, rows = four[0].engine.track_hypotheses_host(
                rgb, depth, K, poses, np.full(3, 200.0), TN, RN, keys, 4, seed=3, fit=FIT_TAU,
                **{'max_translation': 0.02, 'max_rotation_deg': 15})
            assert np.array_equal(host, want) and np.array_equal(four[0].last_choice, choice)
        with pytest.raises(ValueError, match='max_batch'):
            four[0].on_track_batch(synth.raw_poses(5, seed=52), rgb, depth)
    finally:
        for t in [plain, one] + four:
            t.engine.close()
