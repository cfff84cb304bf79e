"""The 'fp8' mode on the H100: every e4m3-written layer checked ALONE against an fp64 conv of its own stored input
(oracle/fp8_ref.py), the calibration against the bf16x3 buffers it reads, and the mode's state rules.

The per-layer check (poisoning, image sampling, the tables `-s` prints) is tests/layer_harness.py's in the fp8 formats of
the buffers: bf16 up to U, e4m3 from CAT to H2.
"""
import numpy as np
import pytest
import torch

import fp8_ref as E
import layer_ref as R
from layer_harness import buffer_bytes, check_poison_outside, poison, run_case, track_inputs

pytestmark = pytest.mark.gpu

TN, RN = 0.03, 5 * np.pi / 180


def _make_engine(pkg, synth, max_batch):
    e = pkg.Engine(max_batch=max_batch)
    e.load_state_dict(synth.make_state_dict(0), 0)
    e.load_state_dict(synth.make_state_dict(1), 1)
    mean, std = synth.default_mean_std()
    e.set_stats(mean, std, 0)
    e.set_stats(mean + 1.5, std * 1.25, 1)
    return e


@pytest.fixture(scope='module')
def eng(pkg, synth):
    e = _make_engine(pkg, synth, 64)
    yield e
    e.close()


@pytest.fixture(scope='module')
def blobs(pkg, synth):
    from importlib import import_module
    pack = import_module(pkg.__name__ + '.weights').pack_state_dict
    return {0: pack(synth.make_state_dict(0)), 1: pack(synth.make_state_dict(1))}


# ------------------------------------------------------------------------------------------- layers
@pytest.mark.parametrize('n', [1, 3, 4, 5, 13, 64])
def test_fp8_forward_layers(synth, eng, blobs, n):
    """Tensor-regime pairs, calibrated on themselves.  n <= 4 is the latency mode's size range, which this mode runs
    without split-K (convAB1 has one e4m3 chunk); 5, 13: ragged unit counts per CTA; 64: the full batch."""
    A, B = synth.tensor_pairs(n, seed=40 + n)
    Ad, Bd = A.to(eng.device), B.to(eng.device)
    eng.calibrate_fp8(Ad, Bd, weight_id=0)
    run_case(eng, 'fp8', 0, n, lambda: eng.forward(Ad, Bd, weight_id=0, precision='fp8', want_feature=True), [0] * n, blobs, 'forward', seed=n)


def test_fp8_forward_many_waves(pkg, synth, blobs):
    """250 images on a 256-image engine; images 250-255 stay poisoned."""
    e = _make_engine(pkg, synth, 256)
    try:
        A, B = synth.tensor_pairs(250, seed=7)
        Ad, Bd = A.to(e.device), B.to(e.device)
        e.calibrate_fp8(Ad, Bd, weight_id=0)
        run_case(e, 'fp8', 0, 250, lambda: e.forward(Ad, Bd, weight_id=0, precision='fp8'), [0] * 250, blobs, 'forward (max_batch 256)')
    finally:
        e.close()


def _calibrate_track_sets(eng, synth, fr, fd, P, ow, A_, dA, wid, wdev):
    """Each set's scales from its own tracks of the frame: input A as given, B cropped at the previous pose."""
    a, b, _, _ = eng.preprocess(fr, fd, synth.CAMERA_K, P, ow, A_, dA, weight_ids=wdev, want_tensors=True)
    for w in (0, 1):
        idx = torch.from_numpy(np.flatnonzero(wid == w)).to(eng.device)
        eng.calibrate_fp8(a[idx], b[idx], weight_id=w)


def test_fp8_track_batch_per_image_weights(synth, eng, blobs):
    """A raw-regime frame, 37 tracks with weight ids 0 / 1: per-set weight maps, biases and fp8 blocks in one step; a
    second call with new poses replays the step's CUDA graph."""
    n = 37
    rgb, depth, poses, rgbA, depthA = track_inputs(synth, n, 5)
    dev = eng.device
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    wid = np.arange(n, dtype=np.int32) % 2
    wdev, P, ow = t(wid), t(poses), t(np.full(n, 200.0))
    fr, fd, A_, dA = t(rgb), t(depth), t(rgbA), t(depthA)
    _calibrate_track_sets(eng, synth, fr, fd, P, ow, A_, dA, wid, wdev)
    out_p = torch.empty_like(P)
    out_t = torch.empty(n, 3, dtype=torch.float32, device=dev); out_r = torch.empty_like(out_t)

    def call():
        eng.track_batch(fr, fd, synth.CAMERA_K, P, ow, A_, dA, TN, RN, weight_ids_host=wid, weight_ids_dev=wdev,
                        precision='fp8', out_poses=out_p, out_trans=out_t, out_rot=out_r)
        return out_t, out_r, None

    run_case(eng, 'fp8', 0, n, call, wid, blobs, 'track_batch, ids 0/1', seed=1)
    P.copy_(t(synth.raw_poses(n, seed=6)))
    run_case(eng, 'fp8', 0, n, call, wid, blobs, 'track_batch graph replay, new poses', seed=2)
    assert eng.last_step_was_graph()


# ------------------------------------------------------------------------------------------- calibration and state
def test_fp8_calibration_is_exact(synth, eng):
    """The scales equal the ones computed from the decoded bf16x3 buffers the calibration's forward left behind."""
    n = 6
    A, B = synth.tensor_pairs(n, seed=3)
    s = eng.calibrate_fp8(A.to(eng.device), B.to(eng.device), weight_id=1)
    torch.cuda.synchronize()
    amax = []
    for buf in ('CAT', 'F1', 'T4', 'F2', 'H1', 'H2'):
        nb = R.image_bytes(buf, 'bf16x3')
        raw = buffer_bytes(eng, buf)[:n * nb].cpu().numpy()
        v = np.stack([R.decode(raw[j * nb:(j + 1) * nb], buf, 'bf16x3').value for j in range(n)])
        if buf in ('H1', 'H2'):
            amax += [np.abs(v[:, :512]).max(), np.abs(v[:, 512:]).max()]
        else:
            amax.append(np.abs(v).max())
    amax = amax[:4] + [amax[4], amax[5], amax[6], amax[7]]
    assert np.array_equal(s, E.calibrate(amax)), (s, E.calibrate(amax))
    assert np.array_equal(eng.fp8_scales(1), s)


def test_fp8_state_rules(pkg, synth, blobs):
    e = _make_engine(pkg, synth, 8)
    L = pkg._lib
    try:
        n = 3
        A, B = synth.tensor_pairs(n, seed=9)
        Ad, Bd = A.to(e.device), B.to(e.device)
        assert e.fp8_scales(0) is None
        # no scales: SE3TN_ERR_STATE naming the id, nothing launched (the poisoned buffers stay)
        poison(e, 'fp8')
        with pytest.raises(L.Se3tnError) as ex:
            e.forward(Ad, Bd, weight_id=0, precision='fp8')
        assert ex.value.code == L.ERR_STATE and 'weight set 0' in str(ex.value)
        rgb, depth, poses, rgbA, depthA = track_inputs(synth, n, 4)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(e.device)
        wid = np.array([1, 0, 1], np.int32)
        e.calibrate_fp8(Ad, Bd, weight_id=1)
        poison(e, 'fp8')
        with pytest.raises(L.Se3tnError) as ex:
            e.track_batch(t(rgb), t(depth), synth.CAMERA_K, t(poses), t(np.full(n, 200.0)), t(rgbA), t(depthA), TN, RN,
                          weight_ids_host=wid, weight_ids_dev=t(wid), precision='fp8')
        assert ex.value.code == L.ERR_STATE and 'weight set 0' in str(ex.value)
        torch.cuda.synchronize()
        check_poison_outside(e, 'fp8', 0, 0)
        # set / get round-trip; invalid scales refused and the old ones kept
        s = np.array([2.0 ** k for k in (-3, 0, 1, 2, -1, 3, 0, 4)], np.float32)
        e.set_fp8_scales(s, 0)
        assert np.array_equal(e.fp8_scales(0), s)
        for bad in (np.nan, np.inf, 0.0, -1.0, 3.0, 2.0 ** -140):
            b = s.copy(); b[5] = bad
            with pytest.raises(L.Se3tnError) as ex:
                e.set_fp8_scales(b, 0)
            assert ex.value.code == L.ERR_INVALID
        assert np.array_equal(e.fp8_scales(0), s)
        # reloading a set's weights drops its scales
        e.load_state_dict(synth.make_state_dict(0), 0)
        assert e.fp8_scales(0) is None and e.fp8_scales(1) is not None
        with pytest.raises(L.Se3tnError) as ex:
            e.forward(Ad, Bd, weight_id=0, precision='fp8')
        assert ex.value.code == L.ERR_STATE
    finally:
        e.close()


def test_fp8_scales_replay_in_graph(synth, eng):
    """Scales sit at fixed device addresses: a captured step replays with the values set last."""
    n = 5
    rgb, depth, poses, rgbA, depthA = track_inputs(synth, n, 12)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(eng.device)
    args = (t(rgb), t(depth), synth.CAMERA_K, t(poses), t(np.full(n, 200.0)), t(rgbA), t(depthA), TN, RN)
    a, b, _, _ = eng.preprocess(*args[:7], want_tensors=True)
    s = eng.calibrate_fp8(a, b, weight_id=0)
    outs = dict(out_poses=torch.empty_like(args[3]),
                out_trans=torch.empty(n, 3, dtype=torch.float32, device=eng.device),
                out_rot=torch.empty(n, 3, dtype=torch.float32, device=eng.device))

    def step():                                       # same arguments and addresses every time: one graph
        eng.track_batch(*args, precision='fp8', **outs)
        return [x.clone() for x in outs.values()]

    out1 = step()
    out2 = step()
    assert eng.last_step_was_graph() and all(torch.equal(x, y) for x, y in zip(out1, out2))
    eng.set_fp8_scales(s * 2, 0)                      # coarser: the replayed graph's results change
    out3 = step()
    assert eng.last_step_was_graph() and not torch.equal(out3[1], out1[1])
    eng.set_fp8_scales(s, 0)
    out4 = step()
    assert eng.last_step_was_graph() and all(torch.equal(x, y) for x, y in zip(out4, out1))


def test_fp8_saturates_beyond_calibration(synth, eng):
    """Inputs 8x beyond the calibration: finite outputs, saturated codes, no NaN code in any e4m3 tensor."""
    n = 4
    A, B = synth.tensor_pairs(n, seed=21)
    Ad, Bd = A.to(eng.device), B.to(eng.device)
    eng.calibrate_fp8(Ad, Bd, weight_id=0)
    tr, ro, _ = eng.forward(Ad * 8, Bd * 8, weight_id=0, precision='fp8')
    torch.cuda.synchronize()
    assert bool(torch.isfinite(tr).all()) and bool(torch.isfinite(ro).all())
    saturated = 0
    for buf in E.E4M3_BUFS:
        u = buffer_bytes(eng, buf)[:n * E.image_bytes(buf)]
        assert not bool(((u & 0x7F) == 0x7F).any()), 'NaN code in ' + buf
        saturated += int(((u & 0x7F) == 0x7E).sum())
    assert saturated > 0


# The 6-vector's worst |error| against the fp32 reference forward in a CPU emulation of this exact arithmetic
# (scripts/fp8_study.py, SE3TN_FP8_HEADROOM = 2; fp32 sums, so the narrower FP8 accumulation is not in it).  The gates are
# 2x these, the way the bf16 mode's gate was set.
EMU_WORST = {'config 1': 0.02489, 'raw set 0': 0.02257, 'raw set 1': 0.02969}


def test_fp8_config1_against_reference(synth, golden_dir, eng):
    """BASELINE config 1 (the shipped pair, batch 1) against the reference's own forward (golden), calibrated on itself."""
    import cv2
    import os
    g = np.load(os.path.join(golden_dir, 'golden_model.npz'))
    rgbA = cv2.imread(os.path.join(golden_dir, 'c1_rgbA.png'))[..., ::-1].copy()
    rgbB = cv2.imread(os.path.join(golden_dir, 'c1_rgbB.png'))[..., ::-1].copy()
    depthA, depthB = synth.depth_from_rgb(rgbA), synth.depth_from_rgb(rgbB)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)[None]).to(eng.device)
    pose = t(synth.config1_pose())
    tA, tB = eng.normalize(t(rgbA), t(depthA), t(rgbB), t(depthB), pose, precision='fp8')
    eng.calibrate_fp8(tA, tB, weight_id=0)
    tr, ro, _ = eng.forward(tA, tB, weight_id=0, precision='fp8')
    ref = np.concatenate([g['c1_trans'], g['c1_rot']], 1)
    err = float(np.abs(torch.cat((tr, ro), 1).cpu().numpy() - ref).max())
    print('\nconfig 1, fp8: max |err| %.4g (emulation %.4g, gate %.4g)' % (err, EMU_WORST['config 1'], 2 * EMU_WORST['config 1']))
    assert err <= 2 * EMU_WORST['config 1']


def test_fp8_raw_regime_batch64_against_reference(synth, eng):
    """The parity tests' raw-regime frame, 64 tracks, weight seeds 0 / 1 on 32 each in one step, each set calibrated on its
    own tracks through Engine.calibrate_fp8_tracks: every 6-vector against the fp32 reference forward (se3_oracle.on_track)."""
    import se3_oracle as O
    n = 64
    rgb, depth, poses, rgbA, depthA = track_inputs(synth, n, 11)
    dev = eng.device
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    wid = np.repeat(np.array([0, 1], dtype=np.int32), n // 2)
    wdev, P, ow = t(wid), t(poses), t(np.full(n, 200.0))
    fr, fd, A_, dA = t(rgb), t(depth), t(rgbA), t(depthA)
    for w in (0, 1):                                  # drop what earlier tests calibrated: reload the sets' weights
        eng.load_state_dict(synth.make_state_dict(w), w)
    assert eng.calibrate_fp8_tracks(fr, fd, synth.CAMERA_K, P, ow, A_, dA, weight_ids=wid) == [0, 1]
    assert eng.calibrate_fp8_tracks(fr, fd, synth.CAMERA_K, P, ow, A_, dA, weight_ids=wid) == []   # both have scales now
    _, tr, ro = eng.track_batch(fr, fd, synth.CAMERA_K, P, ow, A_, dA, TN, RN, weight_ids_host=wid, weight_ids_dev=wdev,
                                precision='fp8')
    out = torch.cat((tr, ro), 1).double().cpu().numpy()
    mean, std = synth.default_mean_std()
    stats = {0: (mean, std), 1: (mean + 1.5, std * 1.25)}
    sds = {0: synth.make_state_dict(0), 1: synth.make_state_dict(1)}
    ref = np.stack([np.concatenate([d['trans'], d['rot']]) for _, d in
                    (O.on_track(sds[int(wid[i])], poses[i], rgb, depth, rgbA[i], depthA[i], synth.CAMERA_K, 200.0,
                                *stats[int(wid[i])], return_all=True) for i in range(n))])
    assert np.isfinite(out).all()
    for w in (0, 1):
        err = float(np.abs(out[wid == w] - ref[wid == w]).max())
        e = EMU_WORST['raw set %d' % w]
        print('\nraw regime n = 64, set %d, fp8: max |err| %.4g (emulation %.4g, gate %.4g)' % (w, err, e, 2 * e))
        assert err <= 2 * e


# ------------------------------------------------------------------------------------------- the callers of the helper
def test_fp8_tracker_calibrates_on_its_first_frame(pkg, synth, tmp_path):
    """Tracker(precision='fp8'): the first on_track calibrates its set on that frame (input A passed in, B cropped at the
    previous pose) -- the same scales as Engine.calibrate_fp8 on those pairs -- and later frames keep the scales."""
    import importlib
    mio = importlib.import_module(pkg.__name__ + '.mesh_io')
    path = str(tmp_path / 'model.ply')
    mio.save_ply_mesh(path, synth.mesh(2, seed=4))
    K = synth.CAMERA_K
    info = {'resolution': 176, 'object_width': 200.0, 'boundingbox': 10,
            'camera': {'focalX': K[0, 0], 'focalY': K[1, 1], 'centerX': K[0, 2], 'centerY': K[1, 2], 'height': 480, 'width': 640}}
    mean, std = synth.default_mean_std()
    trk = pkg.Tracker(info, mean, std, {'state_dict': synth.make_state_dict(0)}, model_path=path, max_batch=8, precision='fp8')
    eng = trk.engine
    try:
        rgb, depth, poses, rgbA, depthA = track_inputs(synth, 1, 14)
        assert eng.fp8_scales(0) is None
        out = trk.on_track(poses[0], rgb, depth, rgbA=rgbA[0], depthA=depthA[0])
        s = eng.fp8_scales(0)
        assert s is not None and np.isfinite(out).all()
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(eng.device)
        A, B, _, _ = eng.preprocess(t(rgb), t(depth), K, t(poses), t(np.full(1, 200.0)), t(rgbA), t(depthA), want_tensors=True)
        assert np.array_equal(eng.calibrate_fp8(A, B, weight_id=0), s)
        eng.set_fp8_scales(s * 2, 0)                  # a later frame, rendered input A inside the step: no recalibration
        out2 = trk.on_track(out, rgb, depth)
        assert np.array_equal(eng.fp8_scales(0), s * 2) and np.isfinite(out2).all()
    finally:
        eng.close()
        importlib.import_module(pkg.__name__ + '.Utils').set_engine(None)   # the Tracker made this engine Utils' own


def test_fp8_problem_validate_calibrates_on_its_first_batch(pkg, synth, tmp_path):
    """problems.evaluate in 'fp8': the set is calibrated on the first validation batch (as eval_pairs normalises it), the
    losses are finite and the 6-vectors stay within twice the emulation's worst of the bf16x3 ones."""
    import importlib
    from test_gpu_validate import write_folder
    P = importlib.import_module(pkg.__name__ + '.problems')
    D = importlib.import_module(pkg.__name__ + '.datasets')
    eng = pkg.Engine(max_batch=8)
    try:
        eng.set_mesh(synth.mesh(), 0)
        mean, std = synth.default_mean_std()
        d = str(tmp_path / 'val')
        write_folder(eng, synth, d, 12, seed=5)
        ds = D.TrackDataset(d, 'val', mean, std, dataset_info={
            'resolution': 176, 'camera': {'focalX': 1066.778, 'focalY': 1067.487, 'centerX': 312.9869, 'centerY': 241.3109}},
            trans_normalizer=TN, rot_normalizer=RN, engine=eng, precision='fp8')
        model = pkg.Se3TrackNet(engine=eng, weight_id=0)
        model.load_state_dict(synth.make_state_dict(0))
        loader = torch.utils.data.DataLoader(ds, batch_size=12, shuffle=False, drop_last=False)
        prob = P.Problem(model, None, loader, config={'loss_weights': {'trans': 1, 'rot': 1}})
        r8 = prob.validation_losses('fp8', keep_predictions=True)
        s = eng.fp8_scales(0)
        assert s is not None and np.isfinite(r8['trans']) and np.isfinite(r8['rot'])
        pairs = [D.read_pair(f) for f in ds.rgbA_files[:8]]                          # the first step's pairs
        st = lambda k, dt: torch.from_numpy(np.stack([p[k] for p in pairs]).astype(dt)).to(eng.device)
        A, B = eng.normalize(st('rgbA', np.uint8), st('depthA', np.uint16), st('rgbB', np.uint8), st('depthB', np.uint16),
                             st('A_in_cam', np.float64))
        assert np.array_equal(eng.calibrate_fp8(A, B, weight_id=0), s)
        r3 = prob.validation_losses('bf16x3', keep_predictions=True)
        assert np.abs(r8['predictions'] - r3['predictions']).max() <= 2 * max(EMU_WORST.values())
    finally:
        eng.close()
