"""GPU parity tests: the CUDA path (through the C ABI / drop-in classes) against the oracle on the
same seeded inputs, and against the golden fixtures produced by the reference's own code.

Tolerances:
  * integer / byte / index work (bbox, crops): bit-exact
  * preprocessing floats (fp32 chain):          bit-exact (same IEEE ops as numpy)
  * network 6-vector, BF16X3 tensor-core path (the default): rtol 1e-3 / atol 1e-4 (BASELINE.json
    north_star) on EVERY case here, including large-magnitude raw-regime inputs and both weight seeds
  * network 6-vector, TF32 tensor-core path:    same gate where its 10-bit operands allow it (tensor
    regime, raw regime with weight seed 0); documented to exceed it on raw regime / weight seed 1
  * network 6-vector, BF16 (1 product) path:    rtol 1e-2 / atol 5e-3 (BASELINE configs[2]: bf16 operands AND 2-byte activations)
  * network 6-vector, FP32 FFMA path:           rtol 1e-4 / atol 2e-6
  * pose update / so(3) log (fp64 + libm trig): atol 1e-7 / 1e-9
  * poses produced from a TF32 6-vector: the gate propagated through datasets.py:169-174,
    |dt| <= (1e-4 + 1e-3)*0.03 m and |dR| <= (1e-4 + 1e-3)*rot_normalizer  ->  POSE_ATOL = 1e-4
"""
import hashlib, importlib, os
import numpy as np
import pytest
import torch
import se3_oracle as O

pytestmark = pytest.mark.gpu
RTOL, ATOL = 1e-3, 1e-4
POSE_ATOL = 1e-4
# bf16: 2-byte activations / weights, fp32 accumulate.  A CPU emulation of exactly that rounding (scripts/precision_study.py)
# gives max |err| 6.2e-4 .. 6.7e-4 on the 6-vector for tensor-regime inputs (16 pairs, both weight seeds); on config 1 (the shipped
# image pair, normalised magnitudes up to ~40) the tensor-core path measured 3.8e-3.  The gate is ~2x that worst case -- 5x tighter than the
# round-1 gate of (5e-2, 2e-2), which would have hidden a 40x regression.
RAW_BF16_GATE = (5e-2, 2e-2)       # bf16 on raw-regime inputs (see test_raw_regime_full_path_batch64_both_weight_seeds)
GATES = {'bf16x3': (RTOL, ATOL), 'tf32': (RTOL, ATOL), 'fp32': (1e-4, 2e-6), 'bf16': (1e-2, 5e-3)}


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.fixture(scope='module')
def eng(pkg, synth):
    e = pkg.Engine(max_batch=64)
    e.load_state_dict(synth.make_state_dict(0), 0)
    e.load_state_dict(synth.make_state_dict(1), 1)
    mean, std = synth.default_mean_std()
    e.set_stats(mean, std, 0)
    e.set_stats(mean + 1.5, std * 1.25, 1)
    yield e
    e.close()


def six(trans, rot):
    return torch.cat((trans, rot), 1).cpu()


def assert_gate(out, ref, rtol=RTOL, atol=ATOL):
    err = (out - ref).abs(); tol = atol + rtol * ref.abs()
    assert torch.isfinite(out).all()
    assert (err <= tol).all(), 'max err/tol %.3f' % (err / tol).max().item()
    return (err / tol).max().item()


# ------------------------------------------------------------------------------- network
def test_config1_parity_gate(pkg, synth, golden_dir, eng):
    """BASELINE config 1: the shipped RGB pair, batch 1, vs the REFERENCE's own forward (golden)."""
    import cv2
    g = np.load(os.path.join(golden_dir, 'golden_model.npz'))
    rgbA = cv2.imread(os.path.join(golden_dir, 'c1_rgbA.png'))[..., ::-1].copy()
    rgbB = cv2.imread(os.path.join(golden_dir, 'c1_rgbB.png'))[..., ::-1].copy()
    depthA, depthB = synth.depth_from_rgb(rgbA), synth.depth_from_rgb(rgbB)
    pose = synth.config1_pose()
    dev = eng.device
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)[None]).to(dev)
    ref = torch.from_numpy(np.concatenate([g['c1_trans'], g['c1_rot']], 1))
    for prec, (rt, at) in GATES.items():
        # `precision` also selects whether the conv-input buffers hold tf32-rounded values
        tA, tB = eng.normalize(t(rgbA), t(depthA), t(rgbB), t(depthB), torch.from_numpy(pose[None]).to(dev), precision=prec)
        assert sha(tA[0].cpu().numpy()) == str(g['c1_dataA_sha']) and sha(tB[0].cpu().numpy()) == str(g['c1_dataB_sha'])
        trans, rot, _ = eng.forward_preprocessed(1, weight_id=0, precision=prec)
        assert_gate(six(trans, rot), ref, rt, at)
        pose_out = eng.pose_update(torch.from_numpy(pose[None]).to(dev), trans, rot, 0.03, 5 * np.pi / 180)[0].cpu().numpy()
        assert np.allclose(pose_out, g['c1_pose_out'], rtol=0, atol={'fp32': 1e-7, 'bf16': 2e-3}.get(prec, POSE_ATOL))


@pytest.mark.parametrize('n', [1, 2, 3, 7])
def test_forward_matches_oracle_small_batches(synth, eng, n):
    sd = synth.make_state_dict(0)
    A, B = synth.tensor_pairs(n, seed=10 + n)
    ref = O.forward(sd, A, B)
    ref6 = torch.cat((ref['trans'], ref['rot']), 1)
    for prec, (rt, at) in GATES.items():
        trans, rot, feat = eng.forward(A.to(eng.device), B.to(eng.device), precision=prec, want_feature=True)
        assert_gate(six(trans, rot), ref6, rt, at)
        ftol = {'tf32': 2e-2, 'bf16x3': 2e-4, 'bf16': 1e-1, 'fp32': 1e-4}[prec]
        assert (feat.cpu() - ref['feature']).abs().max().item() < ftol * ref['feature'].abs().max().item()


def test_forward_golden_fixture(synth, golden_dir, eng):
    g = np.load(os.path.join(golden_dir, 'golden_model.npz'))
    A, B = synth.tensor_pairs(2, seed=0)
    for prec, ftol in (('bf16x3', 2e-4), ('tf32', 2e-2)):
        trans, rot, feat = eng.forward(A.to(eng.device), B.to(eng.device), precision=prec, want_feature=True)
        assert_gate(six(trans, rot), torch.from_numpy(np.concatenate([g['trans'], g['rot']], 1)))
        assert np.abs(feat.cpu().numpy()[:, ::16, ::3, ::3] - g['feature_sub']).max() < ftol * np.abs(g['feature_sub']).max()


def test_batch64_full_size_properties(synth, eng):
    """BASELINE config 2 size.  Oracle on all 64 pairs (~1 s on CPU) + size-independent properties:
    batch-composition independence (a pair's result does not depend on its neighbours) and
    determinism."""
    sd = synth.make_state_dict(0)
    A, B = synth.tensor_pairs(64, seed=2)
    Ad, Bd = A.to(eng.device), B.to(eng.device)
    ref = O.forward(sd, A, B)
    ref6 = torch.cat((ref['trans'], ref['rot']), 1)
    for prec in ('bf16x3', 'tf32'):
        t1, r1, _ = eng.forward(Ad, Bd, precision=prec)
        worst = assert_gate(six(t1, r1), ref6)
        print('batch-64 %s worst err/tol: %.3f' % (prec, worst))
        t2, r2, _ = eng.forward(Ad, Bd, precision=prec)
        assert torch.equal(t1, t2) and torch.equal(r1, r2)                       # deterministic
        perm = torch.randperm(64, generator=torch.Generator().manual_seed(0)).to(eng.device)
        t3, r3, _ = eng.forward(Ad[perm].contiguous(), Bd[perm].contiguous(), precision=prec)
        assert torch.equal(t3, t1[perm]) and torch.equal(r3, r1[perm])           # per-pair independence
        t4, r4, _ = eng.forward(Ad[:5].contiguous(), Bd[:5].contiguous(), precision=prec)
        assert torch.equal(t4, t1[:5]) and torch.equal(r4, r1[:5])               # ragged tail of a batch
    tf, rf, _ = eng.forward(Ad, Bd, precision='fp32')
    assert_gate(six(tf, rf), ref6, 1e-4, 2e-6)
    tb, rb, _ = eng.forward(Ad, Bd, precision='bf16')
    print('batch-64 bf16 worst err/(5e-2,2e-2): %.3f' % assert_gate(six(tb, rb), ref6, 5e-2, 2e-2))


def test_second_weight_set_and_module_api(pkg, synth):
    sd1 = synth.make_state_dict(1)
    net = pkg.Se3TrackNet(image_size=176)
    net.load_state_dict(sd1)
    net = net.cuda(); net.eval()
    A, B = synth.tensor_pairs(2, seed=5)
    with torch.no_grad():
        out = net(A.cuda(), B.cuda())
    assert set(out) == {'feature', 'trans', 'rot'} and out['feature'].shape == (2, 256, 22, 22)
    ref = O.forward(sd1, A, B)
    assert_gate(six(out['trans'], out['rot']), torch.cat((ref['trans'], ref['rot']), 1))
    with pytest.raises(NotImplementedError):
        net.train()


# -------------------------------------------------------------------------- preprocessing
def _frame_case(synth, n, seed):
    rgb, depth = synth.raw_frame(seed)
    poses = synth.raw_poses(n, seed=seed)
    rgbA, depthA = synth.rendered_views(n, poses, seed=seed)
    return rgb, depth, poses, rgbA, depthA


def test_preprocess_bit_exact_vs_oracle(synth, eng):
    n = 8
    rgb, depth, poses, rgbA, depthA = _frame_case(synth, n, 0)
    poses[1, :3, 3] = (-0.13, -0.1, 0.5)          # window clipped at the top-left of the frame
    poses[2, :3, 3] = (0.14, 0.1, 0.45)           # clipped bottom-right
    poses[3, :3, 3] = (0.0, 0.0, 0.25)            # window larger than the frame
    poses[4, :3, 3] = (0.01, 0.02, 1.9)           # far object: 112-px window upsampled
    dev = eng.device
    ow = np.full(n, 200.0); ow[5] = 187.3
    wid = np.array([0, 1, 0, 1, 0, 0, 1, 1], dtype=np.int32)
    mean, std = synth.default_mean_std()
    stats = {0: (mean, std), 1: (mean + 1.5, std * 1.25)}
    tA, tB, crgb, cdepth = eng.preprocess(torch.from_numpy(rgb).to(dev), torch.from_numpy(depth).to(dev), synth.CAMERA_K,
                                          torch.from_numpy(poses).to(dev), torch.from_numpy(ow).to(dev),
                                          torch.from_numpy(rgbA).to(dev), torch.from_numpy(depthA).to(dev),
                                          weight_ids=torch.from_numpy(wid).to(dev), precision='tf32', want_tensors=True, want_crops=True)
    bbs = eng.compute_bbox(torch.from_numpy(poses).to(dev), synth.CAMERA_K, torch.from_numpy(ow).to(dev)).cpu().numpy()
    for i in range(n):
        bb = O.compute_bbox(poses[i], synth.CAMERA_K, ow[i], scale=(1000, 1000, 1000))
        assert np.array_equal(bbs[i], bb)
        rB, dB = O.crop_bbox(rgb, depth, bb, (176, 176))
        assert np.array_equal(crgb[i].cpu().numpy(), rB) and np.array_equal(cdepth[i].cpu().numpy(), dB), i
        m, s = stats[int(wid[i])]
        (dA_, dB_), _ = O.process_data(rgbA[i], depthA[i], poses[i], rB, dB, np.eye(4), m, s)
        assert np.array_equal(tA[i].cpu().numpy(), dA_) and np.array_equal(tB[i].cpu().numpy(), dB_), i
    # the conv-input buffers hold the same values (tf32-rounded) in padded NHWC4
    x0b = eng.debug_buffer(1, n).view(n, 182, 184, 4)[:, 3:179, 3:179, :].permute(0, 3, 1, 2)
    assert (x0b - tB).abs().max().item() <= 2.0 ** -11 * tB.abs().max().item()
    assert float(eng.debug_buffer(1, n).view(n, 182, 184, 4)[:, :3].abs().max()) == 0.0      # halo stays zero


def test_golden_crops_and_process_data(pkg, synth, golden_dir, eng):
    """Against fixtures generated by the reference's own Utils/datasets code."""
    p = np.load(os.path.join(golden_dir, 'golden_pre.npz'))
    dev = eng.device
    rgb, depth, K = p['small_rgb'], p['small_depth'], p['K_small']
    n = len(p['object_width'])
    poses = p['poses']
    bbs = eng.compute_bbox(torch.from_numpy(poses).to(dev), K, torch.from_numpy(p['object_width']).to(dev))
    crgb, cdepth = eng.crop_bbox(torch.from_numpy(rgb).to(dev), torch.from_numpy(depth).to(dev), bbs)
    for i in range(n):
        assert np.array_equal(bbs[i].cpu().numpy(), p[f'bb_{i}'])
        assert sha(crgb[i].cpu().numpy()) == str(p[f'rgbB_sha_{i}']) and sha(cdepth[i].cpu().numpy()) == str(p[f'depthB_sha_{i}'])
    gl = eng.compute_bbox(torch.from_numpy(poses[1:2]).to(dev), K, torch.tensor([200.0], dtype=torch.float64, device=dev),
                          scale=(1000., -1000., 1000.))
    assert np.array_equal(gl[0].cpu().numpy(), p['bb_gl_0'])
    # TrackDataset.processData drop-in, both mean/std dtype chains
    rgbAs, depthAs = synth.rendered_views(n, poses, seed=7)
    mean, std = synth.default_mean_std()
    chains = {'f32': (mean, std), 'f64': (mean.astype(np.float64) + 0.123, std.astype(np.float64) * 1.01)}
    for tag, (m, s) in chains.items():
        e2 = pkg.Engine(max_batch=1)
        ds = pkg.TrackDataset('', 'eval', m, s, None, None, None, None, engine=e2)
        for i in range(n):
            rB, dB = crgb[i].cpu().numpy(), cdepth[i].cpu().numpy()
            sample, (tl, rl), _, _, mA, mB = ds.processData(rgbAs[i], depthAs[i], poses[i].copy(), rB, dB, p[f'gtB_{i}'].copy())
            assert sample[0].dtype == torch.float32 and not sample[0].is_cuda
            assert sha(sample[0].numpy()) == str(p[f'dataA_sha_{tag}_{i}']), (tag, i)
            assert sha(sample[1].numpy()) == str(p[f'dataB_sha_{tag}_{i}']), (tag, i)
            assert np.allclose(tl, p[f'label_trans_{i}'], rtol=0, atol=1e-12)
            assert np.allclose(rl, p[f'label_rot_{i}'], rtol=0, atol=1e-9)
            assert np.array_equal(mA, (depthAs[i] > 100).astype(np.uint8))
        e2.close()


def test_full_frame_golden_crops(synth, golden_dir, eng):
    p = np.load(os.path.join(golden_dir, 'golden_pre.npz'))
    rgb, depth = synth.raw_frame(0)
    poses = synth.raw_poses(8, seed=0)
    dev = eng.device
    ow = torch.full((8,), 200.0, dtype=torch.float64, device=dev)
    bbs = eng.compute_bbox(torch.from_numpy(poses).to(dev), synth.CAMERA_K, ow)
    crgb, cdepth = eng.crop_bbox(torch.from_numpy(rgb).to(dev), torch.from_numpy(depth).to(dev), bbs)
    for i in range(8):
        assert np.array_equal(bbs[i].cpu().numpy(), p[f'full_bb_{i}'])
        assert sha(crgb[i].cpu().numpy()) == str(p[f'full_rgbB_sha_{i}']) and sha(cdepth[i].cpu().numpy()) == str(p[f'full_depthB_sha_{i}'])


def test_utils_dropins(pkg, synth):
    U = importlib.import_module('iros20-6d-pose-tracking_b200.Utils')
    rgb, depth = synth.raw_frame(4, 120, 160)
    K = synth.CAMERA_K.copy(); K[:2] *= 0.25
    pose = synth.raw_poses(1, seed=4)[0]; pose[:3, 3] = (0.01, -0.02, 0.6)
    bb = U.compute_bbox(pose, K, 215.5, scale=(1000, 1000, 1000))
    assert bb.dtype == np.int32 and np.array_equal(bb, O.compute_bbox(pose, K, 215.5, scale=(1000, 1000, 1000)))
    a, b = U.crop_bbox(rgb, depth, bb, (176, 176)); c, d = O.crop_bbox(rgb, depth, bb, (176, 176))
    assert a.dtype == np.uint8 and b.dtype == np.uint16 and np.array_equal(a, c) and np.array_equal(b, d)
    a, b = U.crop_bbox(rgb, depth, bb, (100, 100)); c, d = O.crop_bbox(rgb, depth, bb, (100, 100))
    assert np.array_equal(a, c) and np.array_equal(b, d)


# ------------------------------------------------------------------------------ Lie-algebra ops
def test_pose_update_and_log_vs_golden(golden_dir, eng):
    p = np.load(os.path.join(golden_dir, 'golden_pre.npz'))
    dev = eng.device
    poses = torch.from_numpy(p['pu_poses']).to(dev)
    tr, ro = torch.from_numpy(p['pu_trans']).to(dev), torch.from_numpy(p['pu_rot']).to(dev)
    o5 = eng.pose_update(poses, tr, ro, 0.03, 5 * np.pi / 180).cpu().numpy()
    o30 = eng.pose_update(poses, tr, ro, 0.03, 30 * np.pi / 180).cpu().numpy()
    assert np.abs(o5 - p['pu_out_5deg']).max() < 1e-7 and np.abs(o30 - p['pu_out_30deg']).max() < 1e-7
    assert np.array_equal(o5[0], p['pu_poses'][0])                      # zero residual: exact identity
    assert np.array_equal(o5[:, 3], np.tile([0, 0, 0, 1.0], (len(o5), 1)))
    # round trip: log(exp(w) R, R) == w
    back_t, back_r = eng.so3_log(poses, torch.from_numpy(p['pu_out_30deg']).to(dev), 0.03, 30 * np.pi / 180)
    assert np.abs(back_t.cpu().numpy() - p['pu_trans'].astype(np.float64)).max() < 1e-6
    assert np.abs(back_r.cpu().numpy() - p['pu_rot'].astype(np.float64)).max() < 1e-6


def test_so3_log_near_pi_and_identity(eng):
    import cv2
    dev = eng.device
    ws = [np.zeros(3), np.array([1e-7, 0, 0]), np.array([np.pi - 1e-7, 0, 0]), np.array([0, 3.1, 0.2]),
          np.array([2.2, -2.2, 0.1]), np.array([0.3, 0.2, -0.1])]
    A = np.tile(np.eye(4), (len(ws), 1, 1)); B = A.copy()
    for i, w in enumerate(ws):
        B[i, :3, :3] = cv2.Rodrigues(w)[0]
    _, rl = eng.so3_log(torch.from_numpy(A).to(dev), torch.from_numpy(B).to(dev), 1.0, 1.0)
    ref = np.stack([cv2.Rodrigues(O.normalize_rotation_matrix(B[i, :3, :3].copy()))[0].ravel() for i in range(len(ws))])
    assert np.abs(rl.cpu().numpy() - ref).max() < 1e-7


# ------------------------------------------------------------------------------ end to end
def test_on_track_end_to_end_vs_oracle(pkg, synth):
    """Tracker.on_track drop-in: raw frame + pose in, pose out, against the oracle's on_track."""
    sd = synth.make_state_dict(0)
    mean, std = synth.default_mean_std()
    info = {'resolution': 176, 'boundingbox': 10, 'object_width': 200.0,
            'camera': {'focalX': synth.CAMERA_K[0, 0], 'focalY': synth.CAMERA_K[1, 1], 'centerX': synth.CAMERA_K[0, 2],
                       'centerY': synth.CAMERA_K[1, 2], 'height': 480, 'width': 640}}
    trk = pkg.Tracker(info, mean, std, {'state_dict': sd}, model_path=None, max_batch=8)
    n = 4
    rgb, depth, poses, rgbA, depthA = _frame_case(synth, n, 3)
    for i in range(n):
        got = trk.on_track(poses[i], rgb, depth, rgbA=rgbA[i], depthA=depthA[i])
        ref = O.on_track(sd, poses[i], rgb, depth, rgbA[i], depthA[i], synth.CAMERA_K, 200.0, mean, std)
        assert got.dtype == np.float64 and got.shape == (4, 4)
        assert np.abs(got - ref).max() < POSE_ATOL
    batch = trk.on_track_batch(poses, rgb, depth, rgbA, depthA)
    singles = np.stack([trk.on_track(poses[i], rgb, depth, rgbA=rgbA[i], depthA=depthA[i]) for i in range(n)])
    assert np.array_equal(batch, singles)
    assert trk.frame_cnt == 2 * n
    # host tensors: uploads staged on the tracker's copy stream (double-buffered); result stays on the device
    host = [torch.from_numpy(a) for a in (poses, rgb, depth, rgbA, depthA)]
    for _ in range(3):                                   # exercises both staging slots and their reuse
        staged = trk.on_track_batch(*host)
        assert staged.is_cuda and np.array_equal(staged.cpu().numpy(), batch)


def test_track_host_one_call_equals_device_path(pkg, synth, eng):
    """se3tn_track_host (numpy in / numpy out in ONE library call: pinned staging of the crop-window rectangle, graph replay, read
    back) runs the same kernels on the same bytes as se3tn_track_batch on device tensors: identical poses, for windows inside,
    across and outside the frame, several frame sizes, per-track weight sets and widths, and repeated calls (graph replay)."""
    dev = eng.device
    mean, std = synth.default_mean_std()
    TN, RN = 0.03, 5 * np.pi / 180
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    for n, seed, shape in ((1, 3, None), (3, 4, None), (6, 6, None), (2, 8, (240, 320))):
        rgb, depth, poses, rgbA, depthA = _frame_case(synth, n, seed)
        if shape is not None:                                   # another frame size: the context re-sizes its staging
            rgb, depth = np.ascontiguousarray(rgb[:shape[0], :shape[1]]), np.ascontiguousarray(depth[:shape[0], :shape[1]])
        poses = poses.copy()
        poses[0, :3, 3] = (0.32, -0.2, 0.5)                      # window hangs over the frame's edge
        if n > 1:
            poses[1, :3, 3] = (2.0, 2.0, 0.5)                    # window misses the frame entirely
        ow = np.full(n, 200.0); ow[-1] = 150.0
        wid = (np.arange(n) * 2 // max(n, 1)).astype(np.int32) if n >= 3 else None
        want, wtr, wro = eng.track_batch(t(rgb), t(depth), synth.CAMERA_K, t(poses), t(ow), t(rgbA), t(depthA), TN, RN,
                                         weight_ids_host=wid)
        want, wtr, wro = want.cpu().numpy(), wtr.cpu().numpy(), wro.cpu().numpy()
        for rep in range(3):
            got, tr, ro = eng.track_host(rgb, depth, synth.CAMERA_K, poses, ow, rgbA, depthA, TN, RN, weight_ids=wid, want_residuals=True)
            assert np.array_equal(got, want) and np.array_equal(tr, wtr) and np.array_equal(ro, wro), (n, rep)
        assert eng.last_step_was_graph()
    with pytest.raises(ValueError):
        eng.track_host(rgb, depth.astype(np.float32), synth.CAMERA_K, poses, ow, rgbA, depthA, TN, RN)
    with pytest.raises(RuntimeError):                           # more tracks than the context was created for
        big = 70
        eng.track_host(rgb, depth, synth.CAMERA_K, np.tile(poses[:1], (big, 1, 1)), np.full(big, 200.0), np.tile(rgbA[:1], (big, 1, 1, 1)),
                       np.tile(depthA[:1], (big, 1, 1)), TN, RN)
    # the Tracker's numpy route is this call, its CUDA-tensor route is track_batch -- same poses either way
    info = {'resolution': 176, 'boundingbox': 10, 'object_width': 200.0,
            'camera': {'focalX': synth.CAMERA_K[0, 0], 'focalY': synth.CAMERA_K[1, 1], 'centerX': synth.CAMERA_K[0, 2],
                       'centerY': synth.CAMERA_K[1, 2], 'height': 480, 'width': 640}}
    trk = pkg.Tracker(info, mean, std, {'state_dict': synth.make_state_dict(0)}, model_path=None, engine=eng)
    rgb, depth, poses, rgbA, depthA = _frame_case(synth, 2, 5)
    a = trk.on_track_batch(poses, rgb, depth, rgbA, depthA)
    b = trk.on_track_batch(*map(t, (poses, rgb, depth, rgbA, depthA)))
    assert b.is_cuda and np.array_equal(a, b.cpu().numpy())


def test_track_batch_mixed_weight_sets(synth, eng):
    n = 6
    rgb, depth, poses, rgbA, depthA = _frame_case(synth, n, 6)
    dev = eng.device
    wid = np.array([0, 0, 0, 1, 1, 1], dtype=np.int32)
    ow = torch.full((n,), 200.0, dtype=torch.float64, device=dev)
    args = (torch.from_numpy(rgb).to(dev), torch.from_numpy(depth).to(dev), synth.CAMERA_K, torch.from_numpy(poses).to(dev), ow,
            torch.from_numpy(rgbA).to(dev), torch.from_numpy(depthA).to(dev), 0.03, 5 * np.pi / 180)
    mean, std = synth.default_mean_std()
    stats = {0: (mean, std), 1: (mean + 1.5, std * 1.25)}
    sds = {0: synth.make_state_dict(0), 1: synth.make_state_dict(1)}
    refs = [O.on_track(sds[int(wid[i])], poses[i], rgb, depth, rgbA[i], depthA[i], synth.CAMERA_K, 200.0, *stats[int(wid[i])], return_all=True)
            for i in range(n)]
    ref6 = torch.from_numpy(np.stack([np.concatenate([d['trans'], d['rot']]) for _, d in refs]))
    worst = {}
    for prec in ('bf16x3', 'tf32'):
        out, tr, ro = eng.track_batch(*args, weight_ids_host=wid, precision=prec)
        got6 = torch.cat((tr, ro), 1).cpu()
        err = (got6 - ref6).abs() / (ATOL + RTOL * ref6.abs())
        worst[prec] = err.max().item()
        if prec == 'bf16x3':
            assert_gate(got6, ref6)
            for i in range(n):
                assert np.abs(out[i].cpu().numpy() - refs[i][0]).max() < POSE_ATOL
    print('raw regime, weight seeds 0/1: worst err/tol bf16x3 %.3f, tf32 %.3f' % (worst['bf16x3'], worst['tf32']))
    # Large-magnitude inputs (F13) through 17 layers: TF32's 10-bit operands are not enough for the fp32 gate
    # with weight seed 1 (CPU emulation of exact TF32 rounding predicts err/tol 3.4) -- this is why BF16X3 is the
    # default.  Keep TF32 honest: it must stay in the same ballpark, not silently drift.
    assert worst['bf16x3'] < 0.5 and worst['tf32'] < 8.0



def test_latency_mode_split_k_consistency(synth, eng):
    """n <= 4 runs the trunk with split-K work units (latency mode): results within the gate of the oracle, independent of n inside
    the mode (1 vs 4 pairs: bit-identical), and equal to the throughput mode (n = 5: same pairs) to fp32 rounding."""
    sd = synth.make_state_dict(0)
    A, B = synth.tensor_pairs(5, seed=23)
    Ad, Bd = A.to(eng.device), B.to(eng.device)
    ref = O.forward(sd, A, B); ref6 = torch.cat((ref['trans'], ref['rot']), 1)
    for prec in ('bf16x3', 'tf32', 'bf16'):
        t5, r5, _ = eng.forward(Ad, Bd, precision=prec)                                   # throughput mode
        t4, r4, _ = eng.forward(Ad[:4].contiguous(), Bd[:4].contiguous(), precision=prec)   # latency mode
        assert_gate(six(t4, r4), ref6[:4], *GATES[prec])
        singles = [eng.forward(Ad[i:i + 1].contiguous(), Bd[i:i + 1].contiguous(), precision=prec) for i in range(4)]
        for i, (t1, r1, _) in enumerate(singles):
            assert torch.equal(t1[0], t4[i]) and torch.equal(r1[0], r4[i])
        d = (six(t4, r4) - six(t5, r5)[:4]).abs().max().item()
        # a last-bit change of an fp32 sum can flip the rounding of a stored activation (2^-16 relative in bf16x3, 2^-11 in tf32, 2^-9 in bf16)
        assert d < {'bf16x3': 5e-6, 'tf32': 5e-4, 'bf16': 5e-3}[prec], d
        t4b, r4b, _ = eng.forward(Ad[:4].contiguous(), Bd[:4].contiguous(), precision=prec)
        assert torch.equal(t4, t4b) and torch.equal(r4, r4b)                              # deterministic whatever the arrival order of the pieces


# ------------------------------------------------------------------------------ BASELINE configs at full size
def test_raw_regime_full_path_batch64_both_weight_seeds(synth, eng):
    """BASELINE configs[1] at its real size: 64 tracks of one raw frame (large-magnitude normalised inputs, F13) through
    K0 -> conv stack -> K6, half of the tracks on weight seed 0 and half on seed 1 (per-object checkpoints in the same
    launches), every 6-vector and pose against the oracle.  bf16x3 must meet the north-star gate on all 64."""
    n = 64
    rgb, depth, poses, rgbA, depthA = _frame_case(synth, n, 11)
    dev = eng.device
    wid = np.repeat(np.array([0, 1], dtype=np.int32), n // 2)
    ow = torch.full((n,), 200.0, dtype=torch.float64, device=dev)
    args = (torch.from_numpy(rgb).to(dev), torch.from_numpy(depth).to(dev), synth.CAMERA_K, torch.from_numpy(poses).to(dev), ow,
            torch.from_numpy(rgbA).to(dev), torch.from_numpy(depthA).to(dev), 0.03, 5 * np.pi / 180)
    mean, std = synth.default_mean_std()
    stats = {0: (mean, std), 1: (mean + 1.5, std * 1.25)}
    sds = {0: synth.make_state_dict(0), 1: synth.make_state_dict(1)}
    refs = [O.on_track(sds[int(wid[i])], poses[i], rgb, depth, rgbA[i], depthA[i], synth.CAMERA_K, 200.0, *stats[int(wid[i])], return_all=True)
            for i in range(n)]
    ref6 = torch.from_numpy(np.stack([np.concatenate([d['trans'], d['rot']]) for _, d in refs]))
    ref_pose = np.stack([r[0] for r in refs])
    out, tr, ro = eng.track_batch(*args, weight_ids_host=wid, precision='bf16x3')
    worst = assert_gate(torch.cat((tr, ro), 1).cpu(), ref6)
    assert np.abs(out.cpu().numpy() - ref_pose).max() < POSE_ATOL
    # the same tracks one weight set at a time (single-set launches) give the same bits as the mixed launch
    for w in (0, 1):
        sel = np.nonzero(wid == w)[0]
        a2 = (args[0], args[1], args[2], args[3][sel[0]:sel[-1] + 1].contiguous(), ow[:len(sel)], args[5][sel[0]:sel[-1] + 1].contiguous(),
              args[6][sel[0]:sel[-1] + 1].contiguous(), 0.03, 5 * np.pi / 180)
        o2, _, _ = eng.track_batch(*a2, weight_ids_host=np.full(len(sel), w, np.int32), precision='bf16x3')
        assert torch.equal(o2, out[sel[0]:sel[-1] + 1])
    # bf16 on raw-regime inputs: normalised magnitudes up to ~40 (F13) enter 17 layers of 8-bit-mantissa operands, so the
    # 6-vector error is an order of magnitude above the tensor-regime one; RAW_BF16_GATE is ~3x the worst observed
    out_b, tr_b, ro_b = eng.track_batch(*args, weight_ids_host=wid, precision='bf16')
    worst_b = assert_gate(torch.cat((tr_b, ro_b), 1).cpu(), ref6, *RAW_BF16_GATE)
    print('raw regime n=64, seeds 0/1: worst err/tol bf16x3 %.3f (gate 1e-3/1e-4), bf16 %.3f (gate %g/%g)' % ((worst, worst_b) + RAW_BF16_GATE))


def test_batch256_bf16_and_bf16x3_vs_oracle(pkg, synth):
    """BASELINE configs[2]: batch 256 through one Engine(max_batch=256): the 2-byte bf16 path against its gate and the
    default bf16x3 path against the north-star gate, all 256 pairs vs the oracle; determinism and the equality of a pair's
    result at batch 256 and in a batch of its own."""
    n = 256
    e = pkg.Engine(max_batch=n)
    try:
        sd = synth.make_state_dict(0)
        e.load_state_dict(sd, 0)
        A, B = synth.tensor_pairs(n, seed=5)
        ref = O.forward(sd, A, B)
        ref6 = torch.cat((ref['trans'], ref['rot']), 1)
        Ad, Bd = A.to(e.device), B.to(e.device)
        for prec in ('bf16', 'bf16x3'):
            t1, r1, _ = e.forward(Ad, Bd, precision=prec)
            worst = assert_gate(six(t1, r1), ref6, *GATES[prec])
            print('batch-256 %s worst err/tol: %.3f' % (prec, worst))
            t2, r2, _ = e.forward(Ad, Bd, precision=prec)
            assert torch.equal(t1, t2) and torch.equal(r1, r2)
            t3, r3, _ = e.forward(Ad[200:205].contiguous(), Bd[200:205].contiguous(), precision=prec)      # (n > 4: not the split-K latency mode)
            assert torch.equal(t3, t1[200:205]) and torch.equal(r3, r1[200:205])
    finally:
        e.close()


def test_missing_stats_or_weights_are_errors(pkg, synth):
    """ADVICE r1: an id with weights but no statistics (or statistics but no weights) must be refused, not normalised / convolved
    with garbage."""
    e = pkg.Engine(max_batch=4)
    try:
        mean, std = synth.default_mean_std()
        e.load_state_dict(synth.make_state_dict(0), 0); e.set_stats(mean, std, 0)
        e.load_state_dict(synth.make_state_dict(1), 1)                       # weights, no stats
        e.set_stats(mean, std, 2)                                            # stats, no weights
        n = 2
        rgb, depth, poses, rgbA, depthA = _frame_case(synth, n, 2)
        dev = e.device
        args = (torch.from_numpy(rgb).to(dev), torch.from_numpy(depth).to(dev), synth.CAMERA_K, torch.from_numpy(poses).to(dev),
                torch.full((n,), 200.0, dtype=torch.float64, device=dev), torch.from_numpy(rgbA).to(dev), torch.from_numpy(depthA).to(dev), 0.03, 0.0873)
        for bad in ([0, 1], [0, 2], [0, 7]):
            with pytest.raises(pkg._lib.Se3tnError) as ei:
                e.track_batch(*args, weight_ids_host=np.array(bad, np.int32))
            assert ei.value.code == pkg._lib.ERR_STATE
        A, B = synth.tensor_pairs(1, seed=0)
        with pytest.raises(pkg._lib.Se3tnError):
            e.forward(A.to(dev), B.to(dev), weight_id=2)                     # set_stats alone does not make a weight set
        out, _, _ = e.track_batch(*args, weight_ids_host=np.array([0, 0], np.int32))   # the context still works
        assert torch.isfinite(out).all()
    finally:
        e.close()


def test_empty_and_oversized_batches(synth, eng):
    dev = eng.device
    A0 = torch.empty(0, 4, 176, 176, device=dev); 
    t, r, f = eng.forward(A0, A0.clone(), want_feature=True)
    assert t.shape == (0, 3) and r.shape == (0, 3) and f.shape == (0, 256, 22, 22)
    # more pairs than max_batch: Engine.forward walks the batch in max_batch slices
    sd = synth.make_state_dict(0)
    A, B = synth.tensor_pairs(66, seed=21)
    t, r, _ = eng.forward(A.to(dev), B.to(dev))
    ref = O.forward(sd, A[60:], B[60:])
    assert_gate(six(t[60:], r[60:]), torch.cat((ref['trans'], ref['rot']), 1))
    t2, r2, _ = eng.forward(A[64:].to(dev).contiguous(), B[64:].to(dev).contiguous())
    assert torch.equal(t2, t[64:]) and torch.equal(r2, r[64:])
    with pytest.raises(ValueError):                     # track_batch is one launch sequence: n <= max_batch
        rgb, depth, poses, rgbA, depthA = _frame_case(synth, 65, 1)
        eng.track_batch(torch.from_numpy(rgb).to(dev), torch.from_numpy(depth).to(dev), synth.CAMERA_K, torch.from_numpy(poses).to(dev),
                        torch.full((65,), 200.0, dtype=torch.float64, device=dev), torch.from_numpy(rgbA).to(dev),
                        torch.from_numpy(depthA).to(dev), 0.03, 0.0873)


def test_errors_are_reported_not_fatal(pkg, synth, eng):
    L = importlib.import_module('iros20-6d-pose-tracking_b200._lib')
    A, B = synth.tensor_pairs(1, seed=0)
    with pytest.raises(L.Se3tnError) as ei:
        eng.forward(A.to(eng.device), B.to(eng.device), weight_id=7)
    assert ei.value.code == L.ERR_STATE and 'not loaded' in str(ei.value)
    with pytest.raises(ValueError):
        eng.forward(A.to(eng.device)[:, :3].contiguous(), B.to(eng.device))
    # the context is still usable
    eng.forward(A.to(eng.device), B.to(eng.device), weight_id=0)


# ------------------------------------------------------------------------------ metrics (SURVEY 8f row 1)
def test_add_adi_vocap_vs_reference_fixtures(pkg, synth, golden_dir, eng):
    g = np.load(os.path.join(golden_dir, 'golden_metrics.npz'))
    dev = eng.device
    model = synth.model_points(2620, seed=0)
    pred, gt = synth.pose_pairs(12, seed=0)
    pred[0] = gt[0]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    add, adi = eng.add_adi(t(model), t(pred), t(gt))
    assert np.allclose(add.cpu().numpy(), g['add'], rtol=1e-12, atol=1e-15)
    assert np.allclose(adi.cpu().numpy(), g['adi'], rtol=1e-12, atol=1e-15)
    assert float(add[0]) == 0.0 and float(adi[0]) == 0.0
    for k in ('mixed', 'all_below', 'dups', 'single', 'sorted_add'):
        assert abs(eng.vocap(t(g['curve_' + k])) - float(g['vocap_' + k])) < 1e-12, k
    assert eng.vocap(t(np.array([0.5, 0.7]))) == 0.0          # nothing below 0.1 m (the reference raises here)
    # drop-in functions
    U = importlib.import_module('iros20-6d-pose-tracking_b200.Utils')
    EV = importlib.import_module('iros20-6d-pose-tracking_b200.eval_ycb')
    U.set_engine(eng)
    class Cloud:                                              # what callers hand over: anything with .points
        points = model
    assert abs(U.add(pred[3], gt[3], Cloud()) - g['add'][3]) < 1e-14 and abs(U.adi(pred[3], gt[3], model) - g['adi'][3]) < 1e-14
    assert abs(EV.VOCap(g['curve_mixed']) - float(g['vocap_mixed'])) < 1e-12


def test_add_adi_full_size_properties(synth, eng):
    """YCB-Video scale: 14,025 key-frame poses (eval_ycb.py:154) x 2620 model points; properties that hold at any size."""
    dev = eng.device
    model = torch.from_numpy(synth.model_points(2620, seed=1)).to(dev)
    pred, gt = synth.pose_pairs(2048, seed=3)
    pred, gt = torch.from_numpy(pred).to(dev), torch.from_numpy(gt).to(dev)
    add, adi = eng.add_adi(model, pred, gt)
    assert bool((adi <= add + 1e-12).all()) and bool((add >= 0).all())
    add2, adi2 = eng.add_adi(model, gt, pred)                  # ADD is symmetric in (pred, gt)
    assert torch.allclose(add, add2, rtol=1e-12, atol=0)
    T = torch.from_numpy(synth.raw_poses(1, seed=9)[0]).to(dev)   # a common rigid motion leaves both unchanged
    add3, adi3 = eng.add_adi(model, T @ pred, T @ gt)
    assert torch.allclose(add, add3, rtol=1e-9, atol=1e-12) and torch.allclose(adi, adi3, rtol=1e-9, atol=1e-12)
    perm = torch.randperm(2620, generator=torch.Generator().manual_seed(1)).to(dev)
    add4, adi4 = eng.add_adi(model[perm].contiguous(), pred[:64].contiguous(), gt[:64].contiguous())
    assert torch.allclose(add[:64], add4, rtol=1e-12, atol=0) and torch.allclose(adi[:64], adi4, rtol=1e-12, atol=0)
    ap = eng.vocap(adi)
    assert 0.0 <= ap <= 1.0 and abs(ap - O.vocap(adi.cpu().numpy())) < 1e-12


# ------------------------------------------------------------------------------ input A rasteriser (SURVEY 8f row 2)
def _render_both(eng, synth, mesh, poses, width, mesh_id=0):
    dev = eng.device
    eng.set_mesh(mesh, mesh_id)
    ids = torch.full((len(poses),), mesh_id, dtype=torch.int32, device=dev)
    rgb, dep = eng.render(synth.CAMERA_K, torch.from_numpy(poses).to(dev), torch.full((len(poses),), float(width), dtype=torch.float64, device=dev), ids)
    rgb, dep = rgb.cpu().numpy(), dep.cpu().numpy()
    ref = [O.render_window(p, synth.CAMERA_K, float(width), mesh) for p in poses]
    return rgb, dep, np.stack([r[0] for r in ref]), np.stack([r[1] for r in ref])


def test_render_bit_exact_vs_oracle(pkg, synth, eng):
    """float64 + exact integer edge functions on both sides: the CUDA rasteriser must reproduce the numpy restatement bit for bit
    (coverage, depth in mm, 8-bit colour), dense mesh and coarse mesh (warp-cooperative large triangles) alike."""
    poses = synth.raw_poses(5, seed=11)
    poses[4] = np.eye(4); poses[4, :3, 3] = (0.0, 0.0, 0.45)
    for level, mid in ((3, 0), (0, 1), (1, 2)):
        mesh = synth.mesh(level, seed=level)
        rgb, dep, rrgb, rdep = _render_both(eng, synth, mesh, poses, 200.0, mid)
        assert (dep > 0).sum() > 5000
        assert np.array_equal(dep, rdep), 'level %d: %d depth pixels differ' % (level, (dep != rdep).sum())
        assert np.array_equal(rgb, rrgb), 'level %d: %d colour values differ' % (level, (rgb != rrgb).sum())


def test_render_near_plane_clipping_bit_exact(pkg, synth, eng):
    """Models that pass through the eye plane: triangles with vertices at w <= 0 are cut at the near plane (homogeneous path in
    render.cu) -- same pixels, depths and colours as the numpy restatement, whose clipped surface tests/test_oracle_golden.py
    checks against ray casting."""
    import cv2
    K = synth.CAMERA_K
    poses = []
    for rvec, tr in (((0.05, 0.02, 0.1), (0.045, 0.0, 0.45)), ((0.0, 0.08, 0.5), (0.045, 0.0, 0.45)), ((0.1, -0.05, 1.0), (0.06, 0.0, 0.45)),
                     ((0.3, 0.2, 0.1), (0.02, -0.01, 0.45)), ((1.2, 0.1, -0.4), (0.0, 0.04, 0.4))):
        p = np.eye(4); p[:3, :3] = cv2.Rodrigues(np.array(rvec))[0]; p[:3, 3] = tr
        poses.append(p)
    poses = np.stack(poses)
    for level, mid in ((1, 4), (2, 5)):
        mesh = dict(synth.mesh(level, seed=2))
        mesh['pos'] = (mesh['pos'] * np.array([1.0, 1.0, 24.0], np.float32)).astype(np.float32)
        zcam = mesh['pos'].astype(np.float64) @ poses[0][2, :3] + poses[0][2, 3]
        assert zcam.min() < -0.05 and zcam.max() > 0.8
        rgb, dep, rrgb, rdep = _render_both(eng, synth, mesh, poses, 200.0, mid)
        assert (dep > 0).sum() > 5000
        assert np.array_equal(dep, rdep), 'level %d: %d depth pixels differ' % (level, (dep != rdep).sum())
        assert np.array_equal(rgb, rrgb), 'level %d: %d colour values differ' % (level, (rgb != rrgb).sum())


def test_render_pyrender_mode_bit_exact_vs_oracle(pkg, synth, eng):
    """The reference's other producer of input A (dataset_info['renderer'] == 'pyrenderer': offscreen_renderer.py:77-83, then
    crop_bbox, predict.py:210-214).  The oracle literally renders the whole 480 x 640 camera image and crops it; the CUDA
    rasteriser shades only the camera pixels crop_bbox's nearest-neighbour resize picks -- same bytes, for windows that are
    enlarged (far object), reduced (near object), hang over the image border, and for a model crossing the near plane."""
    import cv2
    K, H, W = synth.CAMERA_K, 480, 640
    poses = synth.raw_poses(4, seed=11)
    poses[0, :3, 3] = (0.05, -0.04, 0.33)           # near: window larger than 176 px -> the resize skips camera pixels
    poses[1, :3, 3] = (-0.08, 0.06, 1.4)            # far: window smaller than 176 px -> camera pixels are repeated
    poses[2, :3, 3] = (0.13, -0.09, 0.55)           # window hangs over the right / top border of the camera image
    for level, mid in ((2, 6), (1, 7)):
        mesh = synth.mesh(level, seed=level)
        eng.set_mesh(mesh, mid)
        dev = eng.device
        ids = torch.full((len(poses),), mid, dtype=torch.int32, device=dev)
        ow = torch.full((len(poses),), 200.0, dtype=torch.float64, device=dev)
        rgb, dep = eng.render(K, torch.from_numpy(poses).to(dev), ow, ids, mode='pyrender', image_hw=(H, W))
        rgb, dep = rgb.cpu().numpy(), dep.cpu().numpy()
        for i, p in enumerate(poses):
            rr, rd = O.render_window_pyrender(p, K, 200.0, mesh, H, W)
            assert np.array_equal(dep[i], rd), 'level %d pose %d: %d depth pixels differ' % (level, i, (dep[i] != rd).sum())
            assert np.array_equal(rgb[i], rr), 'level %d pose %d: %d colour values differ' % (level, i, (rgb[i] != rr).sum())
        assert (dep > 0).sum() > 4000
        # not the vispy-style image: unlit colours, another depth linearisation
        lit, _ = eng.render(K, torch.from_numpy(poses).to(dev), ow, ids)
        assert not np.array_equal(lit.cpu().numpy(), rgb)
    # near-plane straddlers through the same mode
    mesh = dict(synth.mesh(1, seed=2))
    mesh['pos'] = (mesh['pos'] * np.array([1.0, 1.0, 24.0], np.float32)).astype(np.float32)
    eng.set_mesh(mesh, 8)
    p = np.eye(4); p[:3, :3] = cv2.Rodrigues(np.array((0.05, 0.02, 0.1)))[0]; p[:3, 3] = (0.045, 0.0, 0.45)
    rgb, dep = eng.render(K, torch.from_numpy(p[None]).to(eng.device), torch.full((1,), 200.0, dtype=torch.float64, device=eng.device),
                          torch.full((1,), 8, dtype=torch.int32, device=eng.device), mode='pyrender', image_hw=(H, W))
    rr, rd = O.render_window_pyrender(p, K, 200.0, mesh, H, W)
    assert np.array_equal(dep[0].cpu().numpy(), rd) and np.array_equal(rgb[0].cpu().numpy(), rr) and (rd > 0).sum() > 3000
    with pytest.raises(ValueError):
        eng.render(K, torch.from_numpy(p[None]).to(eng.device), torch.full((1,), 200.0, dtype=torch.float64, device=eng.device), mode='pyrender')


def test_tracker_selects_the_pyrender_style_renderer(pkg, synth, tmp_path):
    """dataset_info['renderer'] == 'pyrenderer' with a .obj model (predict.py:161-164): Tracker builds the CUDA rasteriser in
    its full-camera-image mode, and on_track(prev_pose, rgb, depth) equals the oracle fed with the oracle's render."""
    mesh = synth.mesh(2, seed=4)
    obj = str(tmp_path / 'model.obj')
    with open(obj, 'w') as f:
        for v, c in zip(mesh['pos'], mesh['col']):
            f.write('v %.9g %.9g %.9g %.9g %.9g %.9g\n' % (*v, *(c / 255.0)))
        for t in mesh['faces']:
            f.write('f %d %d %d\n' % tuple(t + 1))
    sd = synth.make_state_dict(0)
    mean, std = synth.default_mean_std()
    K = synth.CAMERA_K
    info = {'resolution': 176, 'boundingbox': 10, 'object_width': 200.0, 'renderer': 'pyrenderer',
            'camera': {'focalX': K[0, 0], 'focalY': K[1, 1], 'centerX': K[0, 2], 'centerY': K[1, 2], 'height': 480, 'width': 640}}
    trk = pkg.Tracker(info, mean, std, {'state_dict': sd}, model_path=obj, max_batch=4)
    assert type(trk.renderer).__name__ == 'CudaRenderer' and trk.renderer.mode == 'pyrender' and trk.renderer.image_hw == (480, 640)
    loaded = trk.renderer.mesh
    # vertices come out in order of first use by a face; the triangles are the same ones
    assert np.array_equal(loaded['pos'][loaded['faces']], mesh['pos'][mesh['faces']]) and np.array_equal(loaded['col'][loaded['faces']], mesh['col'][mesh['faces']])
    rgb, depth = synth.raw_frame(9)
    pose = synth.raw_poses(2, seed=9)[1]
    ra, da = trk.render_window(pose)
    ora, oda = O.render_window_pyrender(pose, K, 200.0, loaded, 480, 640)
    assert np.array_equal(ra, ora) and np.array_equal(da, oda) and (da > 0).sum() > 1000
    got = trk.on_track(pose, rgb, depth)
    ref = O.on_track(sd, pose, rgb, depth, ora, oda, K, 200.0, mean, std)
    assert np.abs(got - ref).max() < POSE_ATOL


def test_render_edge_cases(pkg, synth, eng):
    dev = eng.device
    mesh = synth.mesh(2, seed=0)
    eng.set_mesh(mesh, 0)
    K = synth.CAMERA_K
    poses = synth.raw_poses(3, seed=5)
    P = torch.from_numpy(poses).to(dev)
    # zero width -> degenerate window -> empty images (the reference would divide by zero in update_cam_mat)
    rgb, dep = eng.render(K, P, torch.zeros(3, dtype=torch.float64, device=dev))
    assert int(rgb.max()) == 0 and int(dep.to(torch.int32).max()) == 0
    # object beyond the far plane (2 m) is clipped away; behind the camera likewise
    far = poses.copy(); far[:, 2, 3] = 2.5; far[2, 2, 3] = -0.7
    rgb, dep = eng.render(K, torch.from_numpy(far).to(dev), torch.full((3,), 200.0, dtype=torch.float64, device=dev))
    assert int(dep.to(torch.int32).max()) == 0 and int(rgb.max()) == 0
    # per-track models in one launch, n == 0, unknown mesh id falls back to model 0
    eng.set_mesh(synth.mesh(1, seed=1), 3)
    ids = torch.tensor([0, 3, 0], dtype=torch.int32, device=dev)
    w = torch.full((3,), 200.0, dtype=torch.float64, device=dev)
    rgb, dep = eng.render(K, P, w, ids)
    r1 = O.render_window(poses[1], K, 200.0, synth.mesh(1, seed=1))
    assert np.array_equal(dep[1].cpu().numpy(), r1[1]) and np.array_equal(rgb[1].cpu().numpy(), r1[0])
    r0 = O.render_window(poses[2], K, 200.0, mesh)
    assert np.array_equal(dep[2].cpu().numpy(), r0[1])
    e_rgb, e_dep = eng.render(K, P[:0], w[:0])
    assert e_rgb.shape == (0, 176, 176, 3) and e_dep.shape == (0, 176, 176)


def test_render_feeds_track_batch(pkg, synth, eng):
    """Device-resident loop: render -> K0 -> network -> K6 equals the oracle driven with the oracle's own render."""
    dev = eng.device
    mesh = synth.mesh(3, seed=0)
    eng.set_mesh(mesh, 0)
    n = 4
    rgb, depth = synth.raw_frame(seed=2)
    poses = synth.raw_poses(n, seed=6)
    K = synth.CAMERA_K
    w = torch.full((n,), 200.0, dtype=torch.float64, device=dev)
    P = torch.from_numpy(poses).to(dev)
    rgbA, depA = eng.render(K, P, w)
    out_poses, _, _ = eng.track_batch(torch.from_numpy(rgb).to(dev), torch.from_numpy(depth).to(dev), K, P, w, rgbA, depA,
                                      0.03, 5 * np.pi / 180)
    mean, std = synth.default_mean_std()
    sd = synth.make_state_dict(0)
    for i in range(n):
        ra, da = O.render_window(poses[i], K, 200.0, mesh)
        ref = O.on_track(sd, poses[i], rgb, depth, ra, da, K, 200.0, mean, std, 0.03, 5 * np.pi / 180)
        assert np.abs(out_poses[i].cpu().numpy() - ref).max() < POSE_ATOL


def test_tracker_with_cuda_renderer(pkg, synth, tmp_path):
    """The reference's loop shape -- Tracker(model_path=*.ply) ; on_track(prev_pose, rgb, depth) renders input A itself
    (predict.py:229-231) -- with the CUDA rasteriser standing in for VispyRenderer."""
    mio = importlib.import_module('iros20-6d-pose-tracking_b200.mesh_io')
    mesh = synth.mesh(3, seed=0)
    ply = str(tmp_path / 'textured.ply')
    mio.save_ply_mesh(ply, mesh)
    mesh = mio.load_ply_mesh(ply)                                   # what both sides see (normals re-normalised on load)
    info = {'resolution': 176, 'object_width': 200.0, 'boundingbox': 10,
            'camera': {'focalX': synth.CAMERA_K[0, 0], 'focalY': synth.CAMERA_K[1, 1], 'centerX': synth.CAMERA_K[0, 2], 'centerY': synth.CAMERA_K[1, 2],
                       'height': 480, 'width': 640}}
    mean, std = synth.default_mean_std()
    sd = synth.make_state_dict(0)
    trk = pkg.Tracker(info, mean, std, {'state_dict': sd}, model_path=ply, max_batch=8)
    assert type(trk.renderer).__name__ == 'CudaRenderer' and trk.object_cloud is not None
    rgb, depth = synth.raw_frame(seed=4)
    poses = synth.raw_poses(3, seed=8)
    K = synth.CAMERA_K
    ra, da = trk.render_window(poses[0])
    ora, oda = O.render_window(poses[0], K, 200.0, mesh)
    assert ra.dtype == np.uint8 and da.dtype == np.uint16 and np.array_equal(ra, ora) and np.array_equal(da, oda)
    new = trk.on_track(poses[0], rgb, depth)
    ref = O.on_track(sd, poses[0], rgb, depth, ora, oda, K, 200.0, mean, std, 0.03, 5 * np.pi / 180)
    assert new.shape == (4, 4) and np.abs(new - ref).max() < POSE_ATOL
    # all tracks of a frame, input A rendered on the device
    out = trk.on_track_batch(poses, rgb, depth)
    for i in range(3):
        oa, od = O.render_window(poses[i], K, 200.0, mesh)
        ref = O.on_track(sd, poses[i], rgb, depth, oa, od, K, 200.0, mean, std, 0.03, 5 * np.pi / 180)
        assert np.abs(out[i] - ref).max() < POSE_ATOL
    # a chain of frames stays on the device: poses out -> poses in
    P = torch.from_numpy(poses).cuda(); R = torch.from_numpy(rgb).cuda(); D = torch.from_numpy(depth).cuda()
    for _ in range(3):
        P = trk.on_track_batch(P, R, D)
    assert P.is_cuda and torch.isfinite(P).all()
    trk.engine.close()


def test_headless_sequence_driver(pkg, synth, tmp_path):
    """SURVEY 8f row 3: the reference's on-disk formats end to end -- rgb / depth PNGs, annotated pose txt, dataset_info.yml,
    mean.npy / std.npy, model_best_val.pth.tar, model .ply in; %07d.txt poses out -- against the oracle fed from the same files."""
    import cv2, yaml
    pr = importlib.import_module('iros20-6d-pose-tracking_b200.predict')
    mio = importlib.import_module('iros20-6d-pose-tracking_b200.mesh_io')
    K = synth.CAMERA_K
    seq, train, out = tmp_path / 'bleach0', tmp_path / 'data' / 'train', tmp_path / 'out'
    for d in (seq / 'rgb', seq / 'depth_filled', seq / 'annotated_poses', train):
        d.mkdir(parents=True)
    nframes = 3
    for i in range(nframes):
        rgb, depth = synth.raw_frame(seed=20 + i)
        cv2.imwrite(str(seq / 'rgb' / ('%07d.png' % i)), rgb[..., ::-1])
        cv2.imwrite(str(seq / 'depth_filled' / ('%07d.png' % i)), depth)
    pose0 = synth.raw_poses(1, seed=3)[0]
    np.savetxt(str(seq / 'annotated_poses' / '0000000.txt'), pose0)
    info = {'resolution': 176, 'object_width': 200.0, 'boundingbox': 10,
            'camera': {'focalX': float(K[0, 0]), 'focalY': float(K[1, 1]), 'centerX': float(K[0, 2]), 'centerY': float(K[1, 2]), 'height': 480, 'width': 640}}
    yaml.safe_dump(info, open(tmp_path / 'data' / 'dataset_info.yml', 'w'))
    mean, std = synth.default_mean_std()
    np.save(tmp_path / 'mean.npy', mean); np.save(tmp_path / 'std.npy', std)
    sd = synth.make_state_dict(0)
    torch.save({'epoch': 7, 'state_dict': sd, 'best_prec': 0.0}, str(tmp_path / 'model_best_val.pth.tar'))
    mio.save_ply_mesh(str(tmp_path / 'textured.ply'), synth.mesh(3, seed=0))
    pr.main(['--mode', 'ycbineoat', '--YCBInEOAT_dir', str(seq), '--train_data_path', str(train), '--model_path', str(tmp_path / 'textured.ply'),
             '--ckpt_dir', str(tmp_path / 'model_best_val.pth.tar'), '--mean_std_path', str(tmp_path), '--outdir', str(out)])
    mesh = mio.load_ply_mesh(str(tmp_path / 'textured.ply'))
    prev = pose0.copy()
    for i in range(nframes):
        got = np.loadtxt(str(out / ('%07d.txt' % i)))
        rgb, depth = pr.read_rgb(str(seq / 'rgb' / ('%07d.png' % i))), pr.read_depth(str(seq / 'depth_filled' / ('%07d.png' % i)))
        ra, da = O.render_window(prev, K, 200.0, mesh)
        ref = O.on_track(sd, prev, rgb, depth, ra, da, K, 200.0, mean, std, 0.03, 30 * np.pi / 180)
        assert got.shape == (4, 4) and np.abs(got - ref).max() < 6 * POSE_ATOL, 'frame %d: %.3g' % (i, np.abs(got - ref).max())
        prev = got                                                  # follow the written trajectory, as eval_ycb.py reads it


def test_ycb_video_drivers_on_synthetic_layout(pkg, synth, tmp_path):
    """SURVEY 8f row 3, the YCB-Video half (reference predict.py:299-575): a synthetic data set in the YCB-Video layout (two test
    sequences, keyframe.txt, a PoseCNN result file) through predictSequenceYcb (gt init, then PoseCNN init + a re-initialisation
    frame) and getResultsYcb, every written pose against the oracle fed from the same files."""
    import cv2, scipy.io
    pr = importlib.import_module('iros20-6d-pose-tracking_b200.predict')
    mio = importlib.import_module('iros20-6d-pose-tracking_b200.mesh_io')
    K = synth.CAMERA_K
    ycb = tmp_path / 'ycb'
    cls, nframes = 4, 4
    traj = {}
    for seq in (48, 49):
        base = ycb / 'data_organized' / ('%04d' % seq)
        for d in ('color', 'depth_filled', 'seg', 'pose_gt/%d' % cls):
            (base / d).mkdir(parents=True)
        gt = synth.raw_poses(nframes, seed=seq)
        gt[1:, :3, 3] = gt[0, :3, 3] + 0.002 * np.arange(1, nframes)[:, None]     # a slowly drifting object
        gt[1:, :3, :3] = gt[0, :3, :3]
        traj[seq] = gt
        for i in range(nframes):
            rgb, depth = synth.raw_frame(seed=100 * seq + i)
            cv2.imwrite(str(base / 'color' / ('%06d-color.png' % (i + 1))), rgb[..., ::-1])
            cv2.imwrite(str(base / 'depth_filled' / ('%06d-depth.png' % (i + 1))), depth)
            np.savetxt(str(base / 'pose_gt' / str(cls) / ('%06d.txt' % (i + 1))), gt[i])
    (ycb / 'image_sets').mkdir()
    (ycb / 'image_sets' / 'keyframe.txt').write_text('0048/000001\n0048/000002\n0049/000001\n')
    pc = ycb / 'YCB_Video_toolbox' / 'results_PoseCNN_RSS2018'
    pc.mkdir(parents=True)
    from scipy.spatial.transform import Rotation
    def to_icp(pose):
        q = Rotation.from_matrix(pose[:3, :3]).as_quat()              # x y z w
        return np.r_[q[3], q[0], q[1], q[2], pose[:3, 3]]
    posecnn0 = traj[48][0].copy(); posecnn0[:3, 3] += [0.003, -0.002, 0.004]
    posecnn1 = traj[48][1].copy(); posecnn1[:3, 3] += [-0.002, 0.001, 0.002]
    for idx, pz in ((0, posecnn0), (1, posecnn1), (2, traj[49][0])):
        scipy.io.savemat(str(pc / ('%06d.mat' % idx)), {'rois': np.array([[0, 1, 0, 0, 0, 0], [0, cls, 0, 0, 0, 0]], dtype=np.float64),
                                                        'poses_icp': np.stack([to_icp(np.eye(4)), to_icp(pz)])})
    info = {'resolution': 176, 'object_width': 200.0, 'boundingbox': 10,
            'camera': {'focalX': float(K[0, 0]), 'focalY': float(K[1, 1]), 'centerX': float(K[0, 2]), 'centerY': float(K[1, 2]), 'height': 480, 'width': 640}}
    mean, std = synth.default_mean_std()
    sd = synth.make_state_dict(0)
    ply = str(tmp_path / 'textured.ply')
    mio.save_ply_mesh(ply, synth.mesh(3, seed=0))
    mesh = mio.load_ply_mesh(ply)
    trk = pkg.Tracker(info, mean, std, {'state_dict': sd}, model_path=ply, max_batch=4)

    def oracle_chain(seq, start_pose, reinit=None, start=0):
        base = ycb / 'data_organized' / ('%04d' % seq)
        prev, out = start_pose.copy(), [start_pose.copy()]
        for i in range(start + 1, nframes):
            rgb = pr.read_rgb(str(base / 'color' / ('%06d-color.png' % (i + 1)))); depth = pr.read_depth(str(base / 'depth_filled' / ('%06d-depth.png' % (i + 1))))
            if reinit and i in reinit:
                prev = reinit[i].copy()
            ra, da = O.render_window(prev, K, 200.0, mesh)
            prev = O.on_track(sd, prev, rgb, depth, ra, da, K, 200.0, mean, std, 0.03, 5 * np.pi / 180)
            out.append(prev)
        return np.stack(out)

    # (1) one sequence from its ground-truth pose
    poses, auc = pr.predictSequenceYcb(str(ycb / 'data_organized'), 48, cls, info, mean, std, None, ply, str(tmp_path / 'o1'), init='gt', tracker=trk)
    ref = oracle_chain(48, traj[48][0])
    assert poses.shape == (nframes, 4, 4) and np.abs(poses - ref).max() < 6 * POSE_ATOL
    assert np.allclose(np.loadtxt(str(tmp_path / 'o1' / '00002.txt')), poses[2]) and np.allclose(np.loadtxt(str(tmp_path / 'o1' / '00002gt.txt')), traj[48][2])
    ref_adi = np.array([O.adi(ref[i], traj[48][i], np.asarray(trk.object_cloud.points)) for i in range(nframes)])
    assert auc is not None and abs(auc - O.vocap(ref_adi) * 100) < 0.5

    # (2) PoseCNN initialisation (start_frame 1: keyframe 0048/000001 = result file 0) and a re-initialisation at 0048/000004:
    #     frame index i = 3 restarts from PoseCNN's estimate at the keyframe nearest to 0048/%06d % (i - 1) = 000002 -> file 1
    ycb_root = ycb / 'data_organized'
    for sub in ('image_sets', 'YCB_Video_toolbox'):
        os.symlink(str(ycb / sub), str(ycb_root / sub))              # the reference reads both roots from the same --ycb_dir
    poses2, _ = pr.predictSequenceYcb(str(ycb_root), 48, cls, info, mean, std, None, ply, str(tmp_path / 'o2'), init='posecnn',
                                      reinit_frames=['0048/000004'], start_frame=1, tracker=trk)
    ref2 = oracle_chain(48, posecnn0, reinit={3: posecnn1}, start=1)
    assert poses2.shape == ref2.shape == (nframes - 1, 4, 4) and np.abs(poses2 - ref2).max() < 6 * POSE_ATOL
    assert np.abs(poses2[2] - oracle_chain(48, posecnn0, start=1)[2]).max() > 1e-4      # the re-initialisation really took another path

    # (3) every test sequence of the class (what eval_ycb.py scores)
    res = pr.getResultsYcb(str(ycb), cls, info, mean, std, None, ply, str(tmp_path / 'o3'), tracker=trk)
    assert sorted(res) == [48, 49]
    for seq in (48, 49):
        refq = oracle_chain(seq, traj[seq][0])
        got = np.stack([np.loadtxt(str(tmp_path / 'o3' / ('seq%d' % seq) / ('%07d.txt' % i))) for i in range(nframes)])
        assert np.abs(got - refq).max() < 6 * POSE_ATOL and np.allclose(got, res[seq])

    # (4) eval_ycb.py's scoring of those folders (reference eval_ycb.py:67-119): key frames only, model points from CADmodels/*/points.xyz,
    #     keyframe.txt under YCB_Video_toolbox/ -- against the oracle's ADD / ADD-S / VOCap on the same files
    E = importlib.import_module('iros20-6d-pose-tracking_b200.eval_ycb')
    import argparse, shutil
    pts = np.asarray(trk.object_cloud.points)
    for k in range(1, 6):
        d = ycb / 'CADmodels' / ('%03d_object' % k)
        d.mkdir(parents=True)
        np.savetxt(str(d / 'points.xyz'), pts if k == cls else pts * (1 + 0.1 * k))
    shutil.copy(str(ycb / 'image_sets' / 'keyframe.txt'), str(ycb / 'YCB_Video_toolbox' / 'keyframe.txt'))
    adi_errs, add_errs = E.eval_one_class(argparse.Namespace(res_dir=str(tmp_path / 'o3') + '/', ycb_dir=str(ycb), class_id=cls))
    keyed = [(48, 0), (48, 1), (49, 0)]                              # keyframe.txt above: 0048/000001, 0048/000002, 0049/000001
    want_adi = np.sort([O.adi(res[s][i], traj[s][i], pts) for s, i in keyed])
    want_add = np.sort([O.add(res[s][i], traj[s][i], pts) for s, i in keyed])
    assert adi_errs.shape == (3,) and np.allclose(adi_errs, want_adi, rtol=0, atol=1e-12) and np.allclose(add_errs, want_add, rtol=0, atol=1e-12)
    assert abs(E.VOCap(adi_errs) - O.vocap(want_adi)) < 1e-12
    root = tmp_path / 'all'
    for k in range(1, 22):                                            # eval_all: 21 class folders, each with one run folder
        (root / ('%02d' % k)).mkdir(parents=True)
        os.symlink(str(tmp_path / 'o3'), str(root / ('%02d' % k) / 'run'))
    for k in range(6, 22):
        d = ycb / 'CADmodels' / ('%03d_object' % k)
        d.mkdir(parents=True); np.savetxt(str(d / 'points.xyz'), pts)
        (ycb / 'data_organized' / '0048' / 'pose_gt' / str(k)).mkdir()
    for k in list(range(1, cls)) + list(range(cls + 1, 22)):          # the other classes: same poses as ground truth files
        for seq in (48, 49):
            src = ycb / 'data_organized' / ('%04d' % seq) / 'pose_gt' / str(cls)
            dst = ycb / 'data_organized' / ('%04d' % seq) / 'pose_gt' / str(k)
            dst.mkdir(parents=True, exist_ok=True)
            for f in os.listdir(str(src)):
                shutil.copy(str(src / f), str(dst / f))
    adi_ap, add_ap, total = E.main(['--ycb_dir', str(ycb), '--res_root', str(root), '--expected_total', '63'])
    assert total == 63 and 0.0 <= add_ap <= adi_ap <= 100.0
    trk.engine.close()


# ------------------------------------------------------------------------------ depth hole filling (SURVEY 8f row 4)
def test_fill_depth_vs_reference_and_oracle(pkg, synth, golden_dir, eng):
    """Tolerances: metres within 2e-6 (float32 accumulation order of the bilateral sum; everything before it is bit-exact min /
    max / median); millimetres equal except where the reference's value*1000 sits within 3e-3 of an integer (then +-1), and
    except pixels beyond max_depth, whose negative float -> uint16 conversion is undefined behaviour in the reference itself."""
    g = np.load(os.path.join(golden_dir, 'golden_fill.npz'))
    dev = eng.device
    cases = [(g['in_' + k], g['out_m_' + k], g['out_mm_' + k]) for k in 'ab']
    _, full = synth.raw_frame(seed=9)                               # full 480x640 frame, against the oracle
    full = full.copy(); full[100:160, 200:330] = 0
    mm_ref, m_ref = O.fill_depth_mm(full)
    cases.append((full, m_ref, mm_ref))
    for din, m_ref, mm_ref in cases:
        out_mm, out_m = eng.fill_depth(torch.from_numpy(np.ascontiguousarray(din)).to(dev), want_metres=True)
        out_mm, out_m = out_mm.cpu().numpy(), out_m.cpu().numpy()
        assert np.abs(out_m - m_ref).max() < 2e-6, np.abs(out_m - m_ref).max()
        ok = m_ref >= 0                                             # defined conversions only
        diff = np.abs(out_mm.astype(np.int32) - mm_ref.astype(np.int32))
        assert diff[ok].max() <= 1
        # a millimetre may only differ where the reference's own value sits on a truncation boundary (flat, dilation-filled
        # regions give x.xxx000 +- 1 ulp, and which side OpenCV lands on depends on its SIMD summation order)
        mmf = m_ref.astype(np.float64) * 1000
        on_boundary = np.abs(mmf - np.rint(mmf)) < 3e-3
        assert (on_boundary | (diff == 0) | ~ok).all()
    # drop-in function (metres in, float32 metres out)
    U = importlib.import_module('iros20-6d-pose-tracking_b200.Utils')
    U.set_engine(eng)
    got = U.fill_depth(cases[0][0] / 1e3, max_depth=2.0, extrapolate=False)
    assert got.dtype == np.float32 and np.abs(got - cases[0][1]).max() < 2e-6
    # the reference's optional branches: column extrapolation + 31x31 fill (exact max / copy operations before the blur) and the
    # 5x5 Gaussian blur (float32 [1 4 6 4 1]/16 rows then columns; 2e-6 m covers OpenCV's SIMD summation order), vs the
    # reference's own outputs on the two fixtures and vs the oracle on the full frame
    for tag, ex, blur in (('ex', True, 'bilateral'), ('ga', False, 'gaussian'), ('exga', True, 'gaussian')):
        refs = [g['out_m_%s_%s' % (k, tag)] for k in 'ab'] + [O.fill_depth(full / 1e3, 2.0, extrapolate=ex, blur_type=blur)]
        for (din, _, _), ref in zip(cases, refs):
            _, om = eng.fill_depth(torch.from_numpy(np.ascontiguousarray(din)).to(dev), want_metres=True, extrapolate=ex, blur_type=blur)
            assert np.abs(om.cpu().numpy() - ref).max() < 2e-6, (tag, np.abs(om.cpu().numpy() - ref).max())
    got = U.fill_depth(cases[0][0] / 1e3, extrapolate=True, blur_type='gaussian')
    assert np.abs(got - g['out_m_a_exga']).max() < 2e-6
    with pytest.raises(ValueError):
        U.fill_depth(cases[0][0] / 1e3, blur_type='box')
    # a constant image passes through the bilateral untouched (OpenCV copies when max - min < eps) and nothing is invented
    # (800 mm comes back as 799: 2 - float32(0.8) and back is 0.79999995 -- the reference's own round trip)
    flat = np.full((32, 48), 800, dtype=np.uint16)
    assert np.array_equal(eng.fill_depth(torch.from_numpy(flat).to(dev)).cpu().numpy(), O.fill_depth_mm(flat)[0])
    zero = torch.zeros((16, 16), dtype=torch.uint16, device=dev)
    assert int(eng.fill_depth(zero).to(torch.int32).max()) == 0
