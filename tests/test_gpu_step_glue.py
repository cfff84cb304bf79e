"""GPU: the fp64 / fp32 glue either side of the conv stack, bit for bit against the CPU restatements, at every launch shape
a tracking or validation step uses.

K0 (preprocess_kernel) picks its launch from the batch: 11 rows per CTA and 256 threads below 32 tracks, 22 rows below 64,
88 rows and 1024 threads from 64 on.  Its crops, NCHW tensors and the stem buffers X0A / X0B of every precision mode are
compared with crop_bbox, processData and layer_ref.encode at n = 1, 31, 32, 63, 64, 65 and 200, on a frame and views
holding every raw depth 0..2100, 65535 and every 8-bit colour, for the windows of test_step_glue_cpu.SPECIAL_TRACKS.

K6 (pose_update_one: fused into head_pooled_kernel, stand-alone in pose_update_kernel) against process_predict_exact,
whose float32 steps move the pose by less than 1e-7: only bits can show them (test_step_glue_cpu.py)."""
import cv2
import numpy as np
import pytest
import torch
import layer_ref as R
import se3_oracle as O
from test_step_glue_cpu import (K, TN, RN, NORMALIZERS, SPECIAL_TRACKS, assert_pose_update_equal, edge_frame, edge_views,
                                near_pi_cases, oracle_crop, pose_update_cases, step_tracks)

pytestmark = pytest.mark.gpu
MODES = ('fp32', 'tf32', 'bf16x3', 'bf16', 'fp16', 'fp8')
# the stem input's format (storage.cuh stem_input_prec): the bf16x3 split in the 2-byte modes and fp8
STEM_FMT = {'fp32': 'fp32', 'tf32': 'tf32', 'bf16x3': 'stem_hilo', 'bf16': 'stem_hilo', 'fp16': 'stem_hilo', 'fp8': 'stem_hilo'}
K0_BATCHES = (1, 31, 32, 63, 64, 65, 200)
STEM_BYTES = 182 * 184 * 16


def stats(synth, w, dtype):
    mean, std = synth.default_mean_std()
    if w == 1:
        mean, std = mean + 1.5, std * 1.25
    return mean.astype(dtype), std.astype(dtype)


def set_stats(e, synth, dtype):
    for w in (0, 1):
        e.set_stats(*stats(synth, w, dtype), w)


@pytest.fixture(scope='module')
def eng(pkg, synth):
    e = pkg.Engine(max_batch=200)
    for w in (0, 1):
        e.load_state_dict(synth.make_state_dict(w), w)
    yield e
    e.close()


def dev(e, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(e.device)


def stem_bytes(e, x):
    """(n,4,176,176) float32 -> {format: (n, STEM_BYTES) uint8 CUDA tensor}: layer_ref.encode of each image zero-padded by 3
    pixels top, left and bottom and 5 right, as X0A / X0B hold it."""
    out = {}
    pad = np.zeros((4, 182, 184), np.float32)
    for fmt in set(STEM_FMT.values()):
        b = np.empty((len(x), STEM_BYTES), np.uint8)
        for i in range(len(x)):
            pad[:, 3:179, 3:179] = x[i]
            b[i] = R.encode(pad, 'X0A', fmt)
        out[fmt] = dev(e, b)
    return out


def diff_report(got, want, shape, names):
    """Where got != want (CUDA tensors viewed as `shape`): the count and the first few positions."""
    d = (got.reshape(shape) != want.reshape(shape))
    while d.dim() > len(names.split(',')):
        d = d.any(-1)
    return '%d differ, first %s %s' % (int(d.sum()), names, d.nonzero()[:8].tolist())


def assert_same(got, want, shape, names, what):
    if not torch.equal(got, want):
        raise AssertionError('%s: %s' % (what, diff_report(got, want, shape, names)))


def bits(t):
    return t.contiguous().view(torch.int32)


def assert_stems(e, n, stems, mode, what):
    for buf, (name, want) in enumerate((('X0A', stems[0]), ('X0B', stems[1]))):
        got = e.debug_buffer(buf, n).view(torch.uint8).reshape(n, STEM_BYTES)
        assert_same(got, want[STEM_FMT[mode]][:n], (n, 182, 184, 16), '(image, y, x)', '%s, %s %s' % (what, mode, name))


# ------------------------------------------------------------------------------------------- K0
@pytest.fixture(scope='module')
def k0_tracks(synth):
    """200 tracks of one crafted frame, and the crops of each track's window as crop_bbox (or its index form) cuts them."""
    rgb, depth = edge_frame(seed=0)
    poses, widths, ids, labels = step_tracks(200, seed=0)
    rgbA, depthA = edge_views(200, seed=1)
    crops = [oracle_crop(rgb, depth, p, w) for p, w in zip(poses, widths)]
    return dict(rgb=rgb, depth=depth, poses=poses, widths=widths, ids=ids, labels=labels, rgbA=rgbA, depthA=depthA,
                crop_rgb=np.stack([c[0] for c in crops]), crop_depth=np.stack([c[1] for c in crops]))


def test_k0_windows_equal_the_crop_kernel(eng, k0_tracks):
    """The oracle side of the windows K0 is held to: compute_bbox as the device forms it, and crop_kernel (int indices)
    cutting the same crops, the windows wider than crop_bbox's canvas included."""
    T = k0_tracks
    bbs = eng.compute_bbox(dev(eng, T['poses']), K, dev(eng, T['widths']))
    want = np.stack([O.compute_bbox(p, K, w, scale=(1000, 1000, 1000)) for p, w in zip(T['poses'], T['widths'])])
    assert np.array_equal(bbs.cpu().numpy(), want)
    crgb, cdepth = eng.crop_bbox(dev(eng, T['rgb']), dev(eng, T['depth']), bbs)
    assert_same(crgb, dev(eng, T['crop_rgb']), (200, 176, 176, 3), '(track, y, x)', 'crop_kernel rgb')
    assert_same(cdepth, dev(eng, T['crop_depth']), (200, 176, 176), '(track, y, x)', 'crop_kernel depth')


@pytest.mark.parametrize('dtype', [np.float32, np.float64], ids=['f32_stats', 'f64_stats'])
def test_k0_every_launch_shape_bit_exact(eng, synth, k0_tracks, dtype):
    T = k0_tracks
    set_stats(eng, synth, dtype)
    tens = [O.process_data(T['rgbA'][i], T['depthA'][i], T['poses'][i], T['crop_rgb'][i], T['crop_depth'][i], np.eye(4),
                           *stats(synth, int(T['ids'][i]), dtype))[0] for i in range(200)]
    wantA, wantB = np.stack([t[0] for t in tens]), np.stack([t[1] for t in tens])
    stems = stem_bytes(eng, wantA), stem_bytes(eng, wantB)
    wantA, wantB = bits(dev(eng, wantA)), bits(dev(eng, wantB))
    want_rgb, want_depth = dev(eng, T['crop_rgb']), dev(eng, T['crop_depth'])
    frame_rgb, frame_depth, poses, widths, rgbA, depthA, ids = (dev(eng, T[k]) for k in ('rgb', 'depth', 'poses', 'widths', 'rgbA',
                                                                                         'depthA', 'ids'))
    for n in K0_BATCHES:
        for mode in MODES:
            tA, tB, crgb, cdepth = eng.preprocess(frame_rgb, frame_depth, K, poses[:n], widths[:n], rgbA[:n], depthA[:n],
                                                  weight_ids=ids[:n], precision=mode, want_tensors=True, want_crops=True)
            what = 'n=%d %s (tracks: %s)' % (n, mode, ', '.join(T['labels'][:min(n, len(SPECIAL_TRACKS))]))
            assert_same(crgb, want_rgb[:n], (n, 176, 176, 3), '(track, y, x)', 'K0 rgb crop, ' + what)
            assert_same(cdepth, want_depth[:n], (n, 176, 176), '(track, y, x)', 'K0 depth crop, ' + what)
            assert_same(bits(tA), wantA[:n], (n, 4, 176, 176), '(track, channel, y, x)', 'K0 tensor A, ' + what)
            assert_same(bits(tB), wantB[:n], (n, 4, 176, 176), '(track, channel, y, x)', 'K0 tensor B, ' + what)
            assert_stems(eng, n, stems, mode, 'K0 ' + what)


def test_precropped_and_nchw_stems_bit_exact(eng, synth):
    """normalize (K0 on crops: TrackDataset.processData) and forward(A, B) (nchw_to_stem) write the stem buffers of every
    mode exactly as layer_ref.encode does, at n = 1, 40 and 64 (the three K0 launch shapes)."""
    n_max = 64
    rgbA, depthA = edge_views(n_max, seed=3)
    rgbB, depthB = edge_views(n_max, seed=4)
    poses = synth.raw_poses(n_max, seed=5)
    poses[::3, 2, 3] *= -1                                     # GL poses: the depth offset adds z * 1000
    ids = np.random.default_rng(5).integers(0, 2, n_max).astype(np.int32)
    d = [dev(eng, a) for a in (rgbA, depthA, rgbB, depthB, poses, ids)]
    for dtype in (np.float32, np.float64):
        set_stats(eng, synth, dtype)
        tens = [O.process_data(rgbA[i], depthA[i], poses[i], rgbB[i], depthB[i], np.eye(4), *stats(synth, int(ids[i]), dtype))[0]
                for i in range(n_max)]
        wantA, wantB = np.stack([t[0] for t in tens]), np.stack([t[1] for t in tens])
        stems = stem_bytes(eng, wantA), stem_bytes(eng, wantB)
        wantA, wantB = bits(dev(eng, wantA)), bits(dev(eng, wantB))
        for n in (1, 40, 64):
            for mode in MODES:
                tA, tB = eng.normalize(*(x[:n] for x in d[:5]), weight_ids=d[5][:n], precision=mode)
                what = 'normalize n=%d %s %s stats' % (n, mode, np.dtype(dtype).name)
                assert_same(bits(tA), wantA[:n], (n, 4, 176, 176), '(track, channel, y, x)', what + ', tensor A')
                assert_same(bits(tB), wantB[:n], (n, 4, 176, 176), '(track, channel, y, x)', what + ', tensor B')
                assert_stems(eng, n, stems, mode, what)
    set_stats(eng, synth, np.float32)
    A, B = synth.tensor_pairs(n_max, seed=7)
    # rounding ties of both stem encodings: tf32 (13 dropped bits = 0x1000) and bf16 (16 dropped bits = 0x8000), both signs
    for img, low, mask in ((A, 0x1000, 0x1FFF), (B, 0x8000, 0xFFFF)):
        u = img[:4, :, :8].numpy().view(np.uint32)
        u[:] = (u & ~np.uint32(mask)) | np.uint32(low)
    A, B = A.to(eng.device), B.to(eng.device)
    stems = stem_bytes(eng, A.cpu().numpy()), stem_bytes(eng, B.cpu().numpy())
    eng.calibrate_fp8(A, B, weight_id=0)
    for n in (1, 40, 64):
        for mode in MODES:
            eng.forward(A[:n], B[:n], weight_id=0, precision=mode)
            assert_stems(eng, n, stems, mode, 'forward n=%d' % n)


# ------------------------------------------------------------------------------------------- K6
def test_k6_in_the_tracking_step_is_process_predict_exact(eng, synth):
    """The poses track_batch returns equal process_predict_exact of its input poses and its own 6-vectors, bit for bit:
    K6 fused into the head (bf16x3, fp16; n = 4 runs the split-K trunk) and stand-alone (fp32)."""
    set_stats(eng, synth, np.float32)
    rgb, depth = synth.raw_frame(21)
    poses = synth.raw_poses(200, seed=21)
    rgbA, depthA = synth.rendered_views(200, poses, seed=21)
    ids = np.random.default_rng(21).integers(0, 2, 200).astype(np.int32)
    d = [dev(eng, a) for a in (rgb, depth, poses, np.full(200, 200.0), rgbA, depthA)]
    for n in (1, 4, 64, 200):
        for mode in ('bf16x3', 'fp16', 'fp32'):
            out, tr, ro = eng.track_batch(d[0], d[1], K, d[2][:n], d[3][:n], d[4][:n], d[5][:n], TN, RN, weight_ids_host=ids[:n],
                                          precision=mode)
            tr, ro = tr.cpu().numpy(), ro.cpu().numpy()
            assert np.isfinite(tr).all() and np.isfinite(ro).all() and np.abs(ro).max() > 0
            want = O.process_predict_exact(poses[:n], tr, ro, TN, RN)
            assert_pose_update_equal(out.cpu().numpy(), want, ro, RN, 'track_batch n=%d %s' % (n, mode))


@pytest.mark.parametrize('tn,rn', NORMALIZERS)
def test_k6_pose_update_is_process_predict_exact(eng, tn, rn):
    A, tr, ro = pose_update_cases()
    out = eng.pose_update(dev(eng, A), dev(eng, tr), dev(eng, ro), tn, rn).cpu().numpy()
    assert_pose_update_equal(out, O.process_predict_exact(A, tr, ro, tn, rn), ro, rn, 'pose_update')
    assert np.array_equal(out[0, :3, :3], A[0, :3, :3])                   # rot = 0: the identity branch leaves R as it is


# ------------------------------------------------------------------------------------------- K5 and the loss
def test_so3_log_near_pi_keeps_cv2_sign(eng):
    """Angles pi - delta straddling the small-sine branch, every octant and the six half-axes: the label equals
    cv2.Rodrigues of the column-normalised matrix, sign included (a rotation by pi - delta about -a is not one about a)."""
    ws, deltas = near_pi_cases()
    A = np.tile(np.eye(4), (len(ws), 1, 1)); B = A.copy()
    B[:, :3, :3] = np.stack([cv2.Rodrigues(w)[0] for w in ws])
    _, rl = eng.so3_log(dev(eng, A), dev(eng, B), 1.0, 1.0)
    rl = rl.cpu().numpy()
    ref = np.stack([cv2.Rodrigues(O.normalize_rotation_matrix(B[i, :3, :3].copy()))[0].ravel() for i in range(len(ws))])
    err = np.abs(rl - ref).max(axis=1)
    assert (err < 1e-7).all(), [(ws[i].tolist(), deltas[i], rl[i].tolist(), ref[i].tolist()) for i in np.nonzero(err >= 1e-7)[0][:6]]


def test_loss_sums_past_one_pass_of_the_reduction(pkg, synth):
    """n = 300 pairs: thread t of reduce_loss_terms adds pairs t and t + 256.  The step's sums equal se3tn_pair_loss's bit for
    bit and the float64 sum of its own terms to 1e-6."""
    n = 300
    e = pkg.Engine(max_batch=n)
    try:
        e.load_state_dict(synth.make_state_dict(0), 0)
        e.set_stats(*synth.default_mean_std(), 0)
        A, B = synth.pose_pairs(n, seed=31)
        rgbA, depthA = synth.rendered_views(n, A, seed=31)
        rgbB, depthB = synth.rendered_views(n, B, seed=32)
        args = [dev(e, a) for a in (rgbA, depthA, rgbB, depthB, A, B)]
        for mode in ('bf16x3', 'fp32'):
            tr, ro, sums, sq, lab = e.eval_pairs(*args, TN, RN, precision=mode, want_terms=True, want_labels=True)
            lab_np = lab.cpu().numpy()
            six = torch.cat((tr, ro), 1).cpu().numpy()
            expect = np.square(six - lab_np.astype(np.float32))
            assert np.array_equal(sq.cpu().numpy(), expect), mode
            s2 = e.pair_loss(tr, ro, lab[:, :3].contiguous(), lab[:, 3:].contiguous())
            assert torch.equal(sums, s2), mode
            f64 = [expect[:, :3].sum(dtype=np.float64), expect[:, 3:].sum(dtype=np.float64)]
            np.testing.assert_allclose(sums.cpu().numpy(), f64, rtol=1e-6, err_msg=mode)
            head = e.eval_pairs(*(a[:256] for a in args), TN, RN, precision=mode)[2].cpu().numpy()
            assert (sums.cpu().numpy() > head).all(), mode                 # the 44 pairs past the first pass are counted
    finally:
        e.close()
