"""Pose recovery from perturbed starts on the YCB-Video key frames (predict.recoverYcbKeyframes, se3tn_track_render's round_poses,
se3tn_pose_errors_sets) on a synthetic layout of 120 x 160 frames and three classes with their own checkpoints, statistics and
normalisers:

  * the kept rows of each class are the pairs `produce_train_pair_data --mode ycbv` writes (count, order, A_in_cam / B_in_cam bit
    for bit) and random / np.random end in the same state
  * every round of a K = 3 step equals an r-round step bit for bit in bf16x3, bf16, fp8 and fp32, at n <= 4 (split-K latency
    mode) and n > 4; the step with the round output gives the step's own final poses, and replays its graph on a second frame
  * se3tn_pose_errors_sets against numpy (0 and near-180 degree rows included), its ADD / ADD-S against se3tn_add_adi_sets, and
    masked rows left out
  * the AUCs are the eval_ycb VOCap drop-in's, round 0 is A_in_cam scored against B_in_cam
  * two checkpoints x two modes in one pass give each variant's run alone bit for bit; a class with no kept row reports 0 rows
"""
import glob
import importlib
import os
import random

import cv2
import numpy as np
import pytest
import torch
import yaml

import se3_oracle as O

pytestmark = pytest.mark.gpu
PKG = 'iros20-6d-pose-tracking_b200'
H, W = 120, 160
CLASSES = (2, 3, 5)
NUM_SAMPLE, SEED, K = 6, 4, 3


@pytest.fixture(scope='module')
def mods():
    return {k: importlib.import_module(PKG + '.' + k) for k in ('produce_train_pair_data', 'predict', 'engine', '_lib', 'mesh_io',
                                                                 'eval_ycb')}


@pytest.fixture(scope='module')
def layout(synth, mods, tmp_path_factory):
    """<root>/ycb: 6 key frames of sequence 0048; class 2 near the left edge (centre rejections), class 3 not annotated in frame 2,
    class 5 reduced to a 25-pixel patch in frame 4 (rejected by the visibility check), class 7 annotated everywhere but never
    labelled (no kept row).  <root>/cfg/c<id>: dataset_info.yml, mesh, two checkpoints, mean.npy / std.npy."""
    root = tmp_path_factory.mktemp('recover')
    ycb, cfg = root / 'ycb', root / 'cfg'
    Kc = synth.CAMERA_K.copy(); Kc[:2] *= 0.25
    cam = {'focalX': float(Kc[0, 0]), 'focalY': float(Kc[1, 1]), 'centerX': float(Kc[0, 2]), 'centerY': float(Kc[1, 2]), 'height': H, 'width': W}
    meshes = {c: synth.mesh(2, seed=c) for c in CLASSES + (7,)}
    gt = {}
    for c, t, s in ((2, (-0.13, 0.02, 0.5), 3), (3, (0.02, -0.01, 0.6), 4), (5, (0.05, 0.03, 0.55), 5), (7, (0.0, 0.0, 0.6), 6)):
        gt[c] = synth.raw_poses(1, seed=s)[0]; gt[c][:3, 3] = t
    mean, std = synth.default_mean_std()
    for k, c in enumerate(CLASSES + (7,)):
        d = cfg / ('c%d' % c)
        (d / 'train').mkdir(parents=True)
        info = {'resolution': 176, 'object_width': 200.0 + 10 * k, 'boundingbox': 10, 'max_translation': 0.04 + 0.01 * k,
                'max_rotation': 15.0 + 5 * k, 'camera': cam}
        yaml.safe_dump(info, open(d / 'dataset_info.yml', 'w'))
        mods['mesh_io'].save_ply_mesh(str(d / 'textured.ply'), meshes[c])
        torch.save({'state_dict': synth.make_state_dict(10 + c)}, str(d / 'ckpt_a.pth.tar'))
        torch.save({'state_dict': synth.make_state_dict(50 + c)}, str(d / 'ckpt_b.pth.tar'))
        np.save(str(d / 'mean.npy'), mean + k); np.save(str(d / 'std.npy'), std * (1 + 0.1 * k))
    for k in range(1, 22):
        (ycb / 'CADmodels' / ('%03d_obj' % k)).mkdir(parents=True)
    base = ycb / 'data_organized' / '0048'
    for d in ['color', 'depth_filled', 'seg'] + ['pose_gt/%d' % c for c in CLASSES + (7,)]:
        (base / d).mkdir(parents=True)
    Kd = np.array([[cam['focalX'], 0, cam['centerX']], [0, cam['focalY'], cam['centerY']], [0, 0, 1]], np.float32).astype(np.float64)
    for i in range(6):
        rgb, depth = synth.raw_frame(40 + i, H, W)
        seg = np.zeros((H, W), np.uint8)
        for c in CLASSES:
            _, dd = O.render_full_frame_unlit(gt[c], Kd, meshes[c], H, W)
            if c == 5 and i == 3:
                ys, xs = np.nonzero(dd > 0)
                seg[ys[0]:ys[0] + 5, xs[0]:xs[0] + 5] = c
            else:
                seg[dd > 0] = c
        cv2.imwrite(str(base / 'color' / ('%06d-color.png' % (i + 1))), rgb[..., ::-1])
        cv2.imwrite(str(base / 'depth_filled' / ('%06d-depth.png' % (i + 1))), depth)
        cv2.imwrite(str(base / 'seg' / ('%06d-label.png' % (i + 1))), seg)
        for c in CLASSES + (7,):
            if not (c == 3 and i == 1):
                np.savetxt(str(base / 'pose_gt' / str(c) / ('%06d.txt' % (i + 1))), gt[c])
    (ycb / 'image_sets').mkdir()
    (ycb / 'image_sets' / 'keyframe.txt').write_text(''.join('0048/%06d\n' % (i + 1) for i in range(6)))
    c_dir = str(cfg / 'c{class_id}')
    tpl = {'train_data_path': c_dir + '/train', 'model_path': c_dir + '/textured.ply', 'pair_model_path': c_dir + '/textured.ply',
           'ckpt_dir': c_dir + '/ckpt_a.pth.tar', 'mean_std_path': c_dir,
           'trans_normalizer': 0.05, 'rot_normalizer': 10 * np.pi / 180}
    return dict(root=root, ycb=str(ycb), cfg=cfg, tpl=tpl, ckpt_b=c_dir + '/ckpt_b.pth.tar')


def _rng_state():
    return random.getstate(), np.random.get_state()


def _same_rng(a, b):
    return a[0] == b[0] and all(np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y for x, y in zip(a[1], b[1]))


@pytest.fixture(scope='module')
def written(layout, mods):
    """--mode ycbv's kept pairs per class ({class: (A_in_cam stack, B_in_cam stack)}) and the RNG state after writing."""
    out = layout['root'] / 'pairs'
    mods['produce_train_pair_data'].produce_ycbv(layout['ycb'], CLASSES + (7,), layout['tpl'], str(out), num_sample=NUM_SAMPLE, seed=SEED)
    state = _rng_state()
    pairs = {}
    for c in CLASSES + (7,):
        metas = [np.load(f) for f in sorted(glob.glob(str(out / ('%03d_obj' % c) / '*meta.npz')))]
        pairs[c] = (np.array([m['A_in_cam'] for m in metas]).reshape(-1, 4, 4), np.array([m['B_in_cam'] for m in metas]).reshape(-1, 4, 4))
    return pairs, state


@pytest.fixture(scope='module')
def one_pass(layout, mods):
    """Two checkpoints x (bf16x3, fp8) in one pass, and the RNG state after it."""
    random.seed(123); np.random.seed(123)
    tpl = dict(layout['tpl'], ckpt_dir=[layout['tpl']['ckpt_dir'], layout['ckpt_b']])
    res = mods['predict'].recoverYcbKeyframes(layout['ycb'], CLASSES + (7,), tpl, num_sample=NUM_SAMPLE, seed=SEED,
                                              precision=['bf16x3', 'fp8'], iterations=K)
    return res, _rng_state()


def test_kept_rows_are_the_written_pairs(written, one_pass):
    pairs, state = written
    res, after = one_pass
    assert _same_rng(after, state)
    assert set(res) == {(m, K, i) for m in ('bf16x3', 'fp8') for i in (0, 1)}
    for v, r in res.items():
        for c in CLASSES + (7,):
            A, B = pairs[c]
            assert r[c]['rows'] == len(A), (v, c)
            assert np.array_equal(r[c]['A_in_cam'], A) and np.array_equal(r[c]['B_in_cam'], B), (v, c)
            assert r[c]['poses'].shape == (K, len(A), 4, 4) and r[c]['errors'].shape == (K + 1, len(A), 4)
        assert r['all']['rows'] == sum(len(pairs[c][0]) for c in CLASSES)
    assert all(len(pairs[c][0]) > 0 for c in CLASSES) and len(pairs[7][0]) == 0
    assert len(pairs[2][0]) < NUM_SAMPLE * 6                     # class 2: some samples fail the centre or count test


def test_each_variant_is_its_run_alone(layout, mods, one_pass):
    res, _ = one_pass
    for i, ckpt in enumerate((layout['tpl']['ckpt_dir'], layout['ckpt_b'])):
        for m in ('bf16x3', 'fp8'):
            alone = mods['predict'].recoverYcbKeyframes(layout['ycb'], CLASSES + (7,), dict(layout['tpl'], ckpt_dir=ckpt),
                                                        num_sample=NUM_SAMPLE, seed=SEED, precision=m, iterations=K)
            assert list(alone) == [(m, K)]
            a, b = alone[m, K], res[m, K, i]
            for c in CLASSES + (7, 'all'):
                assert a[c]['rows'] == b[c]['rows']
                assert np.array_equal(a[c]['poses'], b[c]['poses']), (i, m, c)
                assert np.array_equal(a[c]['errors'], b[c]['errors'], equal_nan=True), (i, m, c)
                assert a[c]['summary'] == b[c]['summary'], (i, m, c)
    r7 = res['bf16x3', K, 0][7]
    assert r7['rows'] == 0 and all(s['rows'] == 0 and s['add_auc'] is None for s in r7['summary'])


def test_aucs_and_round_zero(mods, one_pass):
    res, _ = one_pass
    P, E = mods['predict'], mods['eval_ycb']
    for v, r in res.items():
        for c in CLASSES + ('all',):
            e = r[c]['errors']
            ref0 = P.pose_errors_np(r[c]['A_in_cam'], r[c]['B_in_cam'])
            assert np.abs(e[0, :, 0] - ref0[:, 0]).max() <= 1e-9 and np.abs(e[0, :, 1] - ref0[:, 1]).max() <= 1e-6
            for k in range(K + 1):
                s = r[c]['summary'][k]
                assert s['rows'] == e.shape[1]
                assert s['add_auc'] == E.VOCap(e[k, :, 2]) and s['adds_auc'] == E.VOCap(e[k, :, 3]), (v, c, k)
                assert s['rot_median'] == float(np.median(e[k, :, 1])) and s['trans_mean'] == float(np.mean(e[k, :, 0]))
            assert np.isfinite(e).all()
        assert r[2]['summary'][0] == res[next(iter(res))][2]['summary'][0]     # round 0 is the same start in every variant


def _engine_setup(mods, layout, synth):
    """An Engine with the three classes' weights, statistics and meshes under their ids, one key frame on the device, and the
    camera of the layout."""
    eng = mods['engine'].Engine(max_batch=16)
    for c in CLASSES:
        d = layout['cfg'] / ('c%d' % c)
        eng.load_state_dict(torch.load(str(d / 'ckpt_a.pth.tar'), map_location='cpu')['state_dict'], c)
        eng.set_stats(np.load(str(d / 'mean.npy')), np.load(str(d / 'std.npy')), c)
        eng.set_mesh(mods['mesh_io'].load_mesh(str(d / 'textured.ply')), c)
    info = yaml.safe_load(open(layout['cfg'] / 'c2' / 'dataset_info.yml'))
    cam = info['camera']
    Kc = np.array([[cam['focalX'], 0, cam['centerX']], [0, cam['focalY'], cam['centerY']], [0, 0, 1]])
    frames = []
    for i in (1, 2):
        base = os.path.join(layout['ycb'], 'data_organized', '0048')
        rgb = cv2.imread(os.path.join(base, 'color', '%06d-color.png' % i))[..., ::-1].copy()
        depth = cv2.imread(os.path.join(base, 'depth_filled', '%06d-depth.png' % i), cv2.IMREAD_UNCHANGED)
        frames.append((torch.from_numpy(rgb).to(eng.device), torch.from_numpy(depth).to(eng.device)))
    return eng, Kc, frames


@pytest.mark.parametrize('n', [3, 10])
def test_rounds_equal_r_round_steps(mods, layout, synth, one_pass, n):
    eng, Kc, frames = _engine_setup(mods, layout, synth)
    r0 = one_pass[0]['bf16x3', K, 0]
    starts = np.concatenate([r0[c]['A_in_cam'] for c in CLASSES])
    cls = np.concatenate([np.full(r0[c]['rows'], c, np.int32) for c in CLASSES])
    pick = np.linspace(0, len(starts) - 1, n).astype(int)
    start = torch.from_numpy(np.ascontiguousarray(starts[pick])).to(eng.device)
    wh = np.ascontiguousarray(cls[pick])
    wd = torch.from_numpy(wh).to(eng.device)
    widths = torch.tensor([200.0 + 10 * CLASSES.index(c) for c in wh], dtype=torch.float64, device=eng.device)
    for w in set(wh.tolist()):
        eng.set_fp8_scales(np.full(8, 2.0 ** -3, np.float32), w)
    out = torch.empty_like(start)
    rounds = torch.empty((K, n, 4, 4), dtype=torch.float64, device=eng.device)
    for m in ('bf16x3', 'bf16', 'fp8', 'fp32'):
        def step(frame, k, out_rounds=None):
            eng.track_render(frame[0], frame[1], Kc, start, widths, 0.05, 10 * np.pi / 180, weight_ids_host=wh, weight_ids_dev=wd,
                             precision=m, out_poses=out, iterations=k, out_rounds=out_rounds)
            torch.cuda.synchronize()
            return out.cpu().numpy().copy()
        final = step(frames[0], K, rounds)
        got = rounds.cpu().numpy().copy()
        for r in range(1, K + 1):
            assert np.array_equal(got[r - 1], step(frames[0], r)), (m, n, r)
        assert np.array_equal(final, got[K - 1]) and np.array_equal(final, step(frames[0], K)), (m, n)
        rounds.fill_(0)
        step(frames[1], K, rounds)
        if m != 'fp32':
            assert eng.last_step_was_graph(), (m, n)        # the second frame replays the step with the round output
        assert np.isfinite(rounds.cpu().numpy()).all()


def test_pose_errors_sets_against_numpy(mods, synth):
    eng = mods['engine'].Engine(max_batch=4)
    P = mods['predict']
    rng = np.random.default_rng(0)
    pts = [rng.standard_normal((m, 3)) * 0.05 for m in (300, 77, 513)]
    n = 12
    gt = synth.raw_poses(n, seed=1)
    pred = synth.raw_poses(n, seed=2)
    pred[0] = gt[0]                                            # exactly 0 degrees, 0 mm
    flip = np.diag([-1.0, -1.0, 1.0])                          # 180 degrees about z, then a hair less
    pred[1, :3, :3] = gt[1, :3, :3] @ flip
    a = np.pi - 1e-4
    pred[2, :3, :3] = gt[2, :3, :3] @ np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    pose_set = rng.integers(0, 3, n).astype(np.int32)
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(eng.device)
    errs, sets = eng.pose_errors_sets(pts, pose_set, dev(pred), dev(gt))
    e = errs.cpu().numpy()
    ref = P.pose_errors_np(pred, gt)
    assert np.abs(e[:, 0] - ref[:, 0]).max() <= 1e-9 and np.abs(e[:, 1] - ref[:, 1]).max() <= 1e-6
    assert e[0, 0] == 0.0 and e[0, 1] == 0.0 and abs(e[1, 1] - 180.0) <= 1e-6 and abs(e[2, 1] - np.degrees(a)) <= 1e-6
    add, adi = eng.add_adi_sets(pts, pose_set, dev(pred), dev(gt))
    assert np.array_equal(e[:, 2], add.cpu().numpy()) and np.array_equal(e[:, 3], adi.cpu().numpy())
    assert np.array_equal(sets.cpu().numpy(), pose_set)
    keep = np.ones(n, np.uint8); keep[[3, 7, 8]] = 0
    errs_m, sets_m = eng.pose_errors_sets(pts, pose_set, dev(pred), dev(gt), keep=dev(keep))
    em, sm = errs_m.cpu().numpy(), sets_m.cpu().numpy()
    assert np.isnan(em[keep == 0]).all() and (sm[keep == 0] == -1).all()
    assert np.array_equal(em[keep == 1], e[keep == 1]) and np.array_equal(sm[keep == 1], pose_set[keep == 1])
