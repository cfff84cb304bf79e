"""The one-pass scorer of perturbed YCB-Video key frames (problems.validate_ycbv, se3tn_append_pairs) on a synthetic layout of
120 x 160 frames, three classes with their own checkpoints, statistics and normalisers:

  * bit-identical to the file route (produce_train_pair_data --mode ycbv, then problems.evaluate on each class's folder) in every
    precision mode, with batches split into steps and latency-mode steps: pair counts, per-batch MSEs, means and predictions
  * random / np.random end in the same state after both routes
  * a class's full batches after its first replay their CUDA graphs
  * se3tn_append_pairs against numpy: kept and rejected rows, several queues with non-zero tails, poisoned slots left alone,
    and every invalid argument refused with every buffer unchanged
  * a class without a kept pair is reported with 0 pairs
"""
import importlib
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
MODES = ['bf16x3', 'tf32', 'bf16', 'fp16', 'fp8', 'fp32']
NUM_SAMPLE, SEED, BATCH, MAX_BATCH = 8, 4, 5, 3


@pytest.fixture(scope='module')
def mods():
    return {k: importlib.import_module(PKG + '.' + k) for k in ('produce_train_pair_data', 'problems', 'engine', 'datasets', '_lib',
                                                                 'mesh_io', 'se3_tracknet')}


@pytest.fixture(scope='module')
def layout(synth, mods, tmp_path_factory):
    """<root>/ycb: 6 key frames of sequence 0048; class 2 near the left edge (centre rejections, clipped windows), class 3 not
    annotated in frame 2, class 5 reduced to a 25-pixel patch in frame 4 (the visibility check rejects it), class 7 annotated
    everywhere but never labelled (no kept pair).  <root>/cfg/c<id>: dataset_info.yml, mesh, checkpoint, mean.npy / std.npy."""
    root = tmp_path_factory.mktemp('ycbv')
    ycb, cfg = root / 'ycb', root / 'cfg'
    K = synth.CAMERA_K.copy(); K[:2] *= 0.25
    cam = {'focalX': float(K[0, 0]), 'focalY': float(K[1, 1]), 'centerX': float(K[0, 2]), 'centerY': float(K[1, 2]), 'height': H, 'width': W}
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
        torch.save({'state_dict': synth.make_state_dict(10 + c)}, str(d / 'model_best_val.pth.tar'))
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
    tpl = {'train_data_path': str(cfg / 'c{class_id}' / 'train'), 'model_path': str(cfg / 'c{class_id}' / 'textured.ply'),
           'ckpt_dir': str(cfg / 'c{class_id}' / 'model_best_val.pth.tar'), 'mean_std_path': str(cfg / 'c{class_id}')}
    return dict(root=root, ycb=str(ycb), cfg=cfg, tpl=tpl)


def _rng_state():
    return random.getstate(), np.random.get_state()


def _same_rng(a, b):
    return a[0] == b[0] and all(np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y for x, y in zip(a[1], b[1]))


@pytest.fixture(scope='module')
def file_route(layout, mods):
    """--mode ycbv into folders, then evaluate on each class's folder: {class: {mode: dict}} and the RNG state after writing."""
    PP, P, D = mods['produce_train_pair_data'], mods['problems'], mods['datasets']
    out = layout['root'] / 'pairs'
    counts = PP.produce_ycbv(layout['ycb'], CLASSES, layout['tpl'], str(out), num_sample=NUM_SAMPLE, seed=SEED)
    state = _rng_state()
    eng = mods['engine'].Engine(max_batch=MAX_BATCH)
    res = {}
    for c in CLASSES:
        d = layout['cfg'] / ('c%d' % c)
        info = yaml.safe_load(open(d / 'dataset_info.yml'))
        ds = D.TrackDataset(str(out / ('%03d_obj' % c)), 'val', np.load(str(d / 'mean.npy')), np.load(str(d / 'std.npy')),
                            dataset_info=info, trans_normalizer=info['max_translation'], rot_normalizer=info['max_rotation'] * np.pi / 180)
        assert len(ds) == counts[c]
        model = mods['se3_tracknet'].Se3TrackNet(engine=eng, weight_id=0)
        model.load_state_dict(torch.load(str(d / 'model_best_val.pth.tar'), map_location='cpu')['state_dict'])
        res[c] = {m: P.evaluate(model, ds, BATCH, precision=m, keep_predictions=True) for m in MODES}
    return counts, state, res


def test_bit_identical_to_the_file_route(layout, mods, file_route):
    counts, state, ref = file_route
    assert all(counts[c] > BATCH for c in CLASSES)
    assert counts[2] < NUM_SAMPLE * 6                                  # class 2 (6 frames): some samples fail the centre or count test
    random.seed(123); np.random.seed(123)
    res = mods['problems'].validate_ycbv(layout['ycb'], CLASSES, layout['tpl'], num_sample=NUM_SAMPLE, seed=SEED, batch_size=BATCH,
                                         max_batch=MAX_BATCH, precisions=MODES, keep_predictions=True)
    assert _same_rng(_rng_state(), state)
    for c in CLASSES:
        plan = mods['problems'].batch_plan(counts[c], BATCH, MAX_BATCH)
        assert any(e - s <= 4 for _, s, e in plan) and len({b for b, _, _ in plan}) > 1
        for m in MODES:
            r, f = res[c][m], ref[c][m]
            assert r['pairs'] == counts[c], (c, m)
            assert np.array_equal(r['batch_trans'], f['batch_trans']) and np.array_equal(r['batch_rot'], f['batch_rot']), (c, m)
            assert r['trans'] == f['trans'] and r['rot'] == f['rot'], (c, m)
            assert np.array_equal(r['predictions'], f['predictions']), (c, m)
            assert np.isfinite(r['trans']) and np.isfinite(r['rot'])


def test_full_batches_replay_their_graphs(layout, mods, file_route):
    counts = file_route[0]
    P = mods['problems']
    eng = mods['engine'].Engine(max_batch=NUM_SAMPLE * len(CLASSES))
    log = []
    inner = eng.eval_pairs

    def eval_pairs(*a, **kw):
        out = inner(*a, **kw)
        log.append((int(kw['weight_ids_host'][0]), kw['precision'], int(a[0].shape[0]), eng.last_step_was_graph()))
        return out

    eng.eval_pairs = eval_pairs
    modes = ['bf16', 'tf32']
    res = P.validate_ycbv(layout['ycb'], CLASSES, layout['tpl'], num_sample=NUM_SAMPLE, seed=SEED, batch_size=BATCH,
                          max_batch=MAX_BATCH, precisions=modes, engine=eng)
    for c in CLASSES:
        assert res[c]['bf16']['pairs'] == counts[c]
        plan = P.batch_plan(counts[c], BATCH, MAX_BATCH)
        for m in modes:
            calls = [x for x in log if x[:2] == (c, m)]
            assert [n for _, _, n, _ in calls] == [e - s for _, s, e in plan]
            for (b, s, e), (_, _, _, graph) in zip(plan, calls):
                if b > 0 and (b + 1) * BATCH <= counts[c]:
                    assert graph, (c, m, b, s)


def test_no_kept_pair(layout, mods, file_route):
    P = mods['problems']
    res = P.validate_ycbv(layout['ycb'], (3, 7), layout['tpl'], num_sample=NUM_SAMPLE, seed=SEED, batch_size=BATCH,
                          max_batch=MAX_BATCH, precisions=['bf16'])
    r = res[7]['bf16']
    assert r['pairs'] == 0 and r['trans'] is None and r['rot'] is None and len(r['batch_trans']) == 0
    assert res[3]['bf16']['pairs'] > 0 and np.isfinite(res[3]['bf16']['trans'])


def test_append_pairs_against_numpy(mods):
    L = mods['_lib']
    eng = mods['engine'].Engine(max_batch=8)
    rng = np.random.default_rng(0)
    S = 176
    Q, cap = 3, 6

    def dev(x):
        return torch.from_numpy(np.ascontiguousarray(x)).to(eng.device)

    def pairs(n):
        return {'rgbA': dev(rng.integers(0, 256, (n, S, S, 3), dtype=np.uint8)), 'depthA': dev(rng.integers(0, 65536, (n, S, S), dtype=np.uint16)),
                'rgbB': dev(rng.integers(0, 256, (n, S, S, 3), dtype=np.uint8)), 'depthB': dev(rng.integers(0, 65536, (n, S, S), dtype=np.uint16))}

    queues = {'rgbA': dev(rng.integers(0, 256, (Q, cap, S, S, 3), dtype=np.uint8)), 'depthA': dev(rng.integers(0, 65536, (Q, cap, S, S), dtype=np.uint16)),
              'rgbB': dev(rng.integers(0, 256, (Q, cap, S, S, 3), dtype=np.uint8)), 'depthB': dev(rng.integers(0, 65536, (Q, cap, S, S), dtype=np.uint16)),
              'A_in_cam': dev(rng.standard_normal((Q, cap, 4, 4))), 'B_in_cam': dev(rng.standard_normal((Q, cap, 4, 4)))}
    tails0 = np.array([1, 0, 2], np.int32)
    tails = dev(tails0)
    p = pairs(7)
    p['count'] = dev(np.array([150, 99, 100, 0, 300, 101, 50], np.int32))
    qids = np.array([2, 0, 2, 1, 0, 2, 2], np.int32)
    A, B = dev(rng.standard_normal((7, 4, 4))), dev(rng.standard_normal((7, 4, 4)))

    def snapshot():
        torch.cuda.synchronize()
        return {k: v.cpu().numpy().copy() for k, v in queues.items()}, tails.cpu().numpy().copy()

    before, _ = snapshot()
    # every invalid argument: SE3TN_ERR_INVALID, nothing queued
    p9 = pairs(9); p9['count'] = dev(np.full(9, 200, np.int32))
    bad = [(p9, dev(np.zeros((9, 4, 4))), dev(np.zeros((9, 4, 4))), np.zeros(9, np.int32), tails0),     # n > max_batch
           (p, A, B, np.array([2, 0, 2, 1, 0, 3, 2], np.int32), tails0),                                  # queue id out of range
           (p, A, B, np.array([2, 0, 2, 1, 0, -1, 2], np.int32), tails0),
           (p, A, B, qids, np.array([1, 0, 3], np.int32))]                                                # queue 2: 3 + 4 rows > 6
    for pp, a, b, q, th in bad:
        with pytest.raises(L.Se3tnError) as e:
            eng.append_pairs(pp, a, b, q, th, tails, queues)
        assert e.value.code == L.ERR_INVALID
        q_now, t_now = snapshot()
        assert np.array_equal(t_now, tails0) and all(np.array_equal(q_now[k], before[k]) for k in before)
    eng.append_pairs(p, A, B, qids, tails0, tails, queues)
    assert eng.last_launch_count() == 1
    after, t_after = snapshot()
    expect = {k: v.copy() for k, v in before.items()}
    t = tails0.copy()
    host = {k: v.cpu().numpy() for k, v in p.items()}
    An, Bn = A.cpu().numpy(), B.cpu().numpy()
    for i, q in enumerate(qids):
        if host['count'][i] < L.PAIR_MIN_SEG:
            continue
        for k in ('rgbA', 'depthA', 'rgbB', 'depthB'):
            expect[k][q, t[q]] = host[k][i]
        expect['A_in_cam'][q, t[q]] = An[i]; expect['B_in_cam'][q, t[q]] = Bn[i]
        t[q] += 1
    assert t.tolist() == [2, 0, 5] and np.array_equal(t_after, t)
    for k in expect:
        assert np.array_equal(after[k], expect[k]), k
