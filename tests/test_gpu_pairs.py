"""The pair generator on the device (se3tn_perturb_pairs, se3tn_visibility, ProducerPurturb, the YCB-Video mode) against the CPU
oracle (oracle/pairs_oracle.py) on synthetic 120 x 160 frames and small meshes:

  * every field of every sample (rgbA, depthA, rgbB, depthB, segB, count) bit-identical to the oracle's generate loop, with
    samples rejected by the centre test and by the seg test and windows that leave the image
  * the visibility counts equal the oracle's full-frame render, a pose that draws nothing included (covered == 0 is kept)
  * one step with several classes and meshes; chunking of n > max_batch; the error codes; graph replay on a second frame
  * generate's folder decodes to the oracle's arrays and Problem.validate gives the same loss as on an oracle-written folder
  * the YCB-Video mode writes what per-class generate calls write
"""
import importlib, os, random
import cv2
import numpy as np
import pytest
import torch
import yaml

import pairs_oracle as PO
import se3_oracle as O

pytestmark = pytest.mark.gpu
PKG = 'iros20-6d-pose-tracking_b200'
H, W = 120, 160


@pytest.fixture(scope='module')
def PP():
    return importlib.import_module(PKG + '.produce_train_pair_data')


@pytest.fixture(scope='module')
def env(synth):
    E = importlib.import_module(PKG + '.engine').Engine
    K = synth.CAMERA_K.copy(); K[:2] *= 0.25
    cam = {'focalX': float(K[0, 0]), 'focalY': float(K[1, 1]), 'centerX': float(K[0, 2]), 'centerY': float(K[1, 2]), 'height': H, 'width': W}
    info = {'resolution': 176, 'object_width': 200.0, 'boundingbox': 10, 'max_translation': 0.06, 'max_rotation': 20.0, 'camera': cam}
    meshes = {3: synth.mesh(2, seed=3), 5: synth.mesh(2, seed=5)}
    eng = E(max_batch=16)
    for mid, m in meshes.items():
        eng.set_mesh(m, mid)
    K32 = np.zeros((3, 3), np.float32); K32[0, 0], K32[1, 1], K32[0, 2], K32[1, 2], K32[2, 2] = K[0, 0], K[1, 1], K[0, 2], K[1, 2], 1
    return dict(eng=eng, info=info, meshes=meshes, K32=K32, K=K32.astype(np.float64))


def frame(synth, env, seed, B, mesh_id, class_id, patch=False):
    """rgb / depth noise and a seg image that labels the model's full-image render at B (or only a 5 x 5 patch of it)."""
    rgb, depth = synth.raw_frame(seed, H, W)
    _, d = O.render_full_frame_unlit(B, env['K'], env['meshes'][mesh_id], H, W)
    seg = np.zeros((H, W), np.uint8)
    seg[20:40, 100:150] = 7                                         # another object
    if patch:
        ys, xs = np.nonzero(d > 0)
        seg[ys[0]:ys[0] + 5, xs[0]:xs[0] + 5] = class_id
    else:
        seg[d > 0] = class_id
    return rgb, depth, seg


def poses(synth):
    B1 = synth.raw_poses(1, seed=3)[0]; B1[:3, 3] = (-0.13, 0.02, 0.5)         # near the left edge: centre rejections, clipped windows
    B2 = synth.raw_poses(1, seed=4)[0]; B2[:3, 3] = (0.02, -0.01, 0.6)
    return B1, B2


def dev(eng, *a):
    return [torch.from_numpy(np.ascontiguousarray(x)).to(eng.device) for x in a]


def check_step(env, rgb, depth, seg, rows, res):
    """rows [(A_in_cam, mesh id, class id)] against the oracle, field by field."""
    for k, (A, mid, cid) in enumerate(rows):
        bb = O.compute_bbox(A, env['K'], 200.0, scale=(1000, 1000, 1000))
        rA, dA = O.render_window_pyrender(A, env['K'], 200.0, env['meshes'][mid], H, W)
        rB, dB, sB = PO.crop_bbox_seg(rgb, depth, bb, (176, 176), seg)
        assert np.array_equal(res['rgbA'][k].cpu().numpy(), rA), k
        assert np.array_equal(res['depthA'][k].cpu().numpy(), dA), k
        assert np.array_equal(res['rgbB'][k].cpu().numpy(), rB), k
        assert np.array_equal(res['depthB'][k].cpu().numpy(), dB), k
        assert np.array_equal(res['segB'][k].cpu().numpy(), (sB == cid).astype(np.uint8)), k
        assert int(res['count'][k]) == int(np.sum(sB == cid)), k


def test_generate_step_matches_oracle(PP, env, synth):
    eng = env['eng']
    statuses, clipped = set(), False
    for seed, B, patch in ((11, poses(synth)[0], False), (12, poses(synth)[1], True)):
        rgb, depth, seg = frame(synth, env, seed, B, 3, 2, patch)
        random.seed(seed); np.random.seed(seed)
        recs = PO.generate(B, rgb, depth, seg, 12, 2, env['K32'], 200.0, 0.06, 20.0, env['meshes'][3])
        stub = type('P', (), {})(); stub.dataset_info = env['info']; stub.cam_K = env['K32']
        random.seed(seed); np.random.seed(seed)
        draws = PP.ProducerPurturb.draw(stub, B, 12)
        assert all(np.array_equal(r['A_in_cam'], A) and (r['status'] != 'centre') == ok for r, (A, ok) in zip(recs, draws))
        inside = [r for r in recs if r['status'] != 'centre']
        A = np.stack([r['A_in_cam'] for r in inside])
        f = dev(eng, rgb, depth, seg)
        res = eng.perturb_pairs(*f, env['K32'], *dev(eng, A, np.full(len(A), 200.0), np.full(len(A), 2, np.int32)),
                                mesh_ids=np.full(len(A), 3, np.int32))
        assert eng.last_launch_count() == 4
        for k, r in enumerate(inside):
            for key in ('rgbA', 'depthA', 'rgbB', 'depthB', 'segB'):
                assert np.array_equal(res[key][k].cpu().numpy(), r[key]), (seed, k, key)
            assert int(res['count'][k]) == r['count']
            top, left, ch, cw = O.crop_window(O.compute_bbox(r['A_in_cam'], env['K'], 200.0, scale=(1000, 1000, 1000)))
            clipped |= top < 0 or left < 0 or top + ch > H or left + cw > W
        statuses |= {r['status'] for r in recs}
    assert statuses == {'centre', 'seg', 'kept'} and clipped


def test_visibility_counts(PP, env, synth):
    eng = env['eng']
    B1, B2 = poses(synth)
    behind = B2.copy(); behind[2, 3] = -0.5                         # draws nothing
    rgb, depth, seg = frame(synth, env, 13, B2, 5, 4)
    rows = [(B2, 5, 4), (B1, 3, 4), (B2, 3, 7), (behind, 5, 4), (B1, 5, 0)]
    vis, cov = PP.visibility(eng, dev(eng, seg)[0], env['K32'], rows)
    for k, (B, mid, cid) in enumerate(rows):
        assert (vis[k], cov[k]) == PO.visibility_counts(seg, cid, B, env['K'], env['meshes'][mid]), k
    assert cov[3] == 0 and vis[3] > 100 and PP.visible_enough(vis[3], cov[3])
    assert cov[0] > 0


def test_mixed_meshes_and_chunking(PP, env, synth):
    eng = env['eng']
    B1, B2 = poses(synth)
    rgb, depth, seg = frame(synth, env, 14, B2, 5, 4)
    seg[40:90, 0:40] = 2                                            # class 2 near B1 (left edge)
    random.seed(1); np.random.seed(1)
    rows = []
    for k in range(20):                                             # 20 rows > max_batch 16: two steps
        B, mid, cid = ((B2, 5, 4), (B1, 3, 2))[k % 2]
        rows.append((B.dot(np.linalg.inv(PO.random_gaussian_magnitude(0.02, 10.0))), 200.0, mid, cid))
    f = dev(eng, rgb, depth, seg)
    res = PP.pair_step(eng, f, env['K32'], rows)
    check_step(env, rgb, depth, seg, [(A, m, c) for A, _, m, c in rows], {k: torch.from_numpy(v) for k, v in res.items()})
    E = type(eng)
    small = E(max_batch=3)
    for mid, m in env['meshes'].items():
        small.set_mesh(m, mid)
    res3 = PP.pair_step(small, dev(small, rgb, depth, seg), env['K32'], rows)
    for k in res:
        assert np.array_equal(res[k], res3[k]), k


def test_errors(env, synth):
    eng = env['eng']
    L = importlib.import_module(PKG + '._lib')
    B1, B2 = poses(synth)
    rgb, depth, seg = frame(synth, env, 15, B2, 5, 4)
    f = dev(eng, rgb, depth, seg)
    A, ow, cid = dev(eng, np.stack([B2, B2]), np.full(2, 200.0), np.full(2, 4, np.int32))
    with pytest.raises(L.Se3tnError) as e:
        eng.perturb_pairs(*f, env['K32'], A, ow, cid, mesh_ids=np.array([5, 9], np.int32))
    assert e.value.code == L.ERR_STATE and '9' in str(e.value)
    with pytest.raises(L.Se3tnError) as e:
        eng.visibility(f[2], env['K32'], A, cid, mesh_ids=np.array([9, 5], np.int32))
    assert e.value.code == L.ERR_STATE
    n = 17
    An, own, cidn = dev(eng, np.stack([B2] * n), np.full(n, 200.0), np.full(n, 4, np.int32))
    with pytest.raises(L.Se3tnError) as e:
        eng.perturb_pairs(*f, env['K32'], An, own, cidn)
    assert e.value.code == L.ERR_INVALID
    with pytest.raises(L.Se3tnError) as e:
        eng.visibility(f[2], env['K32'], An, cidn)
    assert e.value.code == L.ERR_INVALID


def test_graph_replay_on_second_frame(env, synth):
    eng = env['eng']
    B1, B2 = poses(synth)
    random.seed(2); np.random.seed(2)
    A = np.stack([B2.dot(np.linalg.inv(PO.random_gaussian_magnitude(0.02, 10.0))) for _ in range(5)])
    tA, tw, tc = dev(eng, A, np.full(5, 200.0), np.full(5, 4, np.int32))
    f = dev(eng, *frame(synth, env, 16, B2, 5, 4))
    out = eng.perturb_pairs(*f, env['K32'], tA, tw, tc, mesh_ids=np.full(5, 5, np.int32))
    first = eng.last_step_was_graph()
    for seed in (17, 18):                                           # new frames in the same buffers: the captured step replays
        rgb, depth, seg = frame(synth, env, seed, B2, 5, 4)
        for t, x in zip(f, (rgb, depth, seg)):
            t.copy_(torch.from_numpy(x))
        out = eng.perturb_pairs(*f, env['K32'], tA, tw, tc, mesh_ids=np.full(5, 5, np.int32), out=out)
        assert eng.last_step_was_graph() and first and eng.last_launch_count() == 4
        torch.cuda.synchronize()
        check_step(env, rgb, depth, seg, [(a, 5, 4) for a in A], out)


def _write_folder(path, recs, B):
    from PIL import Image
    os.makedirs(path, exist_ok=True)
    i = 0
    for r in recs:
        if r['status'] != 'kept':
            continue
        s = os.path.join(path, '%07d' % i)
        Image.fromarray(r['rgbA']).save(s + 'rgbA.png'); Image.fromarray(r['rgbB']).save(s + 'rgbB.png')
        cv2.imwrite(s + 'depthA.png', r['depthA']); cv2.imwrite(s + 'depthB.png', r['depthB']); cv2.imwrite(s + 'segB.png', r['segB'])
        np.savez(s + 'meta.npz', A_in_cam=r['A_in_cam'], B_in_cam=B)
        i += 1
    return i


def test_generate_folder_and_validate(PP, env, synth, pkg, tmp_path):
    eng = env['eng']
    D = importlib.import_module(PKG + '.datasets')
    P = importlib.import_module(PKG + '.problems')
    B1, B2 = poses(synth)
    rgb, depth, seg = frame(synth, env, 19, B1, 3, 2)
    prod = PP.ProducerPurturb(env['info'], engine=eng, model=env['meshes'][3], mesh_id=3)
    prod.count = 3                                                  # the count carries over between calls
    os.makedirs(tmp_path / 'dev')                                   # generate writes into an existing folder, as the reference does
    random.seed(19); np.random.seed(19)
    prod.generate(str(tmp_path / 'dev') + '/', B1, rgb, depth, 14, 2, current_seg=seg)
    random.seed(19); np.random.seed(19)
    recs = PO.generate(B1, rgb, depth, seg, 14, 2, env['K32'], 200.0, 0.06, 20.0, env['meshes'][3])
    kept = [r for r in recs if r['status'] == 'kept']
    assert len(kept) >= 2 and prod.count == 3 + len(kept)
    files = sorted(f for f in os.listdir(tmp_path / 'dev') if f.endswith('rgbA.png'))
    assert files == ['%07drgbA.png' % i for i in range(3, 3 + len(kept))]
    for i, r in enumerate(kept):
        p = D.read_pair(str(tmp_path / 'dev' / files[i]))
        for key in ('rgbA', 'rgbB', 'depthA', 'depthB', 'segB'):
            assert np.array_equal(p[key], r[key]), (i, key)
        assert np.array_equal(p['A_in_cam'], r['A_in_cam']) and np.array_equal(p['B_in_cam'], B1)
    with pytest.raises(ValueError):
        prod.generate(str(tmp_path / 'dev') + '/', B1, rgb, depth, 1, 2)
    _write_folder(str(tmp_path / 'ora'), recs, B1)
    os.makedirs(tmp_path / 'dev0')
    for f in os.listdir(tmp_path / 'dev'):                          # the oracle folder numbers from 0
        os.rename(tmp_path / 'dev' / f, tmp_path / 'dev0' / ('%07d' % (int(f[:7]) - 3) + f[7:]))
    mean, std = synth.default_mean_std()
    sd = synth.make_state_dict(0)
    losses = []
    for sub in ('dev0', 'ora'):
        ds = D.TrackDataset(str(tmp_path / sub), 'val', mean, std, dataset_info=env['info'], engine=eng)
        loader = torch.utils.data.DataLoader(ds, batch_size=4, shuffle=False, drop_last=False)
        model = pkg.Se3TrackNet(engine=eng, weight_id=0)
        model.load_state_dict(sd)
        losses.append(P.Problem(model, None, loader, config={'loss_weights': {'trans': 1, 'rot': 1}}).validate(precision='bf16x3'))
    assert np.isfinite(losses[0]) and losses[0] == losses[1]


def test_visibility_check_in_generate(PP, env, synth, tmp_path):
    """check_vis: a frame whose class covers <= 100 pixels draws nothing; one that passes draws num_sample offsets."""
    eng = env['eng']
    B1, B2 = poses(synth)
    rgb, depth, seg = frame(synth, env, 20, B2, 5, 4, patch=True)       # 25 labelled pixels
    prod = PP.ProducerPurturb(env['info'], check_vis=True, engine=eng, model=env['meshes'][5], mesh_id=5)
    random.seed(5); np.random.seed(5)
    prod.generate(str(tmp_path) + '/', B2, rgb, depth, 4, 4, current_seg=seg)
    after = random.random()
    random.seed(5)
    assert after == random.random() and prod.count == 0              # no draw
    rgb, depth, seg = frame(synth, env, 20, B2, 5, 4)
    prod.generate(str(tmp_path) + '/', B2, rgb, depth, 4, 4, current_seg=seg)
    assert prod.count > 0


def test_ycbv_mode(PP, env, synth, tmp_path):
    """--mode ycbv on a synthetic YCB-Video layout (two classes, one in every key frame, one in some): one visibility call and one
    pair step per frame write exactly what one check_vis ProducerPurturb per class, called frame by frame, writes."""
    mio = importlib.import_module(PKG + '.mesh_io')
    from PIL import Image
    ycb, cfg = tmp_path / 'ycb', tmp_path / 'cfg'
    classes, nframes = (3, 5), 4
    for c in classes:
        (cfg / ('c%d' % c) / 'train').mkdir(parents=True)
        yaml.safe_dump(env['info'], open(cfg / ('c%d' % c) / 'dataset_info.yml', 'w'))
        mio.save_ply_mesh(str(cfg / ('c%d' % c) / 'textured.ply'), env['meshes'][c])
    for k in range(1, 22):
        (ycb / 'CADmodels' / ('%03d_obj' % k)).mkdir(parents=True)
    base = ycb / 'data_organized' / '0048'
    B1, B2 = poses(synth)
    gt = {3: B1, 5: B2}
    for d in ('color', 'depth_filled', 'seg', 'pose_gt/3', 'pose_gt/5'):
        (base / d).mkdir(parents=True)
    for i in range(nframes):
        rgb, depth, _ = frame(synth, env, 30 + i, B2, 5, 5)
        seg = np.zeros((H, W), np.uint8)
        for c in classes:
            _, d = O.render_full_frame_unlit(gt[c], env['K'], env['meshes'][c], H, W)
            seg[d > 0] = c
        cv2.imwrite(str(base / 'color' / ('%06d-color.png' % (i + 1))), rgb[..., ::-1])
        cv2.imwrite(str(base / 'depth_filled' / ('%06d-depth.png' % (i + 1))), depth)
        cv2.imwrite(str(base / 'seg' / ('%06d-label.png' % (i + 1))), seg)
        for c in classes:
            if c == 3 and i == 1:
                continue                                            # class 3 is not annotated in frame 2
            np.savetxt(str(base / 'pose_gt' / str(c) / ('%06d.txt' % (i + 1))), gt[c])
    (ycb / 'image_sets').mkdir()
    (ycb / 'image_sets' / 'keyframe.txt').write_text('0048/000001\n0048/000002\n0048/000004\n')
    tpl = {'train_data_path': str(cfg / 'c{class_id}' / 'train'), 'model_path': str(cfg / 'c{class_id}' / 'textured.ply')}
    counts = PP.main(['--mode', 'ycbv', '--ycb_dir', str(ycb), '--class_ids', '3,5', '--train_data_path', tpl['train_data_path'],
                      '--model_path', tpl['model_path'], '--outdir', str(tmp_path / 'out'), '--num_sample', '6', '--seed', '3'])
    # the same pairs one class and one frame at a time
    E = type(env['eng'])
    eng2 = E(max_batch=16)
    prods = {c: PP.ProducerPurturb(env['info'], check_vis=True, engine=eng2, model=str(cfg / ('c%d' % c) / 'textured.ply'), mesh_id=c)
             for c in classes}
    random.seed(3); np.random.seed(3)
    for fr in ('000001', '000002', '000004'):
        rgb = np.array(Image.open(str(base / 'color' / (fr + '-color.png'))))[:, :, :3]
        depth = cv2.imread(str(base / 'depth_filled' / (fr + '-depth.png')), cv2.IMREAD_UNCHANGED)
        seg = cv2.imread(str(base / 'seg' / (fr + '-label.png')), cv2.IMREAD_UNCHANGED)
        for c in classes:
            p = base / 'pose_gt' / str(c) / (fr + '.txt')
            if p.exists():
                d = tmp_path / 'ref' / ('%03d_obj' % c)
                d.mkdir(parents=True, exist_ok=True)
                prods[c].generate(str(d) + '/', np.loadtxt(str(p)), rgb, depth, 6, c, current_seg=seg)
    assert counts == {c: prods[c].count for c in classes} and all(v > 0 for v in counts.values())
    for c in classes:
        out, ref = tmp_path / 'out' / ('%03d_obj' % c), tmp_path / 'ref' / ('%03d_obj' % c)
        assert sorted(os.listdir(out)) == sorted(os.listdir(ref))
        for f in os.listdir(out):
            a = np.load(str(out / f)) if f.endswith('.npz') else cv2.imread(str(out / f), cv2.IMREAD_UNCHANGED)
            b = np.load(str(ref / f)) if f.endswith('.npz') else cv2.imread(str(ref / f), cv2.IMREAD_UNCHANGED)
            if f.endswith('.npz'):
                assert all(np.array_equal(a[k], b[k]) for k in ('A_in_cam', 'B_in_cam')), f
            else:
                assert np.array_equal(a, b), f
