"""The result videos on the device: se3tn_draw_tracks against the CPU oracle (oracle/overlay_oracle.py, cv2's own drawing), and
the one-pass drivers with video=True on small synthetic YCB-Video and YCBInEOAT trees.

  * draw_tracks bit for bit the oracle for n = 1, 3 and 5 tracks with repeated point sets, both label orders and no label, with
    points off the image, on its borders and corners, on .5 ties, behind the camera and at z' = 0
  * odd frame sizes, bad offset tables, out-of-range set ids and label rows outside the frame raise with nothing queued
  * getResultsYcbAll / getResultsYcbInEOAT with video=True: the same poses as without, graph replays after each track set's
    first step, every frame handed to the video sink equal to the oracle drawn from the returned poses, complete mp4 files, and
    the same scores
"""
import argparse, contextlib, importlib, io, os, shutil
import cv2
import numpy as np
import pytest
import torch
import yaml

import overlay_oracle as OV

pytestmark = pytest.mark.gpu

PKG = 'iros20-6d-pose-tracking_b200'
H, W = 480, 640


@pytest.fixture(scope='module')
def pr():
    return importlib.import_module(PKG + '.predict')


@pytest.fixture(scope='module')
def eng(pkg):
    e = pkg.Engine(max_batch=1)
    yield e
    e.close()


def special_points(K):
    """Camera-frame points (drawn with the identity pose) that land on the borders and corners, one pixel off them, far off the
    image, on .5 ties, behind the camera but inside the image, and at z' = 0."""
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    uv = [(0, 0), (W - 1, 0), (0, H - 1), (W - 1, H - 1), (W // 2, 0), (W // 2, H - 1), (0, H // 2), (W - 1, H // 2),
          (-1, 100), (W, 100), (100, -1), (100, H), (-1, -1), (W, H), (-2, 50), (W + 1, 50), (5000, 5000), (-1e12, 3)]
    z = 0.8
    pts = [((u - cx) * z / fx, (v - cy) * z / fy, z) for u, v in uv]
    pts += [((10.5 - cx) / fx, (20 - cy) / fy, 1.0), ((11.5 - cx) / fx, (20.5 - cy) / fy, 1.0)]   # ties, exact with K below
    pts += [((u - cx) * -0.5 / fx, (v - cy) * -0.5 / fy, -0.5) for u, v in ((200, 300), (W - 1, 7))]   # behind, landing inside
    pts += [(0.1, 0.05, 0.0), (0.0, 0.0, 0.0), (-0.2, 0.0, 0.0)]                                     # z' = 0: inf and nan
    return np.array(pts, dtype=np.float64)


@pytest.mark.parametrize('n', [1, 3, 5])
@pytest.mark.parametrize('label_order', [None, 'under', 'over'])
def test_draw_tracks_bit_identical_to_the_oracle(pkg, pr, synth, eng, n, label_order):
    dev = eng.device
    K = np.array([[1024.0, 0, 320.0], [0, 1024.0, 240.0], [0, 0, 1]])                 # powers of two: the .5 ties are exact
    rng = np.random.default_rng(n)
    frame = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    frame[rng.random((H, W)) < 0.02] = 255
    frame[:40, :40] = 0
    sets = [synth.mesh(3, seed=1)['pos'].astype(np.float64), special_points(K), synth.mesh(3, seed=2)['pos'].astype(np.float64) * 1.5]
    offsets = np.cumsum([0] + [len(s) for s in sets]).astype(np.int32)
    track_set = np.array([1, 0, 2, 0, 1][:n], dtype=np.int32)                         # repeated sets
    poses = synth.raw_poses(n, seed=n)
    for i in range(n):
        if track_set[i] == 1:
            poses[i] = np.eye(4)
        else:                                                                         # the object near the label
            poses[i, 0, 3], poses[i, 1, 3] = (360 + 40 * i - 320) * poses[i, 2, 3] / 1024, (H - 60 - 240) * poses[i, 2, 3] / 1024
    text = 'frame:%d' % (10 ** n + 7)
    label = None
    if label_order is not None:
        y0, mask = pr.label_strip(text, H, W)
        label = (y0, torch.from_numpy(mask).to(dev))
    table = torch.from_numpy(np.concatenate(sets)).to(dev)
    out = eng.draw_tracks(torch.from_numpy(frame).to(dev), K, torch.from_numpy(poses).to(dev), table, offsets, track_set, label=label,
                          label_order=label_order or 'under').cpu().numpy()
    assert out.shape == (n, H // 2, W // 2, 3)
    for i in range(n):
        want = OV.draw_track(frame, K, poses[i], sets[track_set[i]], None if label_order is None else text, label_order or 'under')
        diff = np.argwhere(out[i] != want)
        assert len(diff) == 0, 'track %d: %d bytes differ, first at %s' % (i, len(diff), diff[:5].tolist())
    if label_order == 'over' and n > 1:                                               # the order matters where dots meet the label
        under = eng.draw_tracks(torch.from_numpy(frame).to(dev), K, torch.from_numpy(poses).to(dev), table, offsets, track_set,
                                label=label, label_order='under').cpu().numpy()
        assert not np.array_equal(under, out)


def test_draw_tracks_refusals_queue_nothing(pkg, pr, eng):
    dev = eng.device
    L = importlib.import_module(PKG + '._lib')
    pts = torch.zeros((4, 3), dtype=torch.float64, device=dev)
    pts[:, 2] = 1.0
    poses = torch.eye(4, dtype=torch.float64, device=dev).repeat(2, 1, 1)
    K = np.array([500.0, 500.0, 320.0, 240.0])

    def call(h=H, w=W, offsets=(0, 2, 4), ids=(0, 1), label=None):
        frame = torch.zeros((h, w, 3), dtype=torch.uint8, device=dev)
        out = torch.full((len(ids), h // 2, w // 2, 3), 7, dtype=torch.uint8, device=dev)
        with pytest.raises(L.Se3tnError) as e:
            eng.draw_tracks(frame, K, poses[:len(ids)], pts, np.array(offsets), np.array(ids), label=label, out=out)
        torch.cuda.synchronize()
        assert e.value.code == L.ERR_INVALID
        assert bool((out == 7).all()), 'a refused call wrote its output'
        return str(e.value)
    assert 'even' in call(h=H - 1) and 'even' in call(w=W - 1)
    assert 'set_offsets' in call(offsets=(1, 2, 4)) and 'set_offsets' in call(offsets=(0, 2, 3))
    assert 'empty' in call(offsets=(0, 0, 4)) and 'empty' in call(offsets=(0, 3, 2, 4), ids=(0, 2))
    assert 'track 1 has set id 2' in call(ids=(0, 2)) and 'track 0 has set id -1' in call(ids=(-1, 0))
    strip = torch.zeros((40, W), dtype=torch.uint8, device=dev)
    assert 'label rows' in call(label=(H - 39, strip)) and 'label rows' in call(label=(-1, strip))


# ------------------------------------------------------------------------------------------------------------ the drivers
def _write_cfg(d, synth, mio, seed, width, cam):
    mean, std = synth.default_mean_std()
    (d / 'train').mkdir(parents=True)
    yaml.safe_dump({'resolution': 176, 'object_width': width, 'boundingbox': 10, 'camera': cam}, open(d / 'dataset_info.yml', 'w'))
    np.save(d / 'mean.npy', mean + seed); np.save(d / 'std.npy', std * (1 + 0.05 * seed))
    torch.save({'epoch': 1, 'state_dict': synth.make_state_dict(seed), 'best_prec': 0.0}, str(d / 'model_best_val.pth.tar'))
    mio.save_ply_mesh(str(d / 'textured.ply'), synth.mesh(3, seed=seed))


def _camera(synth):
    K = synth.CAMERA_K
    return {'focalX': float(K[0, 0]), 'focalY': float(K[1, 1]), 'centerX': float(K[0, 2]), 'centerY': float(K[1, 2]), 'height': H, 'width': W}


def _model_points(pr, model_path):
    """Tracker.object_cloud.points of a Tracker built on model_path."""
    return pr.PointCloud(pr.load_vertices(model_path)).voxel_down_sample(voxel_size=0.005).points


@pytest.fixture(scope='module')
def recorder(pkg):
    """Every Engine.track_render call (n, last_step_was_graph) and every VideoSink.put call (frames on the host, paths, last)."""
    st = importlib.import_module(PKG + '.staging')
    E, S = pkg.Engine, st.VideoSink
    orig_track, orig_put = E.track_render, S.put
    rec = {'steps': [], 'puts': []}

    def track_render(self, *a, **kw):
        out = orig_track(self, *a, **kw)
        rec['steps'].append((int(a[3].shape[0]), self.last_step_was_graph()))
        return out

    def put(self, frames, paths, last=False):
        rec['puts'].append((frames.cpu().numpy(), list(paths), last))
        return orig_put(self, frames, paths, last)
    E.track_render, S.put = track_render, put
    yield rec
    E.track_render, S.put = orig_track, orig_put


YCB_CLASSES = (2, 5, 7)
YCB_SEQS = {48: (2, 5, 7), 49: (2, 5)}
NFRAMES = 4


@pytest.fixture(scope='module')
def ycb_tree(tmp_path_factory, synth):
    mio = importlib.import_module(PKG + '.mesh_io')
    tmp = tmp_path_factory.mktemp('overlay_ycb')
    ycb, cfg = tmp / 'ycb', tmp / 'cfg'
    for c in YCB_CLASSES:
        _write_cfg(cfg / ('c%d' % c), synth, mio, c, 150.0 + 20 * c, _camera(synth))
    for k in range(1, 22):
        (ycb / 'CADmodels' / ('%03d_obj' % k)).mkdir(parents=True)
        np.savetxt(str(ycb / 'CADmodels' / ('%03d_obj' % k) / 'points.xyz'),
                   synth.mesh(3, seed=k if k in YCB_CLASSES else YCB_CLASSES[k % 3])['pos'].astype(np.float64))
    for seq, cls in YCB_SEQS.items():
        base = ycb / 'data_organized' / ('%04d' % seq)
        for d in ['color', 'depth_filled'] + ['pose_gt/%d' % c for c in cls]:
            (base / d).mkdir(parents=True)
        for i in range(NFRAMES):
            rgb, depth = synth.raw_frame(seed=100 * seq + i)
            cv2.imwrite(str(base / 'color' / ('%06d-color.png' % (i + 1))), rgb[..., ::-1])
            cv2.imwrite(str(base / 'depth_filled' / ('%06d-depth.png' % (i + 1))), depth)
        for c in cls:
            p = synth.raw_poses(NFRAMES, seed=10 * seq + c)
            p[1:, :3, 3] = p[0, :3, 3] + 0.002 * np.arange(1, NFRAMES)[:, None]
            p[1:, :3, :3] = p[0, :3, :3]
            for i in range(NFRAMES):
                np.savetxt(str(base / 'pose_gt' / str(c) / ('%06d.txt' % (i + 1))), p[i])
    (ycb / 'image_sets').mkdir()
    (ycb / 'image_sets' / 'keyframe.txt').write_text('0048/000002\n0048/000004\n0049/000003\n')
    (ycb / 'YCB_Video_toolbox').mkdir()
    shutil.copy(str(ycb / 'image_sets' / 'keyframe.txt'), str(ycb / 'YCB_Video_toolbox' / 'keyframe.txt'))
    templates = {'train_data_path': str(cfg / 'c{class_id}' / 'train'), 'mean_std_path': str(cfg / 'c{class_id}'),
                 'ckpt_dir': str(cfg / 'c{class_id}' / 'model_best_val.pth.tar'), 'model_path': str(cfg / 'c{class_id}' / 'textured.ply')}
    return tmp, templates


def test_ycb_all_videos(pr, synth, ycb_tree, recorder):
    tmp, templates = ycb_tree
    ycb = str(tmp / 'ycb')
    plain = pr.getResultsYcbAll(ycb, list(YCB_CLASSES), templates, str(tmp / 'plain'))
    assert not recorder['puts']                                        # video=False hands the sink nothing
    s0 = len(recorder['steps'])
    res = pr.main(['--mode', 'ycbv_all', '--ycb_dir', ycb, '--class_ids', ','.join(map(str, YCB_CLASSES)), '--outdir', str(tmp / 'video'),
                   '--video'] + sum([['--' + k, v] for k, v in templates.items()], []))
    for c in YCB_CLASSES:
        for seq in plain[c]:
            assert np.array_equal(plain[c][seq], res[c][seq]), (c, seq)
    steps, puts = recorder['steps'][s0:], recorder['puts']
    assert [n for n, _ in steps] == [3] * (NFRAMES - 1) + [2] * (NFRAMES - 1)
    for s in (0, NFRAMES - 1):
        assert all(g for _, g in steps[s + 1:s + NFRAMES - 1]), steps
    names = pr.ycb_class_names(ycb)
    assert len(puts) == len(YCB_SEQS) * (NFRAMES - 1)
    k = 0
    for seq, cls in YCB_SEQS.items():
        paths = [os.path.join(pr.ycb_all_res_dir(str(tmp / 'video'), names[c - 1]), 'seq%d.mp4' % seq) for c in cls]
        for t in range(NFRAMES - 1):
            frames, got_paths, last = puts[k]
            k += 1
            assert got_paths == paths and last == (t == NFRAMES - 2)
            rgb = pr.read_rgb(os.path.join(ycb, 'data_organized', '%04d' % seq, 'color', '%06d-color.png' % (t + 2)))
            for j, c in enumerate(cls):
                want = OV.draw_track(rgb, synth.CAMERA_K, res[c][seq][t + 1], _model_points(pr, templates['model_path'].format(class_id=c)),
                                     'frame:%d' % (t + 2), 'under')
                assert np.array_equal(frames[j], want), (seq, c, t, int((frames[j] != want).sum()))
        for p in paths:
            cap = cv2.VideoCapture(p)
            assert cap.isOpened(), p
            assert int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) == NFRAMES - 1
            assert (int(cap.get(cv2.CAP_PROP_FRAME_WIDTH)), int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT))) == (W // 2, H // 2)
            cap.release()
    # eval_ycb.eval_all pools all 21 classes: the others' ground truth and results are copies of one of the three real classes
    for k in range(1, 22):
        if k in YCB_CLASSES:
            continue
        src = YCB_CLASSES[k % 3]
        for seq, cls in YCB_SEQS.items():
            if src in cls:
                shutil.copytree(os.path.join(ycb, 'data_organized', '%04d' % seq, 'pose_gt', str(src)),
                                os.path.join(ycb, 'data_organized', '%04d' % seq, 'pose_gt', str(k)))
        for root in (tmp / 'plain', tmp / 'video'):
            os.makedirs(os.path.join(str(root), names[k - 1]))
            os.symlink(pr.ycb_all_res_dir(str(root), names[src - 1]), pr.ycb_all_res_dir(str(root), names[k - 1]))
    E = importlib.import_module(PKG + '.eval_ycb')
    with contextlib.redirect_stdout(io.StringIO()):
        a = E.eval_all(argparse.Namespace(ycb_dir=ycb, res_root=str(tmp / 'plain')))
        b = E.eval_all(argparse.Namespace(ycb_dir=ycb, res_root=str(tmp / 'video')))
    assert a == b and a[2] > 0, (a, b)


VIDEOS = {'bleach0': 'bleach', 'sugar_box1': 'sugar'}
CAD = {'sugar': '004_sugar_box', 'bleach': '021_bleach_cleanser'}


@pytest.fixture(scope='module')
def ycbineoat_tree(tmp_path_factory, synth):
    mio = importlib.import_module(PKG + '.mesh_io')
    tmp = tmp_path_factory.mktemp('overlay_ycbineoat')
    for j, obj in enumerate(CAD):
        _write_cfg(tmp / 'cfg' / obj, synth, mio, j + 1, 180.0 + 20 * j, _camera(synth))
        (tmp / 'ycb' / 'CADmodels' / CAD[obj]).mkdir(parents=True)
        np.savetxt(str(tmp / 'ycb' / 'CADmodels' / CAD[obj] / 'points.xyz'), synth.mesh(3, seed=j + 1)['pos'].astype(np.float64))
    for v_i, v in enumerate(VIDEOS):
        base = tmp / 'data' / v
        for sub in ('rgb', 'depth_filled', 'annotated_poses'):
            (base / sub).mkdir(parents=True)
        p = synth.raw_poses(NFRAMES, seed=10 + v_i)
        p[1:, :3, 3] = p[0, :3, 3] + 0.002 * np.arange(1, NFRAMES)[:, None]
        p[1:, :3, :3] = p[0, :3, :3]
        for i in range(NFRAMES):
            rgb, depth = synth.raw_frame(seed=100 * v_i + i)
            cv2.imwrite(str(base / 'rgb' / ('%07d.png' % i)), rgb[..., ::-1])
            cv2.imwrite(str(base / 'depth_filled' / ('%07d.png' % i)), depth)
            np.savetxt(str(base / 'annotated_poses' / ('%07d.txt' % i)), p[i])
    templates = {'train_data_path': str(tmp / 'cfg' / '{object}' / 'train'), 'mean_std_path': str(tmp / 'cfg' / '{object}'),
                 'ckpt_dir': str(tmp / 'cfg' / '{object}' / 'model_best_val.pth.tar'), 'model_path': str(tmp / 'cfg' / '{object}' / 'textured.ply')}
    return tmp, templates


def test_ycbineoat_all_videos(pr, synth, ycbineoat_tree, recorder):
    tmp, templates = ycbineoat_tree
    data = str(tmp / 'data')
    plain = pr.getResultsYcbInEOAT(data, templates, str(tmp / 'plain'))
    s0, p0 = len(recorder['steps']), len(recorder['puts'])
    res = pr.main(['--mode', 'ycbineoat_all', '--YCBInEOAT_dir', data, '--outdir', str(tmp / 'video'), '--video']
                  + sum([['--' + k, v] for k, v in templates.items()], []))
    for v in VIDEOS:
        assert np.array_equal(plain[v], res[v]), v
    steps, puts = recorder['steps'][s0:], recorder['puts'][p0:]
    assert len(steps) == len(puts) == NFRAMES * len(VIDEOS)
    for s in range(0, len(steps), NFRAMES):                             # each video tracks another object
        assert all(g for _, g in steps[s + 1:s + NFRAMES]), steps
    k = 0
    for v, obj in VIDEOS.items():
        path = os.path.join(str(tmp / 'video'), v + '.mp4')
        pts = _model_points(pr, templates['model_path'].format(object=obj))
        for t in range(NFRAMES):
            frames, got_paths, last = puts[k]
            k += 1
            assert got_paths == [path] and last == (t == NFRAMES - 1)
            rgb = pr.read_rgb(os.path.join(data, v, 'rgb', '%07d.png' % t))
            want = OV.draw_track(rgb, synth.CAMERA_K, res[v][t], pts, 'frame:%d' % t, 'over')
            assert np.array_equal(frames[0], want), (v, t, int((frames[0] != want).sum()))
        cap = cv2.VideoCapture(path)
        assert cap.isOpened() and int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) == NFRAMES
        assert (int(cap.get(cv2.CAP_PROP_FRAME_WIDTH)), int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT))) == (W // 2, H // 2)
        cap.release()
    ev = importlib.import_module(PKG + '.eval_ycbineoat')
    with contextlib.redirect_stdout(io.StringIO()):
        a = ev.eval_all(argparse.Namespace(res_dir=str(tmp / 'plain') + '/', YCBInEOAT_dir=data, ycb_dir=str(tmp / 'ycb')))
        b = ev.eval_all(argparse.Namespace(res_dir=str(tmp / 'video') + '/', YCBInEOAT_dir=data, ycb_dir=str(tmp / 'ycb')))
    assert a == b and a[3] == NFRAMES * len(VIDEOS), (a, b)


def test_video_sink_raises_a_writer_error_and_releases_every_file(pkg, tmp_path):
    st = importlib.import_module(PKG + '.staging')
    dev = torch.device('cuda', torch.cuda.current_device())
    frames = torch.full((2, 24, 32, 3), 128, dtype=torch.uint8, device=dev)
    sink = st.VideoSink((2, 24, 32, 3), 2, dev)
    good = str(tmp_path / 'a.mp4')
    sink.put(frames, [good, str(tmp_path / 'no_such_dir' / 'b.mp4')])
    with pytest.raises(OSError, match='b.mp4'):                       # raised at a later frame
        for _ in range(4):
            sink.put(frames, [good, str(tmp_path / 'no_such_dir' / 'b.mp4')])
    with pytest.raises(OSError, match='b.mp4'):                       # and at close, which still releases every file
        sink.close()
    cap = cv2.VideoCapture(good)
    assert cap.isOpened() and int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) >= 1
    cap.release()
