"""The one-pass YCB-Video driver (predict.getResultsYcbAll) on a synthetic data set in the YCB-Video layout: two test sequences,
three classes with their own weights, statistics, meshes and widths (class 7 only in sequence 0048, so the two sequences track
3 and 2 objects), six frames each.

  * bit for bit what a plain loop of Tracker.on_track_batch computes over the same frames, tracks, ids and widths (bf16x3, bf16)
  * every step after the first of a sequence is a CUDA graph replay with the launches of one track_render step
  * bit for bit what per-class getResultsYcb runs (n = 1 steps, one weight set each) compute, pose by pose, and so equal
    eval_ycb.eval_all AUCs: the sequences track 3 and 2 objects, so both runs are in the trunk's split-K latency mode (n <= 4),
    where a track's results depend neither on n nor on the weight sets of the other tracks
  * PoseCNN / PoseRBPF initialisation: each track's first pose is the one getResultsYcb starts that class from
"""
import argparse, importlib, os, shutil
import numpy as np
import pytest
import torch
import yaml

pytestmark = pytest.mark.gpu

CLASSES = (2, 5, 7)
SEQS = {48: (2, 5, 7), 49: (2, 5)}
NFRAMES = 6
WIDTHS = {2: 180.0, 5: 200.0, 7: 230.0}
KEYFRAMES = ['0048/000001', '0048/000003', '0048/000006', '0049/000001', '0049/000004']


@pytest.fixture(scope='module')
def pr():
    return importlib.import_module('iros20-6d-pose-tracking_b200.predict')


@pytest.fixture(scope='module')
def tree(tmp_path_factory, synth):
    """<tmp>/ycb: the data set (21 CADmodels folders, keyframe.txt, PoseCNN and PoseRBPF result files); <tmp>/cfg/c<id>: each
    class's dataset_info.yml, mean/std, checkpoint and mesh; -> (tmp, templates, gt poses {(seq, class): (NFRAMES,4,4)})."""
    import cv2, scipy.io
    from scipy.spatial.transform import Rotation
    mio = importlib.import_module('iros20-6d-pose-tracking_b200.mesh_io')
    tmp = tmp_path_factory.mktemp('ycb_all')
    ycb, cfg = tmp / 'ycb', tmp / 'cfg'
    K = synth.CAMERA_K
    cam = {'focalX': float(K[0, 0]), 'focalY': float(K[1, 1]), 'centerX': float(K[0, 2]), 'centerY': float(K[1, 2]), 'height': 480, 'width': 640}
    mean, std = synth.default_mean_std()
    for c in CLASSES:
        d = cfg / ('c%d' % c)
        (d / 'train').mkdir(parents=True)
        yaml.safe_dump({'resolution': 176, 'object_width': WIDTHS[c], 'boundingbox': 10, 'camera': cam}, open(d / 'dataset_info.yml', 'w'))
        np.save(d / 'mean.npy', mean + c); np.save(d / 'std.npy', std * (1 + 0.05 * c))
        torch.save({'epoch': 1, 'state_dict': synth.make_state_dict(c), 'best_prec': 0.0}, str(d / 'model_best_val.pth.tar'))
        mio.save_ply_mesh(str(d / 'textured.ply'), synth.mesh(3, seed=c))
    for k in range(1, 22):
        (ycb / 'CADmodels' / ('%03d_obj' % k)).mkdir(parents=True)
        mesh_of = k if k in CLASSES else CLASSES[k % 3]
        np.savetxt(str(ycb / 'CADmodels' / ('%03d_obj' % k) / 'points.xyz'), synth.mesh(3, seed=mesh_of)['pos'].astype(np.float64))
    gt = {}
    for seq, cls in SEQS.items():
        base = ycb / 'data_organized' / ('%04d' % seq)
        for d in ['color', 'depth_filled', 'seg'] + ['pose_gt/%d' % c for c in cls]:
            (base / d).mkdir(parents=True)
        for i in range(NFRAMES):
            rgb, depth = synth.raw_frame(seed=100 * seq + i)
            cv2.imwrite(str(base / 'color' / ('%06d-color.png' % (i + 1))), rgb[..., ::-1])
            cv2.imwrite(str(base / 'depth_filled' / ('%06d-depth.png' % (i + 1))), depth)
        for c in cls:
            p = synth.raw_poses(NFRAMES, seed=10 * seq + c)
            p[1:, :3, 3] = p[0, :3, 3] + 0.002 * np.arange(1, NFRAMES)[:, None]
            p[1:, :3, :3] = p[0, :3, :3]
            gt[seq, c] = p
            for i in range(NFRAMES):
                np.savetxt(str(base / 'pose_gt' / str(c) / ('%06d.txt' % (i + 1))), p[i])
    (ycb / 'image_sets').mkdir()
    (ycb / 'image_sets' / 'keyframe.txt').write_text('\n'.join(KEYFRAMES) + '\n')
    (ycb / 'YCB_Video_toolbox').mkdir()
    shutil.copy(str(ycb / 'image_sets' / 'keyframe.txt'), str(ycb / 'YCB_Video_toolbox' / 'keyframe.txt'))

    def moved(pose, seed):                                            # an estimate a few mm and degrees off the ground truth
        rng = np.random.default_rng(seed)
        out = pose.copy()
        out[:3, :3] = Rotation.from_rotvec(rng.normal(0, 0.03, 3)).as_matrix() @ pose[:3, :3]
        out[:3, 3] += rng.normal(0, 0.004, 3)
        return out

    def to_icp(pose):
        q = Rotation.from_matrix(pose[:3, :3]).as_quat()              # x y z w
        return np.r_[q[3], q[0], q[1], q[2], pose[:3, 3]]
    pc = ycb / 'YCB_Video_toolbox' / 'results_PoseCNN_RSS2018'
    pc.mkdir()
    for idx, kf in enumerate(KEYFRAMES):
        seq, frame = int(kf[:4]), int(kf[5:]) - 1
        cls = SEQS[seq]
        scipy.io.savemat(str(pc / ('%06d.mat' % idx)), {'rois': np.array([[0, c, 0, 0, 0, 0] for c in cls], dtype=np.float64),
                                                        'poses_icp': np.stack([to_icp(moved(gt[seq, c][frame], 1000 * idx + c)) for c in cls])})
    rb = ycb / 'YCB_Video_toolbox' / 'PoseRBPF_Results' / 'YCB_results_RGBD'
    for k in range(1, 22):
        seqs_k = [s for s, cls in SEQS.items() if k in cls]
        for j, seq in enumerate(seqs_k):
            d = rb / ('%02d_obj' % k) / ('seq_%d' % (j + 1))
            d.mkdir(parents=True)
            p = moved(gt[seq, k][0], 7 * k + seq)
            q = Rotation.from_matrix(p[:3, :3]).as_quat()
            (d / 'Pose_est.txt').write_text('1 %d ' % k + ' '.join('%.17g' % v for v in (*p[:3, 3], q[3], q[0], q[1], q[2])) + '\n')
        if not seqs_k:
            (rb / ('%02d_obj' % k)).mkdir(parents=True)
    templates = {'train_data_path': str(cfg / 'c{class_id}' / 'train'), 'mean_std_path': str(cfg / 'c{class_id}'),
                 'ckpt_dir': str(cfg / 'c{class_id}' / 'model_best_val.pth.tar'), 'model_path': str(cfg / 'c{class_id}' / 'textured.ply')}
    return tmp, templates, gt


@pytest.fixture(scope='module')
def steps(pr):
    """Every Engine.track_render call of the module: (n, last_step_was_graph, last_launch_count)."""
    E = pr.Engine
    orig = E.track_render
    rec = []

    def track_render(self, *a, **kw):
        out = orig(self, *a, **kw)
        rec.append((int(a[3].shape[0]), self.last_step_was_graph(), self.last_launch_count()))
        return out
    E.track_render = track_render
    yield rec
    E.track_render = orig


@pytest.fixture(scope='module')
def driver_runs(pr, tree, steps):
    """The driver through the CLI (bf16x3, scored) and through the Python call in bf16, with the steps each made."""
    tmp, templates, _ = tree
    ycb = str(tmp / 'ycb')
    runs = {}
    n0 = len(steps)
    runs['bf16x3'] = pr.main(['--mode', 'ycbv_all', '--ycb_dir', ycb, '--class_ids', ','.join(map(str, CLASSES)), '--outdir', str(tmp / 'all_bf16x3'),
                              '--score'] + sum([['--' + k, v] for k, v in templates.items()], []))
    runs['bf16x3_steps'] = steps[n0:]
    n0 = len(steps)
    runs['bf16'] = pr.getResultsYcbAll(ycb, list(CLASSES), templates, str(tmp / 'all_bf16'), precision='bf16')
    runs['bf16_steps'] = steps[n0:]
    return runs


def read_seq(pr, ycb, seq):
    base = os.path.join(ycb, 'data_organized', '%04d' % seq)
    return [(pr.read_rgb(os.path.join(base, 'color', '%06d-color.png' % (i + 1))),
             pr.read_depth(os.path.join(base, 'depth_filled', '%06d-depth.png' % (i + 1)))) for i in range(NFRAMES)]


@pytest.mark.parametrize('precision', ['bf16x3', 'bf16'])
def test_bit_identical_to_a_frame_by_frame_on_track_batch_loop(pkg, pr, tree, driver_runs, precision):
    tmp, templates, gt = tree
    ycb = str(tmp / 'ycb')
    res = driver_runs[precision]
    assert sorted(res) == list(CLASSES) and sorted(res[7]) == [48] and sorted(res[2]) == [48, 49]
    classes = pr.ycb_all_classes(ycb, CLASSES, templates, precision)
    eng = pkg.Engine(max_batch=3)
    trk = {k['class_id']: pkg.Tracker(k['dataset_info'], k['mean'], k['std'], k['ckpt_dir'], model_path=k['model_path'], engine=eng,
                                      weight_id=k['class_id'], precision=precision) for k in classes}
    dev = eng.device
    for seq, cls in SEQS.items():
        ids = np.asarray(cls, dtype=np.int32)
        widths = torch.tensor([WIDTHS[c] for c in cls], dtype=torch.float64, device=dev)
        poses = torch.from_numpy(np.stack([gt[seq, c][0] for c in cls])).to(dev)
        loop = [poses.cpu().numpy()]
        for rgb, depth in read_seq(pr, ycb, seq)[1:]:
            poses = trk[cls[0]].on_track_batch(poses, torch.from_numpy(rgb).to(dev), torch.from_numpy(depth).to(dev),
                                               weight_ids=ids, object_width=widths)
            loop.append(poses.cpu().numpy())
        loop = np.stack(loop)
        for j, c in enumerate(cls):
            assert np.array_equal(res[c][seq], loop[:, j]), 'class %d seq %d: max |diff| %.3g' % (c, seq, np.abs(res[c][seq] - loop[:, j]).max())
            files = np.stack([np.loadtxt(os.path.join(pr.ycb_all_res_dir(str(tmp / ('all_' + precision)), '%03d_obj' % c), 'seq%d' % seq,
                                                      '%07d.txt' % i)) for i in range(NFRAMES)])
            assert np.array_equal(files, loop[:, j])                 # np.savetxt's %.18e round-trips a float64
    eng.close()


def test_every_step_after_the_first_is_a_graph_replay(pkg, synth, driver_runs):
    for precision in ('bf16x3', 'bf16'):
        rec = driver_runs[precision + '_steps']
        ns = [n for n, _, _ in rec]
        assert ns == [3] * (NFRAMES - 1) + [2] * (NFRAMES - 1), ns                     # one step per frame, sequence by sequence
        for s0 in (0, NFRAMES - 1):
            assert all(g for _, g, _ in rec[s0 + 1:s0 + NFRAMES - 1]), rec
        # the launches of a single track_render step at that n
        eng = pkg.Engine(max_batch=3)
        mean, std = synth.default_mean_std()
        for w in (2, 5):
            eng.load_state_dict(synth.make_state_dict(w), w); eng.set_stats(mean, std, w); eng.set_mesh(synth.mesh(3, seed=w), w)
        rgb, depth = synth.raw_frame(seed=1)
        dev = eng.device
        for n in (3, 2):
            ids = np.array([2, 5, 5][:n], dtype=np.int32)
            eng.track_render(torch.from_numpy(rgb).to(dev), torch.from_numpy(depth).to(dev), synth.CAMERA_K,
                             torch.from_numpy(synth.raw_poses(n, seed=2)).to(dev), torch.full((n,), 200.0, dtype=torch.float64, device=dev),
                             0.03, 5 * np.pi / 180, weight_ids_host=ids, precision=precision)
            single = eng.last_launch_count()
            assert all(lc == single for m, _, lc in rec if m == n), (n, single, rec)
        eng.close()


def test_equal_to_per_class_runs_and_their_scores(pr, tree, driver_runs):
    tmp, templates, gt = tree
    ycb = str(tmp / 'ycb')
    res = driver_runs['bf16x3']
    names = pr.ycb_class_names(ycb)
    per_class = tmp / 'per_class'
    for k in pr.ycb_all_classes(ycb, CLASSES, templates):
        c = k['class_id']
        one = pr.getResultsYcb(ycb, c, k['dataset_info'], k['mean'], k['std'], k['ckpt_dir'], k['model_path'],
                               pr.ycb_all_res_dir(str(per_class), names[c - 1]), max_batch=1)
        assert sorted(one) == sorted(res[c])
        for seq in one:
            got_dir = os.path.join(pr.ycb_all_res_dir(str(tmp / 'all_bf16x3'), names[c - 1]), 'seq%d' % seq)
            want_dir = os.path.join(pr.ycb_all_res_dir(str(per_class), names[c - 1]), 'seq%d' % seq)
            assert sorted(os.listdir(got_dir)) == sorted(os.listdir(want_dir)) == ['%07d.txt' % i for i in range(NFRAMES)]
            assert np.array_equal(res[c][seq], one[seq]), 'class %d seq %d: max |pose diff| %.3g' % (c, seq, np.abs(res[c][seq] - one[seq]).max())
            for i in range(NFRAMES):                                  # and the files each run wrote
                assert np.array_equal(np.loadtxt(os.path.join(got_dir, '%07d.txt' % i)), np.loadtxt(os.path.join(want_dir, '%07d.txt' % i)))

    # eval_all over both roots: the other 18 classes' folders and ground truth are copies of one of the three real classes
    for k in range(1, 22):
        if k in CLASSES:
            continue
        src = CLASSES[k % 3]
        for seq, cls in SEQS.items():
            if src in cls:
                shutil.copytree(os.path.join(ycb, 'data_organized', '%04d' % seq, 'pose_gt', str(src)),
                                os.path.join(ycb, 'data_organized', '%04d' % seq, 'pose_gt', str(k)))
        for root in (tmp / 'all_bf16x3', per_class):
            os.makedirs(os.path.join(str(root), names[k - 1]))
            os.symlink(pr.ycb_all_res_dir(str(root), names[src - 1]), pr.ycb_all_res_dir(str(root), names[k - 1]))
    E = importlib.import_module('iros20-6d-pose-tracking_b200.eval_ycb')
    a = E.eval_all(argparse.Namespace(ycb_dir=ycb, res_root=str(tmp / 'all_bf16x3')))
    b = E.eval_all(argparse.Namespace(ycb_dir=ycb, res_root=str(per_class)))
    src_of = {k: k if k in CLASSES else CLASSES[k % 3] for k in range(1, 22)}
    assert a[2] == b[2] == sum(src_of[k] in SEQS[int(kf[:4])] for kf in KEYFRAMES for k in range(1, 22))
    assert a[0] == b[0] and a[1] == b[1], (a, b)


@pytest.mark.parametrize('method', ['posecnn', 'poserbpf'])
def test_init_methods_start_each_track_where_getResultsYcb_starts_it(pr, tree, method):
    tmp, templates, gt = tree
    ycb = str(tmp / 'ycb')
    res = pr.getResultsYcbAll(ycb, list(CLASSES), templates, str(tmp / ('init_' + method)), initialize_method=method, max_frames=1)
    for k in pr.ycb_all_classes(ycb, CLASSES, templates):
        c = k['class_id']
        one = pr.getResultsYcb(ycb, c, k['dataset_info'], k['mean'], k['std'], k['ckpt_dir'], k['model_path'],
                               str(tmp / ('init1_%s_%d' % (method, c))), initialize_method=method, max_frames=0, max_batch=1)
        assert sorted(one) == sorted(res[c])
        for seq in one:
            assert np.array_equal(res[c][seq][0], one[seq][0])
            assert np.abs(res[c][seq][0] - gt[seq, c][0]).max() > 1e-3          # really the estimate, not the ground truth
            assert res[c][seq].shape == (2, 4, 4)
