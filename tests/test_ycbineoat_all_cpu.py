"""Host logic of the YCBInEOAT evaluation in one pass (predict.getResultsYcbInEOAT, eval_ycbineoat.eval_all): which object a video
shows, the refused folders and model paths, per-object path templates and missing files, and the output layout the drop-in reads.
CPU only; scores and tracked poses are checked on the GPU (test_gpu_ycbineoat_all.py)."""
import argparse, importlib, os
import numpy as np
import pytest
import torch
import yaml

K_INFO = {'focalX': 319.58, 'focalY': 417.12, 'centerX': 320.0, 'centerY': 244.35, 'height': 480, 'width': 640}


@pytest.fixture(scope='module')
def pr():
    return importlib.import_module('iros20-6d-pose-tracking_b200.predict')


@pytest.fixture(scope='module')
def ev():
    return importlib.import_module('iros20-6d-pose-tracking_b200.eval_ycbineoat')


def video(root, name, frames=2):
    d = root / name
    for sub in ('rgb', 'depth_filled', 'annotated_poses'):
        (d / sub).mkdir(parents=True)
    for i in range(frames):
        np.savetxt(str(d / 'annotated_poses' / ('%07d.txt' % i)), np.eye(4))
        (d / 'rgb' / ('%07d.png' % i)).write_bytes(b'')
        (d / 'depth_filled' / ('%07d.png' % i)).write_bytes(b'')
    return d


def test_video_object_is_the_first_listed_name_in_the_folder(ev):
    assert ev.OBJECTS == ['cracker', 'bleach', 'sugar', 'tomato', 'mustard']
    assert ev.video_object('bleach0') == 'bleach'
    assert ev.video_object('cracker_box_reorient') == 'cracker'
    assert ev.video_object('sugar_box_yalehand0') == 'sugar'
    assert ev.video_object('mustard_easy_00_02') == 'mustard'
    assert ev.video_object('tomato_soup_can_yalehand0') == 'tomato'
    assert ev.video_object('sugar_or_bleach') == 'bleach'                  # OBJECTS order, not position in the name
    assert ev.video_object('banana0') is None


def test_videos_found_under_the_root(pr, tmp_path):
    for name in ('sugar_box1', 'bleach0', 'cracker_box_reorient'):
        video(tmp_path, name)
    (tmp_path / 'mustard0.tar.gz').mkdir()                                # an archive entry, even with the layout, is skipped
    for sub in ('rgb', 'depth_filled', 'annotated_poses'):
        (tmp_path / 'mustard0.tar.gz' / sub).mkdir()
    (tmp_path / 'tomato_notes').mkdir()                                   # no rgb/ depth_filled/ annotated_poses/: not a video
    assert pr.ycbineoat_videos(str(tmp_path)) == [('bleach0', 'bleach'), ('cracker_box_reorient', 'cracker'), ('sugar_box1', 'sugar')]


def test_a_video_naming_no_object_is_refused(pr, ev, tmp_path):
    video(tmp_path / 'data', 'bleach0')
    bad = video(tmp_path / 'data', 'banana0')
    with pytest.raises(ValueError, match='banana0'):
        pr.ycbineoat_videos(str(tmp_path / 'data'))
    res = tmp_path / 'res'
    for v in ('bleach0', 'banana0'):
        pr.write_video_poses(str(res), v, np.stack([np.eye(4)] * 2))
    ycb = tmp_path / 'ycb'
    (ycb / 'CADmodels' / '021_bleach_cleanser').mkdir(parents=True)
    np.savetxt(str(ycb / 'CADmodels' / '021_bleach_cleanser' / 'points.xyz'), np.zeros((3, 3)))
    with pytest.raises(ValueError, match=str(res / 'banana0')):
        ev.eval_all(argparse.Namespace(res_dir=str(res) + '/', YCBInEOAT_dir=str(tmp_path / 'data'), ycb_dir=str(ycb)))
    assert bad.exists()


def test_a_model_matching_only_through_ycb_dir_is_refused(ev, tmp_path):
    ycb = tmp_path / 'sugar_runs' / 'ycb'
    for folder in ('003_cracker_box', '004_sugar_box'):
        (ycb / 'CADmodels' / folder).mkdir(parents=True)
        np.savetxt(str(ycb / 'CADmodels' / folder / 'points.xyz'), np.zeros((3, 3)))
    with pytest.raises(ValueError, match=r'003_cracker_box.*points\.xyz'):
        ev.model_points(str(ycb))
    ok = tmp_path / 'plain'
    for folder, v in (('003_cracker_box', 1.0), ('004_sugar_box', 2.0), ('021_bleach_cleanser', 3.0)):
        (ok / 'CADmodels' / folder).mkdir(parents=True)
        np.savetxt(str(ok / 'CADmodels' / folder / 'points.xyz'), np.full((4, 3), v))
    m = ev.model_points(str(ok))
    assert sorted(m) == ['bleach', 'cracker', 'sugar'] and m['sugar'].shape == (4, 3) and (m['bleach'] == 3.0).all()


def test_template_expansion(pr):
    cfg = {'train_data_path': '/w/{object}/train', 'mean_std_path': '/w/{object}', 'ckpt_dir': '/w/{object}/model_best_val.pth.tar',
           'model_path': '/m/{class_name}/textured.ply'}
    got = pr.expand_object_paths(cfg, 'sugar', '004_sugar_box')
    assert got == {'train_data_path': '/w/sugar/train', 'mean_std_path': '/w/sugar', 'ckpt_dir': '/w/sugar/model_best_val.pth.tar',
                   'model_path': '/m/004_sugar_box/textured.ply'}
    with pytest.raises(ValueError, match='class_name'):                   # {class_name} needs ycb_dir
        pr.expand_object_paths(cfg, 'sugar')
    with pytest.raises(ValueError, match='class_id'):
        pr.expand_object_paths(dict(cfg, ckpt_dir='/c/{class_id}.pth'), 'sugar', 'x')
    with pytest.raises(ValueError, match='model_path'):
        pr.expand_object_paths({k: v for k, v in cfg.items() if k != 'model_path'}, 'sugar', 'x')


def object_files(root, obj, info=None):
    d = root / obj
    (d / 'train').mkdir(parents=True)
    yaml.safe_dump(info or {'resolution': 176, 'object_width': 200.0, 'boundingbox': 10, 'camera': dict(K_INFO)}, open(d / 'dataset_info.yml', 'w'))
    np.save(d / 'mean.npy', np.full(8, 40.0, np.float32))
    np.save(d / 'std.npy', np.full(8, 5.0, np.float32))
    (d / 'ckpt.pth.tar').write_bytes(b'not a checkpoint')
    (d / 'mesh.ply').write_text('ply\n')


def templates(root):
    return {'train_data_path': str(root / '{object}' / 'train'), 'mean_std_path': str(root / '{object}'),
            'ckpt_dir': str(root / '{object}' / 'ckpt.pth.tar'), 'model_path': str(root / '{object}' / 'mesh.ply')}


@pytest.fixture
def no_device(pr, monkeypatch):
    """Every refusal comes before the driver creates its Engine, so before anything is loaded onto a device."""
    def engine(*a, **kw):
        raise AssertionError('the configuration was not checked before the Engine was created')
    monkeypatch.setattr(pr, 'Engine', engine)
    monkeypatch.setattr(pr, 'Tracker', engine)


@pytest.mark.parametrize('missing, what', [('ckpt.pth.tar', 'checkpoint'), ('mean.npy', 'mean'), ('std.npy', 'std'), ('mesh.ply', 'mesh'),
                                           ('dataset_info.yml', 'dataset_info.yml')])
def test_refuses_a_missing_file_naming_object_and_path(pr, tmp_path, no_device, missing, what):
    data, cfg = tmp_path / 'data', tmp_path / 'cfg'
    for v in ('bleach0', 'sugar1'):
        video(data, v)
    for o in ('bleach', 'sugar'):
        object_files(cfg, o)
    path = cfg / 'sugar' / missing
    os.remove(path)
    with pytest.raises(FileNotFoundError) as e:
        pr.getResultsYcbInEOAT(str(data), templates(cfg), str(tmp_path / 'out'))
    msg = str(e.value)
    assert 'object sugar' in msg and what in msg and os.path.normpath(msg.split(' at ')[-1]) == str(path)
    assert not (tmp_path / 'out').exists()


def test_refuses_objects_with_another_camera_and_unknown_class_folders(pr, tmp_path, no_device):
    data, cfg = tmp_path / 'data', tmp_path / 'cfg'
    for v in ('bleach0', 'sugar1'):
        video(data, v)
    object_files(cfg, 'bleach')
    object_files(cfg, 'sugar', {'resolution': 176, 'object_width': 200.0, 'boundingbox': 10, 'camera': dict(K_INFO, focalX=500.0)})
    with pytest.raises(ValueError, match='object sugar: camera'):
        pr.getResultsYcbInEOAT(str(data), templates(cfg), str(tmp_path / 'out'))
    ycb = tmp_path / 'ycb'
    (ycb / 'CADmodels' / '021_bleach_cleanser').mkdir(parents=True)
    with pytest.raises(FileNotFoundError, match='object sugar'):                       # no CADmodels/ folder for {class_name}
        pr.getResultsYcbInEOAT(str(data), templates(cfg), str(tmp_path / 'out'), ycb_dir=str(ycb))
    with pytest.raises(ValueError, match='decode_ahead'):
        pr.getResultsYcbInEOAT(str(data), templates(cfg), str(tmp_path / 'out'), decode_ahead=0)


class FakeEngine:
    """What eval_all asks of the Engine, on the CPU: records the poses it is given and scores every pose 0.01 m."""
    device = torch.device('cpu')

    def add_adi_sets(self, points, pose_set, pred, gt):
        self.points, self.pose_set, self.pred, self.gt = points, np.asarray(pose_set), pred.numpy(), gt.numpy()
        e = torch.full((len(pose_set),), 0.01, dtype=torch.float64)
        return e, e

    def vocap_sets(self, errs, err_set, n_sets):
        self.err_set = err_set.numpy()
        return np.zeros(n_sets + 1)


def test_driver_output_layout_is_what_eval_all_reads(pr, ev, tmp_path, monkeypatch, capsys):
    data, ycb, out = tmp_path / 'data', tmp_path / 'ycb', tmp_path / 'out'
    n = {'bleach0': 3, 'sugar_box1': 12, 'cracker_box_reorient': 2}
    for v, nf in n.items():
        video(data, v, nf)
        for i in range(nf):
            np.savetxt(str(data / v / 'annotated_poses' / ('%07d.txt' % i)), np.eye(4) * (i + 1))
    for folder in ('003_cracker_box', '004_sugar_box', '021_bleach_cleanser'):
        (ycb / 'CADmodels' / folder).mkdir(parents=True)
        np.savetxt(str(ycb / 'CADmodels' / folder / 'points.xyz'), np.ones((5, 3)))
    poses = {v: np.stack([np.eye(4) + 0.001 * i for i in range(nf)]) for v, nf in n.items()}
    for v, p in poses.items():
        pr.write_video_poses(str(out), v, p)
    (out / 'old_run.tar.gz').write_bytes(b'')
    fake = FakeEngine()
    U = importlib.import_module('iros20-6d-pose-tracking_b200.Utils')
    monkeypatch.setattr(U, '_eng', lambda: fake)
    per_object, adi, add, total = ev.eval_all(argparse.Namespace(res_dir=str(out) + '/', YCBInEOAT_dir=str(data), ycb_dir=str(ycb)))
    assert total == sum(n.values()) and set(per_object) == set(ev.OBJECTS)
    folders = [f for f in os.listdir(str(out)) if '.tar.gz' not in f]
    lines = capsys.readouterr().out.splitlines()
    assert lines[:3] == folders and lines[3:8] == ['%s: adi=0.0 add=0.0' % o for o in ev.OBJECTS]
    assert lines[8:] == ['Total pose: %d' % total, '', 'Overall, adi=0.0 add=0.0']
    # every written pose, in frame order, paired with the ground truth of the same frame and the video's object
    want_pred = np.concatenate([poses[f] for f in folders])
    want_gt = np.concatenate([np.stack([np.eye(4) * (i + 1) for i in range(n[f])]) for f in folders])
    assert np.array_equal(fake.pred, want_pred) and np.array_equal(fake.gt, want_gt)
    objs = [ev.video_object(f) for f in folders for _ in range(n[f])]
    assert list(fake.err_set) == [ev.OBJECTS.index(o) for o in objs]
    used = [o for o in ev.OBJECTS if o in ('cracker', 'sugar', 'bleach')]
    assert list(fake.pose_set) == [used.index(o) for o in objs]
    # a video with more poses than ground truth files: the reference's assertion
    pr.write_video_poses(str(out), 'bleach0', np.stack([np.eye(4)] * 4))
    with pytest.raises(AssertionError, match='#pred_files:4, #gt_files:3'):
        ev.eval_all(argparse.Namespace(res_dir=str(out) + '/', YCBInEOAT_dir=str(data), ycb_dir=str(ycb)))


def test_cli_passes_templates_and_options(pr, tmp_path, monkeypatch):
    calls = []
    monkeypatch.setattr(pr, 'getResultsYcbInEOAT', lambda *a, **kw: calls.append((a, kw)) or {})
    base = ['--mode', 'ycbineoat_all', '--YCBInEOAT_dir', str(tmp_path), '--ckpt_dir', '/c/{object}.pth.tar', '--mean_std_path', '/s/{object}',
            '--train_data_path', '/t/{object}/train', '--model_path', '/m/{class_name}.ply', '--outdir', str(tmp_path / 'o')]
    pr.main(base + ['--decode_ahead', '2', '--max_frames', '5', '--ycb_dir', '/ycb'])
    (a, kw), = calls
    assert a[0] == str(tmp_path) and a[1] == {'train_data_path': '/t/{object}/train', 'mean_std_path': '/s/{object}',
                                              'ckpt_dir': '/c/{object}.pth.tar', 'model_path': '/m/{class_name}.ply'}
    assert kw == {'max_frames': 5, 'decode_ahead': 2, 'ycb_dir': '/ycb'}
    with pytest.raises(SystemExit):
        pr.main(base + ['--score'])                                       # scoring needs the model points under --ycb_dir
