"""Host logic of the one-pass YCB-Video driver (predict.getResultsYcbAll): per-class path templates, the track set of each test
sequence, the output folders eval_ycb.eval_all reads, and the configurations it refuses before anything reaches a device.
CPU only; the tracked poses are checked on the GPU (test_gpu_ycb_all.py)."""
import argparse, importlib, os
import numpy as np
import pytest
import yaml

K_INFO = {'focalX': 1066.778, 'focalY': 1067.487, 'centerX': 312.9869, 'centerY': 241.3109, 'height': 480, 'width': 640}


@pytest.fixture(scope='module')
def pr():
    return importlib.import_module('iros20-6d-pose-tracking_b200.predict')


def cad_models(ycb, n=21):
    names = ['%03d_object_%s' % (k, 'abcdefghijklmnopqrstu'[k - 1]) for k in range(1, n + 1)]
    for name in names:
        (ycb / 'CADmodels' / name).mkdir(parents=True)
    return names


def class_files(root, class_id, info=None, mean=None):
    """<root>/c<id>/{train/, dataset_info.yml, mean.npy, std.npy, ckpt.pth.tar, mesh.ply}: placeholders, never loaded here."""
    d = root / ('c%d' % class_id)
    (d / 'train').mkdir(parents=True)
    yaml.safe_dump(info or {'resolution': 176, 'object_width': 200.0, 'boundingbox': 10, 'camera': dict(K_INFO)}, open(d / 'dataset_info.yml', 'w'))
    np.save(d / 'mean.npy', np.full(8, 40.0, np.float32) if mean is None else mean)
    np.save(d / 'std.npy', np.full(8, 5.0, np.float32))
    (d / 'ckpt.pth.tar').write_bytes(b'not a checkpoint')
    (d / 'mesh.ply').write_text('ply\n')
    return d


def templates(root):
    return {'train_data_path': str(root / 'c{class_id}' / 'train'), 'mean_std_path': str(root / 'c{class_id}'),
            'ckpt_dir': str(root / 'c{class_id}' / 'ckpt.pth.tar'), 'model_path': str(root / 'c{class_id}' / 'mesh.ply')}


def test_template_expansion(pr):
    cfg = {'train_data_path': '/w/{class_name}/train', 'mean_std_path': '/w/{class_name}',
           'ckpt_dir': '/w/{class_id:02d}/model_best_val.pth.tar', 'model_path': '/m/{class_name}/textured_{class_id}.ply'}
    got = pr.expand_class_paths(cfg, 2, '002_master_chef_can')
    assert got == {'train_data_path': '/w/002_master_chef_can/train', 'mean_std_path': '/w/002_master_chef_can',
                   'ckpt_dir': '/w/02/model_best_val.pth.tar', 'model_path': '/m/002_master_chef_can/textured_2.ply'}
    assert pr.expand_class_paths(dict(cfg, ckpt_dir='/fixed.pth.tar'), 5, 'x')['ckpt_dir'] == '/fixed.pth.tar'
    with pytest.raises(ValueError, match='class_seq'):
        pr.expand_class_paths(dict(cfg, model_path='/m/{class_seq}.ply'), 2, 'x')        # unknown placeholder
    with pytest.raises(ValueError, match='model_path'):
        pr.expand_class_paths({k: v for k, v in cfg.items() if k != 'model_path'}, 2, 'x')


def test_track_sets_per_sequence(pr, tmp_path):
    data = tmp_path / 'data_organized'
    for seq, classes in ((47, [1, 4]), (48, [9, 4, 2]), (50, [9]), (52, [3]), (59, [4, 21]), (60, [4])):
        for c in classes:
            (data / ('%04d' % seq) / 'pose_gt' / str(c)).mkdir(parents=True)
    # test sequences only (0048..0059), requested classes only, ascending; a sequence with none of them has no track set
    assert pr.ycb_track_sets(str(tmp_path), [9, 4, 21, 2]) == {48: [2, 4, 9], 50: [9], 59: [4, 21]}
    assert pr.ycb_track_sets(str(tmp_path), [4]) == {48: [4], 59: [4]}
    for c in (2, 4, 9, 21):                                           # the sequences a per-class getResultsYcb run visits
        want = pr.findClassContainedVideosYcb(c, str(data) + '/', testset=True)
        assert [s for s, cls in pr.ycb_track_sets(str(tmp_path), [2, 4, 9, 21]).items() if c in cls] == want


def test_output_folders_map_to_class_ids_in_eval_all(pr, tmp_path, monkeypatch):
    E = importlib.import_module('iros20-6d-pose-tracking_b200.eval_ycb')
    ycb = tmp_path / 'ycb'
    names = cad_models(ycb)
    assert pr.ycb_class_names(str(ycb)) == names
    out = tmp_path / 'out'
    for name in reversed(names):                                      # creation order must not matter
        os.makedirs(os.path.join(pr.ycb_all_res_dir(str(out), name), 'seq48'))
    seen = {}

    def fake_eval_one_class(args):
        seen[args.class_id] = args.res_dir
        return np.array([0.01]), np.array([0.02])
    monkeypatch.setattr(E, 'eval_one_class', fake_eval_one_class)
    monkeypatch.setattr(E, 'VOCap', lambda errs: 0.5)
    E.eval_all(argparse.Namespace(ycb_dir=str(ycb), res_root=str(out)))
    assert sorted(seen) == list(range(1, 22))
    for c, res_dir in seen.items():
        assert res_dir == pr.ycb_all_res_dir(str(out), names[c - 1]) + '/'
        # eval_one_class reads the sequence id from the first path component under res_dir
        assert os.listdir(res_dir) == ['seq48']


@pytest.fixture
def no_device(pr, monkeypatch):
    """Every refusal comes before the driver creates its Engine, so before any checkpoint is loaded onto a device."""
    def engine(*a, **kw):
        raise AssertionError('the configuration was not checked before the Engine was created')
    monkeypatch.setattr(pr, 'Engine', engine)
    monkeypatch.setattr(pr, 'Tracker', engine)


def refusal_tree(tmp_path, infos=None):
    ycb = tmp_path / 'ycb'
    cad_models(ycb, 5)
    for c in (2, 4):
        (ycb / 'data_organized' / '0048' / 'pose_gt' / str(c)).mkdir(parents=True)
    root = tmp_path / 'cfg'
    for c in (2, 4):
        class_files(root, c, (infos or {}).get(c))
    return ycb, root


def info_with(**changes):
    info = {'resolution': 176, 'object_width': 200.0, 'boundingbox': 10, 'camera': dict(K_INFO)}
    for k, v in changes.items():
        if k in K_INFO:
            info['camera'][k] = v
        else:
            info[k] = v
    return info


def test_accepts_matching_classes(pr, tmp_path, no_device):
    ycb, root = refusal_tree(tmp_path)
    classes = pr.ycb_all_classes(str(ycb), [4, 2], templates(root))
    assert [k['class_id'] for k in classes] == [2, 4] and [k['name'] for k in classes] == ['002_object_b', '004_object_d']
    assert classes[1]['ckpt_dir'] == str(root / 'c4' / 'ckpt.pth.tar')
    assert classes[0]['trans_normalizer'] == 0.03 and classes[0]['rot_normalizer'] == 5 * np.pi / 180    # getResultsYcb's Tracker


@pytest.mark.parametrize('changes, what', [({'focalX': 1000.0}, 'camera'), ({'centerY': 240.0}, 'camera'), ({'width': 320}, 'camera'),
                                           ({'renderer': 'pyrenderer'}, 'renderer')])
def test_refuses_a_class_with_another_camera(pr, tmp_path, no_device, changes, what):
    ycb, root = refusal_tree(tmp_path, {4: info_with(**changes)})
    with pytest.raises(ValueError, match=r'class 4 \(004_object_d\): %s' % what):
        pr.getResultsYcbAll(str(ycb), [2, 4], templates(root), str(tmp_path / 'out'))


def test_refuses_another_resolution(pr, tmp_path, no_device):
    ycb, root = refusal_tree(tmp_path, {2: info_with(resolution=128), 4: info_with(resolution=128)})
    with pytest.raises(ValueError, match=r'class 2 \(002_object_b\): resolution 128'):
        pr.getResultsYcbAll(str(ycb), [2, 4], templates(root), str(tmp_path / 'out'))


def test_refuses_mismatched_normalisers(pr, tmp_path, no_device):
    ycb, root = refusal_tree(tmp_path)
    cfg = templates(root)
    for key, v in (('trans_normalizer', {2: 0.03, 4: 0.02}), ('rot_normalizer', {2: 5 * np.pi / 180, 4: 15 * np.pi / 180})):
        with pytest.raises(ValueError, match=r'class 4 \(004_object_d\): %s' % key):
            pr.getResultsYcbAll(str(ycb), [2, 4], dict(cfg, **{key: v}), str(tmp_path / 'out'))
    assert len(pr.ycb_all_classes(str(ycb), [2, 4], dict(cfg, trans_normalizer=0.02, rot_normalizer={2: 0.1, 4: 0.1}))) == 2


def test_refuses_unknown_precision_and_class(pr, tmp_path, no_device):
    ycb, root = refusal_tree(tmp_path)
    with pytest.raises(ValueError, match='precision'):
        pr.getResultsYcbAll(str(ycb), [2, 4], templates(root), str(tmp_path / 'out'), precision='fp16')
    with pytest.raises(ValueError, match='class 6'):
        pr.getResultsYcbAll(str(ycb), [2, 6], templates(root), str(tmp_path / 'out'))


@pytest.mark.parametrize('missing, what', [('ckpt.pth.tar', 'checkpoint'), ('mean.npy', 'mean'), ('std.npy', 'std'), ('mesh.ply', 'mesh'),
                                           ('dataset_info.yml', 'dataset_info.yml')])
def test_refuses_a_missing_file_naming_class_and_path(pr, tmp_path, no_device, missing, what):
    ycb, root = refusal_tree(tmp_path)
    path = root / 'c4' / missing
    os.remove(path)
    with pytest.raises(FileNotFoundError) as e:
        pr.getResultsYcbAll(str(ycb), [2, 4], templates(root), str(tmp_path / 'out'))
    msg = str(e.value)
    assert 'class 4 (004_object_d)' in msg and what in msg and os.path.normpath(msg.split(' at ')[-1]) == str(path)
    assert not (tmp_path / 'out').exists()                            # nothing was written either


def test_cli_parses_class_ids_and_passes_templates(pr, tmp_path, monkeypatch):
    ycb = tmp_path / 'ycb'
    cad_models(ycb)
    calls = []
    monkeypatch.setattr(pr, 'getResultsYcbAll', lambda *a, **kw: calls.append((a, kw)) or {})
    base = ['--mode', 'ycbv_all', '--ycb_dir', str(ycb), '--ckpt_dir', '/c/{class_id}.pth.tar', '--mean_std_path', '/s/{class_name}',
            '--train_data_path', '/t/{class_name}/train', '--model_path', '/m/{class_name}.ply', '--outdir', str(tmp_path / 'o')]
    pr.main(base + ['--class_ids', '5,1,3', '--init', 'posecnn'])
    pr.main(base + ['--class_ids', 'all', '--max_frames', '7'])
    (a0, kw0), (a1, kw1) = calls
    assert a0[1] == [1, 3, 5] and kw0['initialize_method'] == 'posecnn' and a1[1] == list(range(1, 22)) and kw1['max_frames'] == 7
    assert a0[2] == {'train_data_path': '/t/{class_name}/train', 'mean_std_path': '/s/{class_name}', 'ckpt_dir': '/c/{class_id}.pth.tar',
                     'model_path': '/m/{class_name}.ply'}
    with pytest.raises(SystemExit):
        pr.main(base + ['--class_ids', 'one,two'])
