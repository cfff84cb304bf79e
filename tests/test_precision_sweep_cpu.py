"""Host logic of the one-pass drivers' precision sweeps (getResultsYcbAll / getResultsYcbInEOAT with a list of modes or 'all', and
predict --precision): which modes a sweep runs, what it refuses before anything reaches a device, where each mode's tree goes,
and which mode the drift is measured from.  CPU only; the tracked poses and scores are checked on the GPU
(test_gpu_precision_sweep.py)."""
import importlib, os
import numpy as np
import pytest
import yaml

K_INFO = {'focalX': 319.58, 'focalY': 417.12, 'centerX': 320.0, 'centerY': 244.35, 'height': 480, 'width': 640}


@pytest.fixture(scope='module')
def pr():
    return importlib.import_module('iros20-6d-pose-tracking_b200.predict')


@pytest.fixture
def no_device(pr, monkeypatch):
    """Every refusal comes before the driver creates its Engine, so before anything is loaded onto a device."""
    def engine(*a, **kw):
        raise AssertionError('the configuration was not checked before the Engine was created')
    monkeypatch.setattr(pr, 'Engine', engine)
    monkeypatch.setattr(pr, 'Tracker', engine)


def test_precisions_are_every_engine_mode(pr):
    from importlib import import_module
    PREC = import_module('iros20-6d-pose-tracking_b200.engine').PREC
    assert sorted(pr.PRECISIONS) == sorted(PREC) and len(set(pr.PRECISIONS)) == len(PREC)
    assert set(pr.YCB_ALL_PRECISIONS) == set(PREC) - {'fp16'}


def test_precision_modes(pr):
    assert pr.precision_modes('bf16', pr.PRECISIONS) == (('bf16',), False)
    assert pr.precision_modes('fp16', pr.YCB_ALL_PRECISIONS) == (('fp16',), False)       # a single name is checked where it always was
    assert pr.precision_modes('all', pr.PRECISIONS) == (pr.PRECISIONS, True)
    assert pr.precision_modes('all', pr.YCB_ALL_PRECISIONS) == (pr.YCB_ALL_PRECISIONS, True)
    assert pr.precision_modes(['fp8', 'bf16x3'], pr.PRECISIONS) == (('fp8', 'bf16x3'), True)
    assert pr.precision_modes(('fp32',), pr.PRECISIONS) == (('fp32',), True)
    with pytest.raises(ValueError, match='no precision'):
        pr.precision_modes([], pr.PRECISIONS)
    with pytest.raises(ValueError, match="'fp4'"):
        pr.precision_modes(['bf16', 'fp4'], pr.PRECISIONS)
    with pytest.raises(ValueError, match='bf16 listed more than once'):
        pr.precision_modes(['bf16', 'fp8', 'bf16'], pr.PRECISIONS)
    with pytest.raises(ValueError, match="precision 'fp16'"):
        pr.precision_modes(['bf16', 'fp16'], pr.YCB_ALL_PRECISIONS)


def test_reference_mode(pr):
    assert pr.sweep_reference(pr.PRECISIONS) == 'fp32'
    assert pr.sweep_reference(('fp8', 'fp32', 'bf16x3')) == 'fp32'
    assert pr.sweep_reference(('fp8', 'bf16', 'bf16x3')) == 'bf16x3'
    assert pr.sweep_reference(('fp8', 'bf16')) == 'fp8'
    assert pr.sweep_reference(('tf32',)) == 'tf32'


def test_cli_parses_precision(pr):
    assert pr.cli_precision(None, 'ycbineoat_all') is None
    assert pr.cli_precision('fp8', 'ycbv') == 'fp8'
    assert pr.cli_precision('all', 'ycbineoat_all') == 'all'
    assert pr.cli_precision('all', 'ycbv_all') == 'all'
    assert pr.cli_precision('bf16x3, fp8,fp16', 'ycbineoat_all') == ['bf16x3', 'fp8', 'fp16']
    for text, mode in (('fp4', 'ycbv'), ('bf16,bf16', 'ycbineoat_all'), ('bf16,fp4', 'ycbineoat_all'), ('bf16,fp16', 'ycbv_all'),
                       (',', 'ycbineoat_all'), ('fp32,', 'ycbineoat_all')):
        with pytest.raises(SystemExit):
            pr.cli_precision(text, mode)


@pytest.mark.parametrize('mode', ['ycbv', 'ycbineoat', 'class'])
@pytest.mark.parametrize('precision', ['all', 'bf16,fp8'])
def test_cli_refuses_lists_outside_the_one_pass_modes(pr, tmp_path, monkeypatch, mode, precision):
    def loaded(*a, **kw):
        raise AssertionError('--precision was not checked first')
    monkeypatch.setattr(pr, 'load_run_config', loaded)
    with pytest.raises(SystemExit, match='ycbv_all or ycbineoat_all'):
        pr.main(['--mode', mode, '--train_data_path', 't', '--model_path', 'm', '--ckpt_dir', 'c', '--mean_std_path', 's',
                 '--outdir', str(tmp_path / 'o'), '--ycb_dir', 'y', '--YCBInEOAT_dir', 'd', '--seq_id', '48', '--precision', precision])


def test_cli_passes_single_modes_and_sweeps(pr, tmp_path, monkeypatch):
    calls = []
    monkeypatch.setattr(pr, 'load_run_config', lambda *a: ({}, None, None))
    monkeypatch.setattr(pr, 'predictSequenceYcbInEOAT', lambda *a, **kw: calls.append(('eoat', kw)) or [])
    monkeypatch.setattr(pr, 'predictSequenceYcb', lambda *a, **kw: calls.append(('ycbv', kw)) or ([], None))
    monkeypatch.setattr(pr, 'getResultsYcb', lambda *a, **kw: calls.append(('class', kw)) or {})
    monkeypatch.setattr(pr, 'getResultsYcbInEOAT', lambda *a, **kw: calls.append(('eoat_all', kw)) or {})
    base = ['--train_data_path', 't', '--model_path', 'm', '--ckpt_dir', 'c', '--mean_std_path', 's', '--outdir', str(tmp_path / 'o'),
            '--ycb_dir', 'y', '--YCBInEOAT_dir', 'd', '--seq_id', '48']
    for mode in ('ycbineoat', 'ycbv', 'class'):
        pr.main(base + ['--mode', mode, '--precision', 'fp16'])
        pr.main(base + ['--mode', mode])
    pr.main(base + ['--mode', 'ycbineoat_all', '--precision', 'fp8,bf16'])
    pr.main(base + ['--mode', 'ycbineoat_all', '--precision', 'all'])
    pr.main(base + ['--mode', 'ycbineoat_all'])
    kws = [kw.get('precision', '-') for _, kw in calls]
    assert [k for k, _ in calls] == ['eoat', 'eoat', 'ycbv', 'ycbv', 'class', 'class', 'eoat_all', 'eoat_all', 'eoat_all']
    assert kws == ['fp16', '-', 'fp16', '-', 'fp16', '-', ['fp8', 'bf16'], 'all', '-']      # the default passes nothing


def refusal_trees(tmp_path):
    """A YCB-Video and a YCBInEOAT layout whose files are placeholders, never loaded here -> (ycb, ycb templates, data, object
    templates)."""
    ycb = tmp_path / 'ycb'
    for k in range(1, 6):
        (ycb / 'CADmodels' / ('%03d_obj' % k)).mkdir(parents=True)
    (ycb / 'data_organized' / '0048' / 'pose_gt' / '2').mkdir(parents=True)
    data = tmp_path / 'data'
    for sub in ('rgb', 'depth_filled', 'annotated_poses'):
        (data / 'bleach0' / sub).mkdir(parents=True)
    np.savetxt(str(data / 'bleach0' / 'annotated_poses' / '0000000.txt'), np.eye(4))
    for name in ('rgb', 'depth_filled'):
        (data / 'bleach0' / name / '0000000.png').write_bytes(b'')
    for d in (tmp_path / 'cfg' / 'c2', tmp_path / 'cfg' / 'bleach'):
        (d / 'train').mkdir(parents=True)
        yaml.safe_dump({'resolution': 176, 'object_width': 200.0, 'boundingbox': 10, 'camera': dict(K_INFO)}, open(d / 'dataset_info.yml', 'w'))
        np.save(d / 'mean.npy', np.full(8, 40.0, np.float32)); np.save(d / 'std.npy', np.full(8, 5.0, np.float32))
        (d / 'ckpt.pth.tar').write_bytes(b'not a checkpoint')
        (d / 'mesh.ply').write_text('ply\n')
    tpl = lambda key: {'train_data_path': str(tmp_path / 'cfg' / key / 'train'), 'mean_std_path': str(tmp_path / 'cfg' / key),
                       'ckpt_dir': str(tmp_path / 'cfg' / key / 'ckpt.pth.tar'), 'model_path': str(tmp_path / 'cfg' / key / 'mesh.ply')}
    return str(ycb), tpl('c{class_id}'), str(data), tpl('{object}')


@pytest.mark.parametrize('precision', [['bf16', 'fp16'], ['fp16'], [], ['bf16', 'bf16'], ['bf16', 'fp4']])
def test_ycbv_sweep_refusals(pr, tmp_path, no_device, precision):
    ycb, ycb_tpl, _, _ = refusal_trees(tmp_path)
    with pytest.raises(ValueError, match='precision'):
        pr.getResultsYcbAll(ycb, [2], ycb_tpl, str(tmp_path / 'out'), precision=precision)
    assert not (tmp_path / 'out').exists()


@pytest.mark.parametrize('precision', [[], ['fp8', 'fp8'], ['bf16', 'fp4']])
def test_ycbineoat_sweep_refusals(pr, tmp_path, no_device, precision):
    _, _, data, obj_tpl = refusal_trees(tmp_path)
    with pytest.raises(ValueError, match='precision'):
        pr.getResultsYcbInEOAT(data, obj_tpl, str(tmp_path / 'out'), precision=precision)
    assert not (tmp_path / 'out').exists()


def test_video_with_two_modes_is_refused_with_nothing_written(pr, tmp_path, no_device):
    ycb, ycb_tpl, data, obj_tpl = refusal_trees(tmp_path)
    with pytest.raises(ValueError, match='video'):
        pr.getResultsYcbAll(ycb, [2], ycb_tpl, str(tmp_path / 'out'), precision=['bf16x3', 'fp8'], video=True)
    with pytest.raises(ValueError, match='video'):
        pr.getResultsYcbInEOAT(data, obj_tpl, str(tmp_path / 'out'), precision='all', video=True)
    assert not (tmp_path / 'out').exists()


def fake_loop(pr, monkeypatch):
    """The drivers without a device: no trackers, and a tracking loop whose poses depend on the mode and the sequence only."""
    monkeypatch.setattr(pr, '_one_pass_trackers', lambda entries, precision, max_batch: (None, {}))

    def loop(eng, trackers, sequences, variants, depth, workers, video, opts, seq_index):
        for k, (rgb_files, _, ids, init) in enumerate(sequences):
            yield {(m, i): np.stack([init + 0.001 * (t + 1) * (pr.PRECISIONS.index(m) + 1) + k for t in range(len(rgb_files))])
                   for m, i in variants}, None
    monkeypatch.setattr(pr, '_track_sequences', loop)


def tree_files(root):
    out = {}
    for d, _, fs in os.walk(root):
        for f in fs:
            with open(os.path.join(d, f), 'rb') as x:
                out[os.path.relpath(os.path.join(d, f), root)] = x.read()
    return out


def test_each_mode_writes_what_a_single_mode_run_writes_under_its_folder(pr, tmp_path, monkeypatch):
    fake_loop(pr, monkeypatch)
    data = tmp_path / 'data'
    for v, nf in (('bleach0', 3), ('sugar_box1', 2)):
        for sub in ('rgb', 'depth_filled', 'annotated_poses'):
            (data / v / sub).mkdir(parents=True)
        for i in range(nf):
            np.savetxt(str(data / v / 'annotated_poses' / ('%07d.txt' % i)), np.eye(4) * (i + 1))
            (data / v / 'rgb' / ('%07d.png' % i)).write_bytes(b'')
            (data / v / 'depth_filled' / ('%07d.png' % i)).write_bytes(b'')
    cfg = tmp_path / 'cfg'
    for o in ('bleach', 'sugar'):
        (cfg / o / 'train').mkdir(parents=True)
        yaml.safe_dump({'resolution': 176, 'object_width': 200.0, 'boundingbox': 10, 'camera': dict(K_INFO)}, open(cfg / o / 'dataset_info.yml', 'w'))
        np.save(cfg / o / 'mean.npy', np.zeros(8)); np.save(cfg / o / 'std.npy', np.ones(8))
        (cfg / o / 'ckpt.pth.tar').write_bytes(b'')
        (cfg / o / 'mesh.ply').write_text('ply\n')
    tpl = {'train_data_path': str(cfg / '{object}' / 'train'), 'mean_std_path': str(cfg / '{object}'),
           'ckpt_dir': str(cfg / '{object}' / 'ckpt.pth.tar'), 'model_path': str(cfg / '{object}' / 'mesh.ply')}
    sweep = pr.getResultsYcbInEOAT(str(data), tpl, str(tmp_path / 'sweep'), precision=['fp8', 'bf16x3'])
    assert list(sweep) == ['fp8', 'bf16x3'] and sorted(os.listdir(tmp_path / 'sweep')) == ['bf16x3', 'fp8']
    assert pr.precision_outdir(str(tmp_path / 'sweep'), 'fp8') == str(tmp_path / 'sweep' / 'fp8')
    for m in ('fp8', 'bf16x3'):
        one = pr.getResultsYcbInEOAT(str(data), tpl, str(tmp_path / 'single' / m), precision=m)
        assert sorted(one) == sorted(sweep[m]) == ['bleach0', 'sugar_box1']
        for v in one:
            assert np.array_equal(one[v], sweep[m][v])
        files = tree_files(str(tmp_path / 'sweep' / m))
        assert files == tree_files(str(tmp_path / 'single' / m)) and len(files) == 5
    assert not np.array_equal(sweep['fp8']['bleach0'], sweep['bf16x3']['bleach0'])
