"""CPU side of `predict --mode ycbv_recover`: CLI parsing and every refusal made before a device is touched, the producer-mesh id
range, the tables from a hand-made result, and the numpy restatement of the pose errors on poses with known angles and offsets."""
import importlib

import numpy as np
import pytest
import yaml

P = importlib.import_module('iros20-6d-pose-tracking_b200.predict')


def _args(*extra):
    return ['--mode', 'ycbv_recover', '--ycb_dir', 'ycb', '--class_ids', '1,2', '--train_data_path', 't/{class_id}',
            '--model_path', 'm/{class_id}.ply', '--ckpt_dir', 'c/{class_id}', '--mean_std_path', 's/{class_id}'] + list(extra)


@pytest.mark.parametrize('extra, text', [
    (['--iterations', '0'], '--iterations'), (['--iterations', '9'], '--iterations'), (['--iterations', '1,2'], '--iterations'),
    (['--precision', 'fp16'], 'fp16'), (['--precision', 'bf16,fp16'], 'fp16'), (['--precision', 'bf16,bf16'], 'more than once'),
    (['--gpus', '2'], 'one GPU'), (['--class_ids', '1,x'], '--class_ids')])
def test_cli_refusals(extra, text):
    with pytest.raises(SystemExit) as e:
        P.main(_args(*extra))
    assert text in str(e.value)


def test_cli_arguments():
    import argparse
    ns = argparse.Namespace(mode='ycbv_recover', ycb_dir='ycb', class_ids='3,1', gpus=None, precision='bf16x3,fp8', iterations='4',
                            train_data_path='t', model_path='m/{class_id}.ply', ckpt_dir='a,b', mean_std_path='s',
                            pair_model_path=None, num_sample=7, seed=3, max_frames=2)
    ids, config, kw = P.cli_recover(ns)
    assert ids == [1, 3] and config['ckpt_dir'] == ['a', 'b'] and 'pair_model_path' not in config
    assert kw == dict(num_sample=7, seed=3, precision=['bf16x3', 'fp8'], iterations=4, max_frames=2)
    assert P.pair_model_template(config) == 'm/{class_id}.obj'
    assert P.pair_model_template(dict(config, pair_model_path='x.obj')) == 'x.obj'


def test_front_refusals():
    assert P.recover_front('all', 8) == (P.YCB_ALL_PRECISIONS, 8)
    for bad in (dict(precision='fp16'), dict(iterations=0), dict(iterations=9), dict(iterations=[1, 2]), dict(gpus=2),
                dict(precision=['tf32', 'nope'])):
        with pytest.raises(ValueError):
            P.recover_front(**bad)


def test_pair_mesh_ids_stay_apart():
    assert P.pair_mesh_base([1, 21], 1) == 32 and P.pair_mesh_base([1, 21], 3) == 96
    with pytest.raises(ValueError, match='also weight ids'):
        P.pair_mesh_base([1, 33], 1)                       # producer mesh 33 would replace class 33's tracking mesh
    with pytest.raises(SystemExit, match='weight ids'):
        P.cli_recover(__import__('argparse').Namespace(
            mode='ycbv_recover', ycb_dir='ycb', class_ids='2,34', gpus=None, precision=None, iterations=None, train_data_path='t',
            model_path='m', ckpt_dir='c', mean_std_path='s', pair_model_path=None, num_sample=10, seed=0, max_frames=None))


def test_mismatched_normalisers_refused_before_loading(tmp_path):
    ycb = tmp_path / 'ycb'
    for k in range(1, 4):
        (ycb / 'CADmodels' / ('%03d_obj' % k)).mkdir(parents=True)
    for c in (1, 2):
        d = tmp_path / ('c%d' % c)
        (d / 'train').mkdir(parents=True)
        yaml.safe_dump({'resolution': 176, 'object_width': 200.0, 'camera': {'focalX': 1.0, 'focalY': 1.0, 'centerX': 1.0,
                                                                            'centerY': 1.0, 'height': 4, 'width': 4}},
                       open(d / 'dataset_info.yml', 'w'))
        for f in ('ckpt', 'mesh.ply'):
            (d / f).write_text('x')
        np.save(str(d / 'mean.npy'), np.zeros(8)); np.save(str(d / 'std.npy'), np.ones(8))
    cfg = {'train_data_path': str(tmp_path / 'c{class_id}' / 'train'), 'model_path': str(tmp_path / 'c{class_id}' / 'mesh.ply'),
           'ckpt_dir': str(tmp_path / 'c{class_id}' / 'ckpt'), 'mean_std_path': str(tmp_path / 'c{class_id}'),
           'trans_normalizer': {1: 0.03, 2: 0.04}}
    with pytest.raises(ValueError, match='trans_normalizer'):
        P.recoverYcbKeyframes(str(ycb), [1, 2], cfg)


def _rot(axis, deg):
    a = np.radians(deg)
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    Kx = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(a) * Kx + (1 - np.cos(a)) * Kx @ Kx


def test_numpy_pose_errors_known_values():
    rng = np.random.default_rng(1)
    gt, pred = [], []
    cases = [((0, 0, 1), 0.0, (0, 0, 0)), ((1, 2, 3), 30.0, (0.003, -0.004, 0)), ((0, 1, 0), 90.0, (0, 0, 0.01)),
             ((1, 0, 1), 179.0, (0.001, 0, 0)), ((0, 0, 1), 180.0, (0, 0, 0))]
    for axis, deg, off in cases:
        g = np.eye(4); g[:3, :3] = _rot(rng.standard_normal(3), rng.uniform(0, 180)); g[:3, 3] = rng.standard_normal(3)
        p = g.copy(); p[:3, :3] = g[:3, :3] @ _rot(axis, deg); p[:3, 3] = g[:3, 3] + off
        gt.append(g); pred.append(p)
    e = P.pose_errors_np(np.array(pred), np.array(gt))
    assert np.allclose(e[:, 0], [0, 5, 10, 1, 0], atol=1e-9)
    assert np.allclose(e[:, 1], [0, 30, 90, 179, 180], atol=1e-5)


def test_tables_from_a_hand_made_result(capsys):
    s = lambda n, a: dict(rows=n, add_auc=a, adds_auc=a + 0.1, rot_mean=2.0, rot_median=1.5, trans_mean=3.0, trans_median=2.5)
    empty = dict(rows=0, add_auc=None, adds_auc=None, rot_mean=None, rot_median=None, trans_mean=None, trans_median=None)
    res = {('bf16x3', 2, 0): {1: dict(rows=4, summary=[s(4, 0.5), s(4, 0.6), s(4, 0.7)]), 2: dict(rows=0, summary=[empty] * 3),
                              'all': dict(rows=4, summary=[s(4, 0.5), s(4, 0.6), s(4, 0.7)])},
           ('fp8', 2, 1): {1: dict(rows=4, summary=[s(4, 0.5), s(4, 0.65), s(4, 0.75)]), 2: dict(rows=0, summary=[empty] * 3),
                           'all': dict(rows=4, summary=[s(4, 0.5), s(4, 0.65), s(4, 0.75)])}}
    P.print_recover_tables(res, {1: '001_obj', 2: '002_obj'})
    out = capsys.readouterr().out.splitlines()
    assert out[0].startswith('class 1 (001_obj): 4 rows') and out[1].split()[:4] == ['ckpt', 'mode', 'round', 'rows']
    assert out[2].split() == ['-', 'start', '0', '4', '50.000', '60.000', '2', '1.5', '3', '2.5']
    assert [l.split()[:3] for l in out[3:7]] == [['0', 'bf16x3', '1'], ['0', 'bf16x3', '2'], ['1', 'fp8', '1'], ['1', 'fp8', '2']]
    assert out[7].startswith('class 2 (002_obj): 0 rows') and out[9].split() == ['-', 'start', '0', '0']
    assert out[14].startswith('all classes: 4 rows') and len(out) == 21
