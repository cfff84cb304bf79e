"""CPU: the checkpoint dimension of validation and of the one-pass drivers without a device -- argument lists and their
refusals (all before anything loads), the output trees of each variant, the return value's nesting and the selection rule."""
import importlib
import os

import numpy as np
import pytest
import torch

PKG = 'iros20-6d-pose-tracking_b200'


@pytest.fixture(scope='module')
def pr():
    return importlib.import_module(PKG + '.predict')


@pytest.fixture(scope='module')
def P():
    return importlib.import_module(PKG + '.problems')


@pytest.fixture
def no_load(monkeypatch, pr):
    """Loading a checkpoint or making an Engine fails the test: every refusal must come first."""
    def fail(*a, **kw):
        raise AssertionError('loaded before the refusal')
    monkeypatch.setattr(torch, 'load', fail)
    monkeypatch.setattr(pr, 'Engine', fail)
    monkeypatch.setattr(pr, '_one_pass_trackers', fail)


def test_checkpoint_list(pr):
    assert pr.checkpoint_list('a', 's') == [('a', 's')]
    assert pr.checkpoint_list(['a', 'b'], 's') == [('a', 's'), ('b', 's')]
    assert pr.checkpoint_list(['a', 'b'], ['s', 't']) == [('a', 's'), ('b', 't')]
    with pytest.raises(ValueError, match='2 entries for 3 checkpoints'):
        pr.checkpoint_list(['a', 'b', 'c'], ['s', 't'])
    with pytest.raises(ValueError, match='listed more than once'):
        pr.checkpoint_list(['a', 'b', 'a'], 's')
    with pytest.raises(ValueError, match='empty'):
        pr.checkpoint_list(['a', ''], 's')
    cfg = {'ckpt_dir': 'c', 'mean_std_path': 'm', 'model_path': 'x', 'train_data_path': 't'}
    assert pr.checkpoint_configs(cfg) == [cfg]
    two = pr.checkpoint_configs(dict(cfg, ckpt_dir=['c', 'd']))
    assert [(k['ckpt_dir'], k['mean_std_path'], k['model_path']) for k in two] == [('c', 'm', 'x'), ('d', 'm', 'x')]


def test_ids_out_of_range(pr):
    pr._check_checkpoint_ids([1, 21, 31], 2, 'class')
    pr._check_checkpoint_ids([40], 1, 'class')                       # one checkpoint: ids as today
    with pytest.raises(ValueError, match='class 32: with 2 checkpoints'):
        pr._check_checkpoint_ids([5, 32], 2, 'class')


def test_weight_sets_over_budget(monkeypatch):
    E = importlib.import_module(PKG + '.engine')
    L = importlib.import_module(PKG + '._lib')
    each = L.load().se3tn_weight_set_bytes()
    # the blob in fp32, conv weights in tf32, bf16x3, bf16, fp16 and fp8: 17 bytes per blob float, plus the small tables
    assert 17 * L.WEIGHT_BLOB_FLOATS < each < 17 * L.WEIGHT_BLOB_FLOATS + 8_000_000
    monkeypatch.setattr(torch.cuda, 'mem_get_info', lambda dev=None: (3 * each, 80 * 10 ** 9))
    assert E.check_weight_sets_fit(3, 0) == each
    with pytest.raises(ValueError, match=r'4 weight sets need .* GB .* cuda:0 has'):
        E.check_weight_sets_fit(4, 0)


def test_val_dir_refusals_before_any_load(P, tmp_path, monkeypatch, no_load, capsys):
    base = ['--val_dir', str(tmp_path), '--dataset_info', str(tmp_path / 'info.yml')]
    with pytest.raises(SystemExit):
        P.main(base + ['--ckpt', 'a,b,c', '--mean_std_path', 's,t'])
    assert '2 entries for 3 checkpoints' in capsys.readouterr().err
    with pytest.raises(SystemExit):
        P.main(base + ['--ckpt', 'a,b,a', '--mean_std_path', 's'])
    assert 'listed more than once' in capsys.readouterr().err
    L = importlib.import_module(PKG + '._lib')
    monkeypatch.setattr(torch.cuda, 'current_device', lambda: 0)
    monkeypatch.setattr(torch.cuda, 'mem_get_info', lambda dev=None: (L.load().se3tn_weight_set_bytes(), 80 * 10 ** 9))
    with pytest.raises(ValueError, match='2 checkpoints need'):
        P.main(base + ['--ckpt', 'a,b', '--mean_std_path', 's'])


def test_ycb_dir_refusal_before_any_load(P, tmp_path, no_load, capsys):
    (tmp_path / 'CADmodels' / '001_a').mkdir(parents=True)
    with pytest.raises(SystemExit):
        P.main(['--ycb_dir', str(tmp_path), '--class_ids', '1', '--ckpt_dir', 'a,b', '--mean_std_path', 's,t,u',
                '--train_data_path', 't', '--model_path', 'm'])
    assert '3 entries for 2 checkpoints' in capsys.readouterr().err


def test_driver_refusals_before_any_load(pr, tmp_path, no_load):
    cfg = {'train_data_path': 't', 'mean_std_path': 's', 'ckpt_dir': ['a', 'b'], 'model_path': 'm'}
    with pytest.raises(ValueError, match='one checkpoint, not of 2'):
        pr.getResultsYcbInEOAT(str(tmp_path), cfg, str(tmp_path / 'o'), video=True)
    with pytest.raises(ValueError, match='one checkpoint, not of 2'):
        pr.getResultsYcbAll(str(tmp_path), [1], cfg, str(tmp_path / 'o'), video=True)
    with pytest.raises(ValueError, match='listed more than once'):
        pr.getResultsYcbInEOAT(str(tmp_path), dict(cfg, ckpt_dir=['a', 'a']), str(tmp_path / 'o'))
    with pytest.raises(ValueError, match='2 entries for 3 checkpoints'):
        pr.getResultsYcbAll(str(tmp_path), [1], dict(cfg, ckpt_dir=['a', 'b', 'c'], mean_std_path=['s', 't']), str(tmp_path / 'o'))
    for k in range(1, 34):
        (tmp_path / 'CADmodels' / ('%03d_obj' % k)).mkdir(parents=True)
    with pytest.raises(ValueError, match='class 33: with 2 checkpoints'):
        pr.getResultsYcbAll(str(tmp_path), [3, 33], cfg, str(tmp_path / 'o'))
    with pytest.raises(SystemExit):
        pr.main(['--mode', 'ycbineoat_all', '--YCBInEOAT_dir', str(tmp_path), '--train_data_path', 't', '--model_path', 'm',
                 '--ckpt_dir', 'a,b', '--mean_std_path', 's,t,u', '--outdir', str(tmp_path / 'o')])


def test_variant_trees(pr):
    out = '/o'
    one = pr._sweep_variants(out, ('bf16x3',), False, (1,), False)
    assert one == [('bf16x3', 1, out)] and one == pr._sweep_variants(out, ('bf16x3',), False, (1,), False, 1)
    assert pr._sweep_variants(out, ('fp8', 'fp32'), True, (1, 2), True, 1) == pr._sweep_variants(out, ('fp8', 'fp32'), True, (1, 2), True)
    two = pr._sweep_variants(out, ('bf16x3',), False, (1,), False, 2)
    assert two == [('bf16x3', 1, 0, os.path.join(out, 'ckpt0')), ('bf16x3', 1, 1, os.path.join(out, 'ckpt1'))]
    full = pr._sweep_variants(out, ('bf16x3', 'fp8'), True, (1, 2), True, 2)
    assert [v[-1] for v in full] == [os.path.join(out, 'ckpt%d' % c, 'iter%d' % k, m) for c in (0, 1) for k in (1, 2) for m in ('bf16x3', 'fp8')]
    res = pr._sweep_results({v[:-1]: '%s%d%d' % v[:3] for v in full}, full, True, True)
    assert res == {c: {k: {m: '%s%d%d' % (m, k, c) for m in ('bf16x3', 'fp8')} for k in (1, 2)} for c in (0, 1)}
    assert pr._sweep_results({v[:-1]: v[2] for v in two}, two, False, False) == {0: 0, 1: 1}
    assert pr._sweep_results({('bf16x3', 1): 'r'}, one, False, False) == 'r'
    assert pr._checkpoints([v[:-1] for v in full]) == [0, 1] and pr._checkpoints([('fp8', 1)]) == [0]
    seqs = [('r', 'd', (2, 5), 'i')]
    assert pr._checkpoint_sequences(seqs, 0) is seqs and pr._checkpoint_sequences(seqs, 1) == [('r', 'd', (34, 37), 'i')]
    assert pr._rank_weight_ids(seqs, [0], [v[:-1] for v in two]) == {2, 5, 34, 37}


def test_selection_tie_rule(P, pr, capsys):
    assert P.best_checkpoint([0.3, 0.2, 0.2, 0.25]) == 1             # the first of equal lowest losses
    assert P.best_checkpoint([0.2]) == 0
    rows = {'ckpt0/fp8': {'adds': 80.0}, 'ckpt1/fp8': {'adds': 90.0}, 'ckpt2/fp8': {'adds': 90.0},
            'ckpt0/fp32': {'adds': 70.0}, 'ckpt1/fp32': {'adds': 60.0}, 'ckpt2/fp32': {'adds': 70.0}}
    assert pr.best_checkpoints(rows) == {'fp8': (1, 90.0), 'fp32': (0, 70.0)}
    assert pr.best_checkpoints({'ckpt0': {'adds': 1.0}, 'ckpt1': {'adds': 2.0}}) == {'': (1, 2.0)}
    pr.print_best_checkpoints(rows, ['a', 'b', 'c'])
    out = capsys.readouterr().out
    assert 'best fp8: checkpoint 1 (b), ADD-S 90.0000' in out and 'best fp32: checkpoint 0 (a), ADD-S 70.0000' in out
    r = lambda t: {'trans': t, 'rot': 0.0, 'predictions': np.zeros((1, 6), np.float32)}
    P._print_checkpoints(['a', 'b'], ['fp32'], {(0, 'fp32'): r(0.5), (1, 'fp32'): r(0.5)}, {'trans': 1, 'rot': 1})
    assert 'best fp32: checkpoint 0 (a)' in capsys.readouterr().out
