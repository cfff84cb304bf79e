"""ICP in the drivers without a GPU: step_options' icp parsing and refusals, the CLI's --icp / --icp_tau (modes that refuse them,
ranges, hypotheses), and that the one-pass loop and the CLI pass icp through unchanged, and not at all without it."""
import importlib
import numpy as np
import pytest

PKG = 'iros20-6d-pose-tracking_b200'
BASE = ['--train_data_path', 'x', '--model_path', 'x', '--ckpt_dir', 'x', '--mean_std_path', 'x', '--outdir', 'x']


@pytest.fixture(scope='module')
def pr():
    return importlib.import_module(PKG + '.predict')


def test_driver_icp(pr):
    assert pr.step_options(icp=0).icp is None and pr.step_options(icp=None).icp is None
    assert pr.step_options(icp=3).icp == 3 and pr.step_options(icp=2, icp_tau=5).icp == {'iterations': 2, 'tau_mm': 5}
    assert pr.step_options(icp={'iterations': 2, 'min_inliers': 50}).icp == {'iterations': 2, 'min_inliers': 50}
    for icp, tau, S in ((17, None, 1), (-1, None, 1), (3, 0, 1), (3, 1001, 1), (0, 5, 1), (3, None, 2), (2, 5, 4)):
        with pytest.raises(ValueError, match='icp'):
            pr.step_options(hypotheses=S, icp=icp, icp_tau=tau)
    with pytest.raises(ValueError, match='ICP inside hypothesis steps is not supported'):
        pr.step_options(hypotheses=4, icp=2)
    assert pr.step_options(hypotheses=4, icp=0).icp is None


@pytest.mark.parametrize('mode', ['ycbv', 'ycbineoat'])
def test_cli_refuses_icp_outside_the_one_pass_drivers(pr, mode):
    for extra in (['--icp', '2'], ['--icp_tau', '10']):
        with pytest.raises(SystemExit, match='--icp / --icp_tau need --mode ycbv_all, ycbineoat_all or ycbv_recover'):
            pr.main(['--mode', mode] + BASE + extra)


@pytest.mark.parametrize('extra', [['--icp', '17'], ['--icp', '-1'], ['--icp', '2', '--icp_tau', '0'], ['--icp_tau', '10'],
                                   ['--icp', '2', '--hypotheses', '4']])
def test_cli_refuses_bad_icp(pr, extra):
    with pytest.raises(SystemExit, match='--icp'):
        pr.main(['--mode', 'ycbineoat_all', '--YCBInEOAT_dir', 'x'] + BASE + extra)


def test_cli_passes_icp_to_the_drivers(pr, monkeypatch, tmp_path):
    got = {}

    def fake(ycbineoat_dir, config, outdir, **kw):
        got.clear(); got.update(kw)
        return {}
    monkeypatch.setattr(pr, 'getResultsYcbInEOAT', fake)
    base = ['--mode', 'ycbineoat_all', '--YCBInEOAT_dir', 'x'] + BASE[:-1] + [str(tmp_path)]
    pr.main(base + ['--icp', '3', '--icp_tau', '12'])
    assert got['icp'] == 3 and got['icp_tau'] == 12
    pr.main(base + ['--icp', '0'])
    assert got['icp'] == 0 and 'icp_tau' not in got
    pr.main(base)
    assert 'icp' not in got and 'icp_tau' not in got


def test_cli_passes_icp_to_recover(pr):
    import argparse
    ns = argparse.Namespace(mode='ycbv_recover', ycb_dir='ycb', class_ids='3,1', gpus=None, precision=None, iterations='2',
                            train_data_path='t', model_path='m/{class_id}.ply', ckpt_dir='c', mean_std_path='s', pair_model_path=None,
                            num_sample=7, seed=3, max_frames=None, icp=4, icp_tau=None)
    assert pr.cli_recover(ns)[2] == dict(num_sample=7, seed=3, precision='bf16x3', iterations=2, max_frames=None, icp=4)
    ns.icp, ns.icp_tau = None, None
    assert 'icp' not in pr.cli_recover(ns)[2]


def test_one_pass_loop_gets_icp(pr, monkeypatch, tmp_path):
    calls = []
    monkeypatch.setattr(pr, '_one_pass_trackers', lambda entries, precision, max_batch, device=None: (None, {}))
    monkeypatch.setattr(pr, '_calibrate_borrowed', lambda *a: None)

    def loop(eng, trackers, sequences, variants, depth, workers, video, opts, seq_index):
        calls.append(opts)
        for rgb_files, _, ids, init in sequences:
            yield {v: np.stack([init] * len(rgb_files)) for v in variants}, None
    monkeypatch.setattr(pr, '_track_sequences', loop)
    run = lambda **step: pr._OnePass(1, 'bf16x3', [('bf16x3', 1, str(tmp_path))], False, False, [{}], pr.step_options(**step))
    seqs = [(['a', 'b'], ['a', 'b'], (0,), np.eye(4)[None])]
    got = []
    pr._one_pass_back(run(icp=2, icp_tau=30), [], 1, seqs, 1, 1, None, [(lambda t: got.append(t) or {},)], lambda w, k: w)
    assert calls[-1] == pr.step_options(icp=2, icp_tau=30) and calls[-1].icp == {'iterations': 2, 'tau_mm': 30}
    assert calls[-1].fit is None and got[-1][1] is None
    pr._one_pass_back(run(icp=None), [], 1, seqs, 1, 1, None, [(lambda t: got.append(t) or {},)], lambda w, k: w)
    assert calls[-1] == pr.step_options() and calls[-1].icp is None and got[-1][1] is None


def test_recover_table_labels_icp_rows(pr, capsys):
    s = dict(rows=2, add_auc=0.5, adds_auc=0.6, rot_mean=1.0, rot_median=1.0, trans_mean=2.0, trans_median=2.0)
    res = {('bf16x3', 2): {'all': dict(rows=2, summary=[s] * 5, icp=2)}}
    pr.print_recover_tables(res, {})
    out = capsys.readouterr().out.splitlines()
    assert [l.split()[2] for l in out[2:]] == ['0', '1', '2', 'icp', 'icp']
    assert out[-2].split()[2:4] == ['icp', '1'] and out[-1].split()[2:4] == ['icp', '2']
