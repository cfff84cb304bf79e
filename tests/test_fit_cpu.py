"""The fit check without a GPU: oracle/fit_ref.py on hand-made arrays, fit_fractions and roc_auc, step_options' fit and --fit
parsing and refusals, and the FIT_FILE layout the drivers write (tracking faked)."""
import importlib
import os
import pickle
import sys
import numpy as np
import pytest
import torch

PKG = 'iros20-6d-pose-tracking_b200'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import fit_ref  # noqa: E402


@pytest.fixture(scope='module')
def pr():
    return importlib.import_module(PKG + '.predict')


def test_oracle_columns_and_tau_edges():
    tau = 10
    R = np.array([[0, 500, 500, 500, 500, 500, 500, 500]], np.uint16)
    O = np.array([[700, 0, 490, 510, 489, 511, 505, 60000]], np.uint16)
    rows = fit_ref.fit_rows(R, O, tau)
    # model 7; observed 6 (the O = 0 pixel is out); inliers at exactly -tau, +tau and +5; front 489; behind 511 and 60000
    assert rows.dtype == np.int32 and rows.tolist() == [7, 6, 3, 1, 2, 10 + 10 + 5]
    assert rows[1] == rows[2] + rows[3] + rows[4]


def test_oracle_empty_model_and_zero_observed():
    R = np.zeros((2, 176, 176), np.uint16)
    O = np.full((2, 176, 176), 800, np.uint16)
    assert fit_ref.fit_rows(R, O, 5).tolist() == [[0] * 6] * 2
    R[1, 10:20, 10:30] = 900
    rows = fit_ref.fit_rows(R, np.zeros_like(O), 5)
    assert rows.tolist() == [[0] * 6, [200, 0, 0, 0, 0, 0]]
    rows = fit_ref.fit_rows(R, O, 5)
    assert rows[1].tolist() == [200, 200, 0, 200, 0, 0]
    with pytest.raises(ValueError):
        fit_ref.fit_rows(R, O[:1], 5)


def test_fit_fractions_and_roc_auc(pr):
    rows = np.array([[100, 90, 80, 5, 5, 160], [0, 0, 0, 0, 0, 0], [-1] * 6], np.int32)
    f = pr.fit_fractions(rows)
    assert np.allclose(f['inlier'][:2], [0.8, 0]) and np.allclose(f['front'][:2], [0.05, 0]) and np.allclose(f['residual'][:2], [2, 0])
    assert all(np.isnan(v[2]) for v in f.values())
    assert np.allclose(pr.fit_fractions(torch.from_numpy(rows[:1]))['behind'], [0.05])
    assert pr.roc_auc([0.1, 0.9, 0.5, 0.5], [False, True, True, False]) == 0.875
    assert pr.roc_auc([1, 2, 3], [True, True, False]) == 0.0
    assert np.isnan(pr.roc_auc([1, 2], [True, True]))


def test_fit_argument(pr):
    for bad in (0, 1001, -1, 2.5, True, '10'):
        with pytest.raises(ValueError, match='fit'):
            pr.step_options(fit=bad)
    assert pr.step_options().fit is None and pr.step_options(fit=1000).fit == 1000 and pr.step_options(fit=np.int64(7)).fit == 7
    # rows are kept for a given fit only; the check runs at it, or at FIT_TAU_DEFAULT when hypotheses rank the starts
    assert pr.step_options(fit=7).tau == 7 and pr.step_options().tau is None
    hyp = pr.step_options(hypotheses=4)
    assert hyp.fit is None and hyp.tau == pr.FIT_TAU_DEFAULT and pr.step_options(fit=7, hypotheses=4).tau == 7
    # the Tracker's switch: True is FIT_TAU_DEFAULT, False is off and refuses hypotheses
    on = pr.step_options(fit=True, fit_switch=True)
    assert on.fit == on.tau == pr.FIT_TAU_DEFAULT and pr.step_options(fit=False, fit_switch=True).tau is None
    with pytest.raises(ValueError, match='fit must not be off'):
        pr.step_options(fit=False, hypotheses=4, fit_switch=True)
    with pytest.raises(ValueError, match='fit'):
        pr.step_options(fit=np.bool_(True), fit_switch=True)
    assert pickle.loads(pickle.dumps(hyp)) == hyp                   # the ranks of a multi-GPU run receive it pickled


@pytest.mark.parametrize('mode', ['ycbv', 'ycbineoat', 'ycbv_recover'])
def test_cli_refuses_fit_outside_the_one_pass_drivers(pr, mode):
    args = ['--mode', mode, '--train_data_path', 'x', '--model_path', 'x', '--ckpt_dir', 'x', '--mean_std_path', 'x',
            '--outdir', 'x', '--fit', '10']
    with pytest.raises(SystemExit, match='--fit needs --mode ycbv_all or ycbineoat_all'):
        pr.main(args)


@pytest.mark.parametrize('tau', ['0', '1001'])
def test_cli_refuses_tau_out_of_range(pr, tau):
    args = ['--mode', 'ycbineoat_all', '--train_data_path', 'x', '--model_path', 'x', '--ckpt_dir', 'x', '--mean_std_path', 'x',
            '--outdir', 'x', '--YCBInEOAT_dir', 'x', '--fit', tau]
    with pytest.raises(SystemExit, match='--fit %s' % tau):
        pr.main(args)


def test_cli_passes_fit_to_the_driver(pr, monkeypatch, tmp_path):
    got = {}

    def fake(ycbineoat_dir, config, outdir, **kw):
        got.update(kw)
        return {}
    monkeypatch.setattr(pr, 'getResultsYcbInEOAT', fake)
    base = ['--mode', 'ycbineoat_all', '--train_data_path', 'x', '--model_path', 'x', '--ckpt_dir', 'x', '--mean_std_path', 'x',
            '--outdir', str(tmp_path), '--YCBInEOAT_dir', 'x']
    pr.main(base + ['--fit', '25'])
    assert got['fit'] == 25
    got.clear()
    pr.main(base)
    assert 'fit' not in got


def test_fit_file_layout(pr, tmp_path):
    """The writers with the fit on: pose files byte for byte those without it, and FIT_FILE inside each sequence folder."""
    init = np.tile(np.eye(4), (2, 1, 1)); init[:, 2, 3] = 0.5
    poses = {('bf16x3', 1): np.stack([init * (1 + 0.01 * t) for t in range(3)])}
    rows = {('bf16x3', 1): np.arange(3 * 2 * 6, dtype=np.int32).reshape(3, 2, 6)}
    dirs = lambda root: {('bf16x3', 1): {2: str(tmp_path / root / 'c2'), 5: str(tmp_path / root / 'c5')}}
    a = pr._write_ycb_all_sequence(dirs('plain'), 48, (2, 5), init, (poses, None))
    b = pr._write_ycb_all_sequence(dirs('fit'), 48, (2, 5), init, (poses, rows))
    assert all(np.array_equal(a[k], b[k]) for k in a)
    for j, c in enumerate((2, 5)):
        sdir = tmp_path / 'fit' / ('c%d' % c) / 'seq48'
        txt = sorted(f for f in os.listdir(sdir) if f.endswith('.txt'))
        assert txt == sorted(os.listdir(tmp_path / 'plain' / ('c%d' % c) / 'seq48'))
        assert all((sdir / f).read_bytes() == (tmp_path / 'plain' / ('c%d' % c) / 'seq48' / f).read_bytes() for f in txt)
        f = np.load(str(sdir / pr.FIT_FILE))
        assert f.dtype == np.int32 and f.shape == (4, 6) and (f[0] == -1).all() and np.array_equal(f[1:], rows[('bf16x3', 1)][:, j])
    roots = {('bf16x3', 1): str(tmp_path / 'eoat')}
    one = {('bf16x3', 1): poses[('bf16x3', 1)][:, :1]}
    out = pr._write_ycbineoat_video(roots, 'bleach0', (one, {k: v[:, :1] for k, v in rows.items()}))
    assert np.array_equal(out[('bf16x3', 1)], one[('bf16x3', 1)][:, 0])
    plain = pr._write_ycbineoat_video({('bf16x3', 1): str(tmp_path / 'eoat_plain')}, 'bleach0', (one, None))
    assert np.array_equal(plain[('bf16x3', 1)], out[('bf16x3', 1)])
    assert sorted(os.listdir(tmp_path / 'eoat_plain' / 'bleach0')) == sorted(x for x in os.listdir(tmp_path / 'eoat' / 'bleach0')
                                                                           if x.endswith('.txt'))
    assert sorted(os.listdir(tmp_path / 'eoat')) == ['bleach0']                 # nothing at the tree's root
    f = np.load(str(tmp_path / 'eoat' / 'bleach0' / pr.FIT_FILE))
    assert np.array_equal(f, rows[('bf16x3', 1)][:, 0]) and len([x for x in os.listdir(tmp_path / 'eoat' / 'bleach0') if x.endswith('.txt')]) == 3
    assert not pr.FIT_FILE.endswith('.txt')


def test_drivers_pass_fit_through_the_sequence_loop(pr, tmp_path, monkeypatch):
    """_one_pass_back hands the run's options to _track_sequences: with fit, a value whose fit is the given one, and writes[k]
    gets the rows; without it, fit and the check off, and writes[k] gets None for rows."""
    calls = []
    monkeypatch.setattr(pr, '_one_pass_trackers', lambda entries, precision, max_batch, device=None: (None, {}))
    monkeypatch.setattr(pr, '_calibrate_borrowed', lambda *a: None)

    def loop(eng, trackers, sequences, variants, depth, workers, video, opts, seq_index):
        calls.append(opts)
        for rgb_files, _, ids, init in sequences:
            poses = {v: np.stack([init] * len(rgb_files)) for v in variants}
            yield poses, ({v: np.zeros((len(rgb_files), len(ids), 6), np.int32) for v in variants} if opts.fit else None)
    monkeypatch.setattr(pr, '_track_sequences', loop)
    run = lambda **step: pr._OnePass(1, 'bf16x3', [('bf16x3', 1, str(tmp_path))], False, False, [{}], pr.step_options(**step))
    seqs = [(['a', 'b'], ['a', 'b'], (0,), np.eye(4)[None])]
    got = []
    pr._one_pass_back(run(fit=7), [], 1, seqs, 1, 1, None, [(lambda t: got.append(t) or {},)], lambda w, k: w)
    assert calls[-1] == pr.step_options(fit=7) and calls[-1].fit == calls[-1].tau == 7
    assert isinstance(got[-1], tuple) and got[-1][1] is not None
    pr._one_pass_back(run(), [], 1, seqs, 1, 1, None, [(lambda t: got.append(t) or {},)], lambda w, k: w)
    assert calls[-1] == pr.step_options() and calls[-1].fit is None and calls[-1].tau is None
    assert isinstance(got[-1][0], dict) and got[-1][1] is None
