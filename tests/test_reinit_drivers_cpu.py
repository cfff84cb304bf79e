"""The re-initialisation options of the one-pass drivers without a GPU: --reinit_below needs --mode ycbv_all, --reinit_after
needs --reinit_below, values are checked before anything is read, the --init_* options set its restarts, and step_options
carries it as a trailing StepOptions field that turns the fit check on."""
import importlib
import pickle
import pytest

PKG = 'iros20-6d-pose-tracking_b200'
BASE = ['--train_data_path', 'nowhere/train', '--model_path', 'nowhere/m.ply']
CKPT = ['--ckpt_dir', 'nowhere/c.pth', '--mean_std_path', 'nowhere']


@pytest.fixture(scope='module')
def pr():
    return importlib.import_module(PKG + '.predict')


@pytest.mark.parametrize('mode', ['ycbv', 'ycbineoat', 'ycbineoat_all', 'ycbv_recover', 'ycbv_init', 'other'])
def test_reinit_needs_ycbv_all(pr, mode):
    with pytest.raises(SystemExit, match='--reinit_below needs --mode ycbv_all'):
        pr.main(['--mode', mode, '--reinit_below', '0.5'] + BASE + CKPT)


def test_reinit_after_needs_reinit_below(pr):
    with pytest.raises(SystemExit, match='--reinit_after needs --reinit_below'):
        pr.main(['--mode', 'ycbv_all', '--reinit_after', '2'] + BASE + CKPT)


@pytest.mark.parametrize('extra', [['--reinit_below', '0'], ['--reinit_below', '1.5'], ['--reinit_below', '0.1234'],
                                   ['--reinit_below', '0.5', '--reinit_after', '0'], ['--reinit_below', '0.5', '--reinit_after', '1001']])
def test_reinit_values_are_checked_first(pr, extra):
    with pytest.raises(SystemExit, match='--reinit_below / --reinit_after'):
        pr.main(['--mode', 'ycbv_all'] + extra + BASE + CKPT)


def test_init_options_go_with_reinit(pr, monkeypatch):
    seen = {}

    def fake(ycb_dir, class_ids, config, outdir, **kw):
        seen.update(kw)
        raise SystemExit('stop')
    monkeypatch.setattr(pr, 'getResultsYcbAll', fake)
    monkeypatch.setattr(pr, 'ycb_class_names', lambda d: ['c%d' % i for i in range(21)])
    with pytest.raises(SystemExit, match='stop'):
        pr.main(['--mode', 'ycbv_all', '--ycb_dir', 'nowhere', '--class_ids', '2', '--outdir', 'o', '--reinit_below', '0.25',
                 '--init_keep', '3', '--init_icp', '0'] + BASE + CKPT)
    assert seen['reinit'] == {'below': 0.25, 'init': {'keep': 3, 'icp': 0}} and 'init' not in seen
    with pytest.raises(SystemExit, match='stop'):
        pr.main(['--mode', 'ycbv_all', '--ycb_dir', 'nowhere', '--class_ids', '2', '--outdir', 'o', '--reinit_below', '0.5',
                 '--reinit_after', '4'] + BASE + CKPT)
    assert seen['reinit'] == {'below': 0.5, 'after': 4, 'init': None}
    # refused today, refused still: --init_* without --init mask or --reinit_below
    with pytest.raises(SystemExit, match='need --init mask'):
        pr.main(['--mode', 'ycbv_all', '--init_keep', '3'] + BASE + CKPT)


def test_step_options_carry_reinit(pr):
    off = pr.step_options()
    assert off.reinit is None and off.tau is None and off == pr.StepOptions(None, None, None, 1, 0)
    on = pr.step_options(reinit={'below': 0.4})
    assert on.reinit == {'below': 0.4, 'after': 3, 'init': None} and on.tau == pr.FIT_TAU_DEFAULT and on.fit is None
    assert pr.step_options(fit=7, reinit={}).tau == 7
    assert pickle.loads(pickle.dumps(on)) == on
    assert pr.reinit_keep(off) == 1 and pr.reinit_keep(on) == 8 and pr.reinit_keep(pr.step_options(reinit={'init': {'keep': 3}})) == 3
    with pytest.raises(ValueError, match='fit must not be off'):
        pr.step_options(fit=False, fit_switch=True, reinit={})
    with pytest.raises(ValueError, match='below'):
        pr.step_options(reinit={'below': 0})


def test_driver_refuses_bad_reinit_before_reading(pr):
    with pytest.raises(ValueError, match='after'):
        pr.getResultsYcbAll('nowhere', [1], {}, 'out', reinit={'below': 0.5, 'after': 0})
