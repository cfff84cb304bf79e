"""The start-from-mask options of the command line without a GPU: --init_* need --init mask (with --mode ycbv_all) or --mode
ycbv_init, --init mask needs --mode ycbv_all, ycbv_init refuses the tracking options, and values Engine.init_spec refuses are
refused before anything is read."""
import importlib
import pytest

PKG = 'iros20-6d-pose-tracking_b200'
BASE = ['--train_data_path', 'nowhere/train', '--model_path', 'nowhere/m.ply']
CKPT = ['--ckpt_dir', 'nowhere/c.pth', '--mean_std_path', 'nowhere']


@pytest.fixture(scope='module')
def pr():
    return importlib.import_module(PKG + '.predict')


@pytest.mark.parametrize('argv', [
    ['--mode', 'ycbv_all', '--init_viewpoints', '12'] + CKPT,
    ['--mode', 'ycbv_all', '--init', 'gt', '--init_keep', '3'] + CKPT,
    ['--mode', 'ycbv_all', '--init', 'posecnn', '--init_icp', '0'] + CKPT,
    ['--mode', 'ycbineoat_all', '--init_inplane', '4'] + CKPT,
])
def test_init_options_need_init_mask(pr, argv):
    with pytest.raises(SystemExit, match='need --init mask'):
        pr.main(argv + BASE)


@pytest.mark.parametrize('mode', ['ycbv', 'ycbineoat', 'ycbineoat_all', 'ycbv_recover', 'ycbv_init', 'other'])
def test_init_mask_needs_ycbv_all(pr, mode):
    with pytest.raises(SystemExit, match='--init mask needs --mode ycbv_all'):
        pr.main(['--mode', mode, '--init', 'mask'] + BASE + CKPT)


@pytest.mark.parametrize('mode', ['ycbv', 'ycbineoat', 'ycbv_recover', 'other'])
def test_ycbv_init_options_are_refused_in_other_modes(pr, mode):
    with pytest.raises(SystemExit, match='need --init mask'):
        pr.main(['--mode', mode, '--init_keep', '2'] + BASE + CKPT)


@pytest.mark.parametrize('extra', [['--outdir', 'x'], ['--precision', 'bf16'], ['--icp', '2'], ['--gpus', '2'], ['--score'],
                                   ['--iterations', '2']])
def test_ycbv_init_refuses_tracking_options(pr, extra):
    with pytest.raises(SystemExit, match='does not track'):
        pr.main(['--mode', 'ycbv_init', '--ycb_dir', 'nowhere', '--class_ids', '1'] + extra + BASE)


@pytest.mark.parametrize('flag,value', [('--init_viewpoints', '0'), ('--init_inplane', '361'), ('--init_keep', '33'),
                                        ('--init_icp', '17')])
def test_init_values_are_checked_first(pr, flag, value):
    for argv in (['--mode', 'ycbv_all', '--init', 'mask'] + CKPT, ['--mode', 'ycbv_init']):
        with pytest.raises(SystemExit, match='--init_'):
            pr.main(argv + [flag, value] + BASE)


def test_ycbv_init_needs_no_checkpoint_but_the_others_do(pr):
    with pytest.raises(SystemExit, match='needs --ycb_dir and --class_ids'):
        pr.main(['--mode', 'ycbv_init'] + BASE)
    with pytest.raises(SystemExit):
        pr.main(['--mode', 'ycbv_all'] + BASE)


def test_driver_refuses_init_options_without_mask(pr):
    with pytest.raises(ValueError, match="initialize_method='mask'"):
        pr.getResultsYcbAll('nowhere', [1], {}, 'out', initialize_method='gt', init=dict(keep=2))
    with pytest.raises(ValueError):
        pr.getResultsYcbAll('nowhere', [1], {}, 'out', initialize_method='mask', init=dict(keep=0))
