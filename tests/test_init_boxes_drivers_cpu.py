"""The start-from-box options of the command line and the drivers without a GPU: --init box needs --mode ycbv_all or
ycbv_init and refuses --reinit_below, --init_depths needs --init box and a value in [1, 8], and the drivers' own arguments are
refused before anything is read."""
import importlib
import numpy as np
import pytest

PKG = 'iros20-6d-pose-tracking_b200'
BASE = ['--train_data_path', 'nowhere/train', '--model_path', 'nowhere/m.ply']
CKPT = ['--ckpt_dir', 'nowhere/c.pth', '--mean_std_path', 'nowhere']


@pytest.fixture(scope='module')
def pr():
    return importlib.import_module(PKG + '.predict')


@pytest.mark.parametrize('mode', ['ycbv', 'ycbineoat', 'ycbineoat_all', 'ycbv_recover', 'other'])
def test_init_box_needs_ycbv_all_or_ycbv_init(pr, mode):
    with pytest.raises(SystemExit, match='--init box needs --mode ycbv_all or ycbv_init'):
        pr.main(['--mode', mode, '--init', 'box'] + BASE + CKPT)


@pytest.mark.parametrize('argv', [
    ['--mode', 'ycbv_all', '--init_depths', '2'],
    ['--mode', 'ycbv_all', '--init', 'mask', '--init_depths', '2'],
    ['--mode', 'ycbv_init', '--init_depths', '3'],
])
def test_init_depths_need_init_box(pr, argv):
    with pytest.raises(SystemExit, match='--init_depths needs --init box'):
        pr.main(argv + BASE + CKPT)


@pytest.mark.parametrize('depths', ['0', '9', '-1'])
def test_init_depths_out_of_range(pr, depths):
    with pytest.raises(SystemExit, match='--init_depths: init depths must be an integer in \\[1, 8\\]'):
        pr.main(['--mode', 'ycbv_all', '--init', 'box', '--init_depths', depths] + BASE + CKPT)


def test_init_box_refuses_restarts(pr):
    with pytest.raises(SystemExit, match='--init box with --reinit_below'):
        pr.main(['--mode', 'ycbv_all', '--init', 'box', '--reinit_below', '0.5'] + BASE + CKPT)


def test_init_box_takes_the_init_options(pr):
    # the --init_* options are accepted with --init box; the run then fails on the missing data set, not on the options
    with pytest.raises(SystemExit) as e:
        pr.main(['--mode', 'ycbv_all', '--init', 'box', '--init_depths', '2', '--init_keep', '3'] + BASE + CKPT)
    assert 'need --init mask' not in str(e.value) and 'init_depths' not in str(e.value)


def test_driver_arguments(pr):
    with pytest.raises(ValueError, match="depths needs initialize_method='box'"):
        pr.getResultsYcbAll('nowhere', [1], {}, 'out', initialize_method='mask', depths=2)
    with pytest.raises(ValueError, match="need initialize_method='mask' or 'box'"):
        pr.getResultsYcbAll('nowhere', [1], {}, 'out', initialize_method='gt', init={'keep': 2})
    with pytest.raises(ValueError, match='depths'):
        pr.getResultsYcbAll('nowhere', [1], {}, 'out', initialize_method='box', depths=0)
    with pytest.raises(ValueError, match='depths needs box'):
        pr.initYcbKeyframes('nowhere', [1], {}, depths=2)


def test_label_boxes(pr):
    seg = np.zeros((6, 8), np.uint8)
    seg[1:3, 2:5] = 3
    seg[5, 7] = 3
    seg[0, 0] = 9
    assert pr.label_boxes(seg, [3, 9, 4]).tolist() == [[2, 1, 8, 6], [0, 0, 1, 1], [0, 0, 0, 0]]
