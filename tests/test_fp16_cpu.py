"""The 'fp16' precision mode's entry points on the CPU: the mode table, and the one-pass drivers' choice of modes."""
import importlib

import numpy as np
import pytest

from test_ycbineoat_all_cpu import no_device, object_files, pr, templates, video   # noqa: F401 (fixtures)


def test_fp16_is_a_mode():
    lib = importlib.import_module('iros20-6d-pose-tracking_b200._lib')
    engine = importlib.import_module('iros20-6d-pose-tracking_b200.engine')
    assert lib.PREC_FP16 == 5 and engine.PREC['fp16'] == lib.PREC_FP16
    assert sorted(engine.PREC.values()) == list(range(6))


def test_ycb_all_modes_are_engine_modes_but_fp16(pr):
    engine = importlib.import_module('iros20-6d-pose-tracking_b200.engine')
    assert set(pr.YCB_ALL_PRECISIONS) == set(engine.PREC) - {'fp16'}


def test_ycbineoat_driver_takes_fp16(pr, tmp_path, no_device):
    """'fp16' passes the YCBInEOAT driver's precision check: the first refusal is the missing checkpoint that follows it."""
    data, cfg = tmp_path / 'data', tmp_path / 'cfg'
    video(data, 'bleach0')
    object_files(cfg, 'bleach')
    (cfg / 'bleach' / 'ckpt.pth.tar').unlink()
    with pytest.raises(FileNotFoundError, match='checkpoint'):
        pr.getResultsYcbInEOAT(str(data), templates(cfg), str(tmp_path / 'out'), precision='fp16')
    with pytest.raises(ValueError, match='precision'):
        pr.getResultsYcbInEOAT(str(data), templates(cfg), str(tmp_path / 'out'), precision='fp4')
