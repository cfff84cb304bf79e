"""Multi-hypothesis tracking in the drivers on the synthetic layouts of the driver tests: --hypotheses 1 writes the trees a run
without it writes, --hypotheses 4 --fit writes the kept poses and rows of its track_hypotheses steps, two GPUs write one GPU's
trees, and ycbv_recover's selected / best-of-S rows follow the steps and bound each other."""
import importlib
import os
import numpy as np
import pytest
import torch
import yaml
from test_gpu_precision_sweep import eoat, ycbv, pr      # noqa: F401
from test_gpu_fit import _poses_tree, _fits

pytestmark = pytest.mark.gpu
PKG = 'iros20-6d-pose-tracking_b200'
TAU = 15


def _with_spread(cfg_root):
    """The layouts' dataset_info.yml with the spread of training pairs (dataset_info.yml:12-13) the hypotheses draw with."""
    for d, _, fs in os.walk(str(cfg_root)):
        if 'dataset_info.yml' in fs:
            p = os.path.join(d, 'dataset_info.yml')
            info = yaml.safe_load(open(p))
            info.setdefault('max_translation', 0.02)
            info.setdefault('max_rotation', 15)
            yaml.safe_dump(info, open(p, 'w'))


def _recording(pr):
    E = pr.Engine
    orig = E.track_hypotheses
    got = []

    def rec(self, *a, **kw):
        res = orig(self, *a, **kw)
        got.append((res[0].cpu().numpy().copy(), res[2].cpu().numpy().copy(), kw.get('seed')))
        return res
    return E, rec, got


def test_ycbineoat_hypotheses(pr, eoat, monkeypatch):
    tmp, tpl = eoat
    _with_spread(tmp / 'cfg')
    data, ycb = str(tmp / 'data'), str(tmp / 'ycb')
    run = lambda out, **kw: pr.getResultsYcbInEOAT(data, tpl, str(tmp / 'hyp' / out), ycb_dir=ycb, max_frames=4, **kw)
    run('plain', fit=TAU)
    run('one', fit=TAU, hypotheses=1, seed=5)
    a, b = str(tmp / 'hyp' / 'plain'), str(tmp / 'hyp' / 'one')
    assert _poses_tree(a) == _poses_tree(b) and all(np.array_equal(x, _fits(b)[k]) for k, x in _fits(a).items())
    E, rec, got = _recording(pr)
    monkeypatch.setattr(E, 'track_hypotheses', rec)
    four = run('four', fit=TAU, hypotheses=4, seed=5)
    fits = _fits(str(tmp / 'hyp' / 'four'))
    steps = iter(got)
    for v, _ in sorted(pr.ycbineoat_videos(data)):                  # one n = 1 step per frame, videos in run order
        want = [next(steps) for _ in range(len(four[v]))]
        assert np.array_equal(four[v], np.stack([w[0][0] for w in want]))
        assert np.array_equal(fits[v], np.stack([w[1][0] for w in want])) and all(w[2] == 5 for w in want)
    assert next(steps, None) is None
    again = run('again', fit=TAU, hypotheses=4, seed=5)
    assert all(np.array_equal(four[v], again[v]) for v in four)
    if torch.cuda.device_count() >= 2:
        run('two', fit=TAU, hypotheses=4, seed=5, gpus=2)
        assert _poses_tree(str(tmp / 'hyp' / 'two')) == _poses_tree(str(tmp / 'hyp' / 'four'))


def test_ycbv_hypotheses(pr, ycbv):
    tmp, tpl = ycbv
    _with_spread(tmp / 'cfg')
    ycb = str(tmp / 'ycb')
    run = lambda out, **kw: pr.getResultsYcbAll(ycb, [2, 5, 7], tpl, str(tmp / 'hyp' / out), **kw)
    run('plain')
    run('one', hypotheses=1)
    assert _poses_tree(str(tmp / 'hyp' / 'plain')) == _poses_tree(str(tmp / 'hyp' / 'one'))
    run('four', hypotheses=4, fit=TAU)
    fits = _fits(str(tmp / 'hyp' / 'four'))
    assert fits and all((f[0] == -1).all() and (f[1:, 0] > 0).all() for f in fits.values())
    if torch.cuda.device_count() >= 2:
        run('two', hypotheses=4, fit=TAU, gpus=2)
        assert _poses_tree(str(tmp / 'hyp' / 'two')) == _poses_tree(str(tmp / 'hyp' / 'four'))


from test_gpu_ycbv_recover import mods, layout, CLASSES, NUM_SAMPLE, SEED      # noqa: E402,F401


def test_recover_hypotheses(layout, mods):
    pr = mods['predict']
    E = pr.Engine
    orig, seen = E.track_hypotheses, []

    def rec(self, *a, **kw):
        res = orig(self, *a, **kw)
        seen.append(res[0].cpu().numpy().copy())
        return res
    E.track_hypotheses = rec
    try:
        res = pr.recoverYcbKeyframes(layout['ycb'], CLASSES + (7,), layout['tpl'], num_sample=NUM_SAMPLE, seed=SEED, iterations=2,
                                     hypotheses=4)
    finally:
        E.track_hypotheses = orig
    (v, r), = res.items()
    allr = r['all']
    assert allr['rows'] > 0 and set(allr) >= {'selected', 'best'}
    sel, best = allr['selected'], allr['best']
    # every selected pose is one the steps kept (rows are kept in step order, some rows masked out)
    stepped = np.concatenate(seen)
    assert all(any(np.array_equal(p, q) for q in stepped) for p in sel['poses'])
    adds0, adds_sel, adds_best = allr['errors'][-1][:, 3], sel['errors'][:, 3], best['errors'][:, 3]
    assert (adds_best <= adds0).all() and (adds_best <= adds_sel).all()
    assert ((sel['choice'] >= 0) & (sel['choice'] < 4)).all()
    assert sel['summary']['rows'] == best['summary']['rows'] == allr['rows']
    pr.print_recover_tables(res, {c: str(c) for c in CLASSES + (7,)})
