"""ICP in the drivers on the synthetic layouts of the driver tests: icp=0 writes the trees a run without it writes, icp=M writes
the poses its ICP steps returned (one ICP step per frame, the fit rows after ICP), and ycbv_recover's icp rows follow
round K with the round rows unchanged."""
import numpy as np
import pytest
import torch
from test_gpu_precision_sweep import eoat, ycbv, pr      # noqa: F401
from test_gpu_fit import _poses_tree, _fits
from test_gpu_ycbv_recover import mods, layout, CLASSES, NUM_SAMPLE, SEED      # noqa: F401

pytestmark = pytest.mark.gpu
TAU = 15


def _recording(pr):
    E = pr.Engine
    orig = E.track_render
    got = []

    def rec(self, *a, **kw):
        res = orig(self, *a, **kw)
        got.append((res[0].cpu().numpy().copy(), kw.get('icp')))
        return res
    return E, rec, got


def test_ycbineoat_icp(pr, eoat, monkeypatch):
    tmp, tpl = eoat
    data, ycb = str(tmp / 'data'), str(tmp / 'ycb')
    run = lambda out, **kw: pr.getResultsYcbInEOAT(data, tpl, str(tmp / 'icp' / out), ycb_dir=ycb, max_frames=4, **kw)
    run('plain', fit=TAU)
    run('zero', fit=TAU, icp=0)
    a, b = str(tmp / 'icp' / 'plain'), str(tmp / 'icp' / 'zero')
    assert _poses_tree(a) == _poses_tree(b) and all(np.array_equal(x, _fits(b)[k]) for k, x in _fits(a).items())
    E, rec, got = _recording(pr)
    monkeypatch.setattr(E, 'track_render', rec)
    two = run('two', icp=2, icp_tau=30)
    steps = iter(got)
    for v, _ in sorted(pr.ycbineoat_videos(data)):                  # one n = 1 step per frame, videos in run order
        want = [next(steps) for _ in range(len(two[v]))]
        assert np.array_equal(two[v], np.stack([w[0][0] for w in want]))
        assert all(w[1] == {'iterations': 2, 'tau_mm': 30} for w in want)
    assert next(steps, None) is None
    monkeypatch.undo()
    with_fit = run('two_fit', icp=2, icp_tau=30, fit=TAU)
    assert all(np.array_equal(two[v], with_fit[v]) for v in two)       # the fit check reads the refined poses, never writes them
    if torch.cuda.device_count() >= 2:
        run('two_gpus', icp=2, icp_tau=30, gpus=2)
        assert _poses_tree(str(tmp / 'icp' / 'two_gpus')) == _poses_tree(str(tmp / 'icp' / 'two'))


def test_ycbv_icp(pr, ycbv):
    tmp, tpl = ycbv
    ycb = str(tmp / 'ycb')
    run = lambda out, **kw: pr.getResultsYcbAll(ycb, [2, 5, 7], tpl, str(tmp / 'icp' / out), **kw)
    run('plain')
    run('zero', icp=0)
    assert _poses_tree(str(tmp / 'icp' / 'plain')) == _poses_tree(str(tmp / 'icp' / 'zero'))
    three = run('three', icp=3, fit=TAU)
    again = run('again', icp=3)
    assert all(np.array_equal(three[c][s], again[c][s]) for c in three for s in three[c])
    fits = _fits(str(tmp / 'icp' / 'three'))
    assert fits and all((f[0] == -1).all() for f in fits.values())
    with pytest.raises(ValueError, match='hypotheses'):
        run('refused', icp=2, hypotheses=4)


def test_recover_icp(layout, mods):
    pr = mods['predict']
    kw = dict(num_sample=NUM_SAMPLE, seed=SEED, iterations=2)
    plain = pr.recoverYcbKeyframes(layout['ycb'], CLASSES, layout['tpl'], **kw)
    icp = pr.recoverYcbKeyframes(layout['ycb'], CLASSES, layout['tpl'], icp=3, **kw)
    assert list(plain) == list(icp)
    for v in plain:
        for c in plain[v]:
            p, q = plain[v][c], icp[v][c]
            assert q['icp'] == 3 and len(q['summary']) == 2 + 1 + 3 and q['poses'].shape[0] == 2 + 3
            assert np.array_equal(p['poses'], q['poses'][:2]) and np.array_equal(p['errors'], q['errors'][:3])
            assert p['summary'] == q['summary'][:3]
    assert icp[next(iter(icp))]['all']['rows'] > 0
    pr.print_recover_tables(icp, {c: str(c) for c in CLASSES})
