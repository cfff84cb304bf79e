"""Several checkpoints in one pass, against runs of each checkpoint alone, on synthetic checkpoints with distinct seeds and
statistics:

  * problems.evaluate with 3 checkpoints x {bf16x3, fp8, fp32}, plain and augmented: every (checkpoint, mode) result bit for bit
    a one-model evaluate, a partial last batch of 4 pairs (the latency-mode step) included, each pair decoded once
  * input B augmented once by se3tn_augment_crops, then se3tn_eval_pairs: bit for bit se3tn_eval_pairs_augmented, sums included
  * problems.validate_ycbv with 2 checkpoints: per checkpoint what validate_ycbv of that checkpoint alone returns
  * getResultsYcbInEOAT / getResultsYcbAll with 2 checkpoints x {bf16x3, fp8} x iterations [1, 2]: each checkpoint's tree file for
    file, its return value and fp8 scales those of a run of it alone; each frame decoded once and stepped once per variant, and
    every captured variant replaying its graph after its first steps; gpus=2 (two ranks on cuda:0) equal to one process
  * --score over checkpoints: the reference row has no drift, and the selection line names the highest ADD-S AUC
"""
import contextlib, importlib, io, os, threading
import numpy as np
import pytest
import torch

from test_gpu_validate import write_folder, TN, RN
from test_gpu_augment import REF_CONFIG
from test_gpu_precision_sweep import pr, eoat, ycbv, recording, same_tree, VIDEOS, CLASSES as YCB_CLASSES   # noqa: F401
from test_gpu_validate_ycbv import mods, layout, CLASSES as VAL_CLASSES, NUM_SAMPLE, SEED   # noqa: F401

pytestmark = pytest.mark.gpu
PKG = 'iros20-6d-pose-tracking_b200'
MODES = ['bf16x3', 'fp8', 'fp32']
N_PAIRS, BATCH = 13, 9                      # batches of 9 and 4 pairs: the last one runs the latency-mode step
INFO = {'resolution': 176, 'max_translation': TN, 'max_rotation': 15,
        'camera': {'focalX': 1066.778, 'focalY': 1067.487, 'centerX': 312.9869, 'centerY': 241.3109}}


def M(name):
    return importlib.import_module(PKG + '.' + name)


@pytest.fixture(scope='module')
def val(tmp_path_factory, synth):
    folder = str(tmp_path_factory.mktemp('ckval') / 'val')
    eng = M('engine').Engine(max_batch=BATCH)
    eng.set_mesh(synth.mesh(), 0)
    write_folder(eng, synth, folder, N_PAIRS, seed=3)
    eng.close()
    mean, std = synth.default_mean_std()
    stats = [(mean + 0.5 * i, std * (1 + 0.05 * i)) for i in range(3)]
    sds = [synth.make_state_dict(20 + i) for i in range(3)]
    return folder, stats, sds


def dataset(folder, mean, std, augment):
    aug = M('data_augmentation').from_config(REF_CONFIG) if augment else None
    return M('datasets').TrackDataset(folder, 'val', mean, std, None, aug, None, dataset_info=INFO, trans_normalizer=TN,
                                      rot_normalizer=RN, augment_seed=7)


@pytest.mark.parametrize('augment', [False, True])
def test_evaluate_checkpoints_equal_single_runs(val, augment, monkeypatch):
    P, S, E = M('problems'), M('se3_tracknet'), M('engine')
    folder, stats, sds = val
    single, scales = {}, {}
    for i, sd in enumerate(sds):
        eng = E.Engine(max_batch=BATCH)
        model = S.Se3TrackNet(engine=eng, weight_id=0)
        model.load_state_dict(sd)
        ds = dataset(folder, *stats[i], augment)
        for m in MODES:
            single[i, m] = P.evaluate(model, ds, BATCH, precision=m, keep_predictions=True)
        scales[i] = eng.fp8_scales(0)
        eng.close()
    reads, lock, orig = [], threading.Lock(), P.read_pair

    def read_pair(path):
        with lock:
            reads.append(path)
        return orig(path)
    monkeypatch.setattr(P, 'read_pair', read_pair)
    eng = E.Engine(max_batch=BATCH)
    models = []
    for i, sd in enumerate(sds):
        models.append(S.Se3TrackNet(engine=eng, weight_id=i))
        models[-1].load_state_dict(sd)
    res = P.evaluate(models, dataset(folder, *stats[0], augment), BATCH, False, MODES, keep_predictions=True, stats=stats)
    assert sorted(reads) == sorted(set(reads)) and len(reads) == N_PAIRS        # each pair decoded once for all 9 variants
    assert list(res) == [(i, m) for i in range(3) for m in MODES]
    for key, r in res.items():
        f = single[key]
        assert np.array_equal(r['batch_trans'], f['batch_trans']) and np.array_equal(r['batch_rot'], f['batch_rot']), key
        assert r['trans'] == f['trans'] and r['rot'] == f['rot'], key
        assert np.array_equal(r['predictions'], f['predictions']), key
    for i in range(3):
        assert np.array_equal(eng.fp8_scales(i), scales[i]), i
    assert res[0, 'fp32']['trans'] != res[1, 'fp32']['trans']                  # the checkpoints do differ
    eng.close()


def test_augment_once_equals_the_augmented_step(val):
    D, E = M('datasets'), M('engine')
    folder, stats, sds = val
    ds = dataset(folder, *stats[0], True)
    eng = E.Engine(max_batch=N_PAIRS)
    eng.load_state_dict(sds[0], 0)
    eng.set_stats(np.asarray(stats[0][0]), np.asarray(stats[0][1]), 0)
    pairs = [D.read_pair(f) for f in ds.rgbA_files]
    t = lambda k, dt=None: torch.from_numpy(np.ascontiguousarray(np.stack([p[k] for p in pairs]))).to(eng.device)
    d = {k: t(k) for k in ('rgbA', 'depthA', 'rgbB', 'depthB', 'A_in_cam', 'B_in_cam')}
    seg = torch.from_numpy(np.stack([D.segB_plane(p['segB'] if p['segB'] is not None else p['depthB'] > 100) for p in pairs])).to(eng.device)
    idx = torch.arange(N_PAIRS, dtype=torch.int64, device=eng.device)
    for m in ('bf16x3', 'fp32'):
        for s, e in ((0, N_PAIRS), (2, 6)):
            fused = eng.eval_pairs(d['rgbA'][s:e], d['depthA'][s:e], d['rgbB'][s:e], d['depthB'][s:e], d['A_in_cam'][s:e],
                                   d['B_in_cam'][s:e], TN, RN, precision=m, augment=ds.augment, segB=seg[s:e], pair_index=idx[s:e])
            fused = [x.clone() for x in fused[:3]]
            rB, dB = eng.augment_crops(ds.augment, d['rgbB'][s:e], d['depthB'][s:e], idx[s:e], segB=seg[s:e])
            once = eng.eval_pairs(d['rgbA'][s:e], d['depthA'][s:e], rB, dB, d['A_in_cam'][s:e], d['B_in_cam'][s:e], TN, RN, precision=m)
            for a, b in zip(fused, once[:3]):
                assert torch.equal(a, b), (m, s, e)
    eng.close()


def second_checkpoints(root, synth, names, seed0):
    """A second checkpoint and statistics per name under root/ck2 -> (checkpoint template, statistics template) with {key}."""
    mean, std = synth.default_mean_std()
    for j, n in enumerate(names):
        os.makedirs(root / 'ck2' / n, exist_ok=True)
        torch.save({'state_dict': synth.make_state_dict(seed0 + j)}, str(root / 'ck2' / n / 'model.pth.tar'))
        np.save(str(root / 'ck2' / n / 'mean.npy'), mean - 1 - j); np.save(str(root / 'ck2' / n / 'std.npy'), std * (0.9 - 0.02 * j))
    return str(root / 'ck2' / '{key}' / 'model.pth.tar'), str(root / 'ck2' / '{key}')


def same_results(a, b):
    if isinstance(a, dict):
        assert list(a) == list(b)
        for k in a:
            same_results(a[k], b[k])
    elif isinstance(a, np.ndarray):
        assert np.array_equal(a, b)
    else:
        assert a == b


def test_validate_ycbv_checkpoints(layout, mods, synth):
    P = mods['problems']
    ck, st = second_checkpoints(layout['root'], synth, ['c%d' % c for c in VAL_CLASSES + (7,)], 60)
    tpl2 = dict(layout['tpl'], ckpt_dir=ck.replace('{key}', 'c{class_id}'), mean_std_path=st.replace('{key}', 'c{class_id}'))
    both = dict(layout['tpl'], ckpt_dir=[layout['tpl']['ckpt_dir'], tpl2['ckpt_dir']],
                mean_std_path=[layout['tpl']['mean_std_path'], tpl2['mean_std_path']])
    kw = dict(num_sample=NUM_SAMPLE, seed=SEED, batch_size=5, max_batch=3, precisions=['bf16x3', 'fp8'], keep_predictions=True)
    res = P.validate_ycbv(layout['ycb'], VAL_CLASSES, both, **kw)
    assert sorted(res) == [0, 1]
    for i, tpl in enumerate((layout['tpl'], tpl2)):
        same_results(res[i], P.validate_ycbv(layout['ycb'], VAL_CLASSES, tpl, **kw))


def with_checkpoints(root, synth, templates, key, names):
    """templates with a second checkpoint of every class / object ({key} placeholder) -> (both, second alone)."""
    ck, st = second_checkpoints(root, synth, names, 80)
    second = dict(templates, ckpt_dir=ck.replace('{key}', key), mean_std_path=st.replace('{key}', key))
    both = dict(templates, ckpt_dir=[templates['ckpt_dir'], second['ckpt_dir']],
                mean_std_path=[templates['mean_std_path'], second['mean_std_path']])
    return both, second


SWEEP = dict(precision=['bf16x3', 'fp8'], iterations=[1, 2])


def check_against_single(pr, run, tmp, both, alone, wids, frames):
    """run(templates, outdir, **kw) with both checkpoints against runs of each alone."""
    with recording(pr) as (steps, decodes):
        res = run(both, str(tmp / 'both'), **SWEEP)
        eng = steps[-1][0]
        scales = {w + 32 * i: eng.fp8_scales(w + 32 * i) for w in wids for i in range(2)}
    assert decodes == {'rgb': frames, 'depth': frames}
    assert len(steps) == frames * 8                                       # 2 checkpoints x 2 modes x 2 counts per frame
    firsts = {}
    for _, m, w, n, graph in steps:
        if not graph:
            firsts[m, w, n] = firsts.get((m, w, n), 0) + 1
    for (m, w, n), count in firsts.items():
        assert m == 'fp32' or count <= 2, (m, w, n, count)                   # one capture per count k, then replays
    assert sorted(os.listdir(tmp / 'both')) == ['ckpt0', 'ckpt1']
    for i, tpl in enumerate(alone):
        with recording(pr) as (steps, _):
            one = run(tpl, str(tmp / ('alone%d' % i)), **SWEEP)
            eng = steps[-1][0]
            for w in wids:
                assert np.array_equal(eng.fp8_scales(w), scales[w + 32 * i]), (i, w)
        same_results(res[i], one)
        same_tree(str(tmp / 'both' / ('ckpt%d' % i)), str(tmp / ('alone%d' % i)))
    return res


def test_ycbineoat_all_checkpoints(pr, eoat, synth):
    tmp, templates = eoat
    objects = M('eval_ycbineoat').OBJECTS
    both, second = with_checkpoints(tmp, synth, templates, '{object}', sorted(set(VIDEOS.values())))
    wids = sorted(set(objects.index(o) for o in VIDEOS.values()))
    run = lambda tpl, out, **kw: pr.getResultsYcbInEOAT(str(tmp / 'data'), tpl, out, **kw)
    res = check_against_single(pr, run, tmp / 'ck_eoat', both, (templates, second), wids, 4 * len(VIDEOS))
    # two processes on the one card: the same trees and return value
    with pytest.MonkeyPatch.context() as m:
        m.setattr(torch.cuda, 'device_count', lambda: 2)
        m.setattr(pr, '_rank_devices', lambda n: [0] * n)
        two = run(both, str(tmp / 'ck_eoat' / 'two'), gpus=2, **SWEEP)
    same_results(res, two)
    for i in range(2):
        same_tree(str(tmp / 'ck_eoat' / 'both' / ('ckpt%d' % i)), str(tmp / 'ck_eoat' / 'two' / ('ckpt%d' % i)))
    # --score: one row per variant, drift from ckpt0/iter1/bf16x3, and the best ADD-S per mode and count
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        pr.main(['--mode', 'ycbineoat_all', '--YCBInEOAT_dir', str(tmp / 'data'), '--ycb_dir', str(tmp / 'ycb'),
                 '--train_data_path', templates['train_data_path'], '--model_path', templates['model_path'],
                 '--ckpt_dir', ','.join(both['ckpt_dir']), '--mean_std_path', ','.join(both['mean_std_path']),
                 '--outdir', str(tmp / 'ck_eoat' / 'cli'), '--precision', 'bf16x3,fp8', '--iterations', '1,2', '--score'])
    text = out.getvalue()
    ref, rows = pr.score_checkpoints(res, str(tmp / 'ck_eoat' / 'both'), str(tmp / 'ycb'), both, str(tmp / 'data'), ['bf16x3', 'fp8'], [1, 2])
    assert ref == os.path.join('ckpt0', 'iter1', 'bf16x3') and rows[ref]['add_max'] == 0 and rows[ref]['adds_max'] == 0
    assert len(rows) == 8 and 'checkpoint sweep' in text
    for sub in ('iter1/bf16x3', 'iter1/fp8', 'iter2/bf16x3', 'iter2/fp8'):
        adds = [rows['ckpt%d/%s' % (i, sub)]['adds'] for i in range(2)]
        b = 0 if adds[0] >= adds[1] else 1
        assert ('best %s: checkpoint %d (%s)' % (sub, b, both['ckpt_dir'][b])) in text


def test_ycbv_all_checkpoints(pr, ycbv, synth):
    tmp, templates = ycbv
    both, second = with_checkpoints(tmp, synth, templates, 'c{class_id}', ['c%d' % c for c in YCB_CLASSES])
    run = lambda tpl, out, **kw: pr.getResultsYcbAll(str(tmp / 'ycb'), list(YCB_CLASSES), tpl, out, **kw)
    check_against_single(pr, run, tmp / 'ck_ycbv', both, (templates, second), list(YCB_CLASSES), 3 * 2)
