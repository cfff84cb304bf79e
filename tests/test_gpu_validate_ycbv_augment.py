"""The one-pass scorer of perturbed YCB-Video key frames under the train-time augmentations (problems.validate_ycbv with
augmentations, se3tn_append_pairs_seg), on the synthetic layout of test_gpu_validate_ycbv and the reference's config.yml chain:

  * bit-identical to the file route (produce_train_pair_data --mode ycbv, then problems.evaluate on each class's folder through
    TrackDataset(augmentations=..., augment_seed=...)) in every precision mode, with batches split into steps and latency-mode
    steps, under an augmentation seed other than the generator's: pair counts, per-batch MSEs, means and predictions; every stage
    of the chain fires on some pair, and the losses differ from the plain one pass
  * random / np.random end in the same state after both routes; fp8's scales of every class equal the file route's
  * two checkpoints: each one's results those of a run of it alone, with each batch augmented once, not once per variant
  * a class's full batches after its first replay their CUDA graphs; a class without a kept pair is reported with 0 pairs
  * se3tn_append_pairs_seg against numpy (kept and rejected rows, several queues with non-zero tails, segB in its row's slot,
    poisoned slots left alone, null or misaligned seg pointers refused with every buffer unchanged), and its other planes, poses
    and tails byte for byte those of se3tn_append_pairs
"""
import ctypes as C
import importlib
import random

import numpy as np
import pytest
import torch
import yaml

from test_gpu_augment import REF_CONFIG
from test_gpu_validate_ycbv import mods, layout, _rng_state, _same_rng, CLASSES, MODES, NUM_SAMPLE, SEED, BATCH, MAX_BATCH  # noqa: F401
from test_gpu_checkpoint_sweep import second_checkpoints, same_results

pytestmark = pytest.mark.gpu
AUG = importlib.import_module('iros20-6d-pose-tracking_b200.data_augmentation')
AUG_SEED = 11                                                   # not the generator's seed: the draws follow it


def _chain():
    """train.py:85-92's chain from the reference's config.yml, every stage on."""
    return AUG.from_config(REF_CONFIG)


@pytest.fixture(scope='module')
def file_route(layout, mods):
    """--mode ycbv into folders, then the augmented evaluate on each class's folder: (counts, RNG state after writing,
    {class: {mode: dict}}, {class: fp8 scales})."""
    PP, P, D = mods['produce_train_pair_data'], mods['problems'], mods['datasets']
    out = layout['root'] / 'pairs_aug'
    counts = PP.produce_ycbv(layout['ycb'], CLASSES, layout['tpl'], str(out), num_sample=NUM_SAMPLE, seed=SEED)
    state = _rng_state()
    eng = mods['engine'].Engine(max_batch=MAX_BATCH)
    res, scales = {}, {}
    for c in CLASSES:
        d = layout['cfg'] / ('c%d' % c)
        info = yaml.safe_load(open(d / 'dataset_info.yml'))
        ds = D.TrackDataset(str(out / ('%03d_obj' % c)), 'val', np.load(str(d / 'mean.npy')), np.load(str(d / 'std.npy')), None,
                            _chain(), None, dataset_info=info, trans_normalizer=info['max_translation'],
                            rot_normalizer=info['max_rotation'] * np.pi / 180, augment_seed=AUG_SEED)
        assert len(ds) == counts[c]
        model = mods['se3_tracknet'].Se3TrackNet(engine=eng, weight_id=0)
        model.load_state_dict(torch.load(str(d / 'model_best_val.pth.tar'), map_location='cpu')['state_dict'])
        res[c] = {}
        for m in MODES:
            res[c][m] = P.evaluate(model, ds, BATCH, precision=m, keep_predictions=True)
            if m == 'fp8':
                scales[c] = eng.fp8_scales(0)
    return counts, state, res, scales, out


def test_every_stage_fires(mods, file_route):
    """The chain's draws on the written pairs, as evaluate keys them: every stage is taken on some pair."""
    D, counts, out = mods['datasets'], file_route[0], file_route[4]
    eng = mods['engine'].Engine(max_batch=max(counts.values()))
    aug = AUG.chain_config(_chain(), AUG_SEED)
    fired = np.zeros(5, bool)
    for c in CLASSES:
        files = sorted(str(f) for f in (out / ('%03d_obj' % c)).glob('*rgbA.png'))
        pairs = [D.read_pair(f) for f in files]
        dB = torch.from_numpy(np.stack([p['depthB'] for p in pairs])).to(eng.device)
        seg = torch.from_numpy(np.stack([D.segB_plane(p['segB']) for p in pairs])).to(eng.device)
        params, _, _ = eng.augment_draws(aug, dB, torch.arange(len(files), dtype=torch.int64, device=eng.device), segB=seg)
        p = params.cpu().numpy()
        fired |= [p[:, 1:4].any(), p[:, 7].any(), (p[:, 9] + p[:, 11]).any(), (p[:, 13] + p[:, 15]).any(),
                  ((p[:, 17] > 0) & (p[:, 20] >= 0)).any()]
    assert fired.all(), fired


def test_bit_identical_to_the_augmented_file_route(layout, mods, file_route):
    counts, state, ref, scales, _ = file_route
    P = mods['problems']
    assert all(counts[c] > BATCH for c in CLASSES)
    random.seed(123); np.random.seed(123)
    eng = mods['engine'].Engine(max_batch=NUM_SAMPLE * len(CLASSES))
    res = P.validate_ycbv(layout['ycb'], CLASSES, layout['tpl'], num_sample=NUM_SAMPLE, seed=SEED, batch_size=BATCH,
                          max_batch=MAX_BATCH, precisions=MODES, keep_predictions=True, engine=eng, augmentations=_chain(),
                          augment_seed=AUG_SEED)
    assert _same_rng(_rng_state(), state)
    for c in CLASSES:
        plan = P.batch_plan(counts[c], BATCH, MAX_BATCH)
        assert any(e - s <= 4 for _, s, e in plan) and len({b for b, _, _ in plan}) > 1
        for m in MODES:
            r, f = res[c][m], ref[c][m]
            assert r['pairs'] == counts[c], (c, m)
            assert np.array_equal(r['batch_trans'], f['batch_trans']) and np.array_equal(r['batch_rot'], f['batch_rot']), (c, m)
            assert r['trans'] == f['trans'] and r['rot'] == f['rot'], (c, m)
            assert np.array_equal(r['predictions'], f['predictions']), (c, m)
            assert np.isfinite(r['trans']) and np.isfinite(r['rot'])
        assert scales[c] is not None and np.array_equal(eng.fp8_scales(c), scales[c]), c
    plain = P.validate_ycbv(layout['ycb'], CLASSES, layout['tpl'], num_sample=NUM_SAMPLE, seed=SEED, batch_size=BATCH,
                            max_batch=MAX_BATCH, precisions=['bf16x3'])
    assert any(plain[c]['bf16x3']['pairs'] == counts[c] and plain[c]['bf16x3']['trans'] != res[c]['bf16x3']['trans'] for c in CLASSES)


def test_two_checkpoints_augment_each_batch_once(layout, mods, synth, file_route):
    counts = file_route[0]
    P = mods['problems']
    ck, st = second_checkpoints(layout['root'], synth, ['c%d' % c for c in CLASSES + (7,)], 90)
    tpl2 = dict(layout['tpl'], ckpt_dir=ck.replace('{key}', 'c{class_id}'), mean_std_path=st.replace('{key}', 'c{class_id}'))
    both = dict(layout['tpl'], ckpt_dir=[layout['tpl']['ckpt_dir'], tpl2['ckpt_dir']],
                mean_std_path=[layout['tpl']['mean_std_path'], tpl2['mean_std_path']])
    kw = dict(num_sample=NUM_SAMPLE, seed=SEED, batch_size=BATCH, max_batch=MAX_BATCH, precisions=['bf16x3', 'fp8'],
              keep_predictions=True, augmentations=_chain(), augment_seed=AUG_SEED)
    eng = mods['engine'].Engine(max_batch=NUM_SAMPLE * len(CLASSES))
    calls = []
    inner = eng.augment_crops

    def augment_crops(*a, **kw):
        calls.append(int(a[3].shape[0]))
        return inner(*a, **kw)

    eng.augment_crops = augment_crops
    res = P.validate_ycbv(layout['ycb'], CLASSES, both, engine=eng, **kw)
    # one call per step of each class's batches (the drain interleaves the classes), not one per checkpoint and mode
    assert sorted(calls) == sorted(e - s for c in CLASSES for _, s, e in P.batch_plan(counts[c], BATCH, MAX_BATCH))
    assert sorted(res) == [0, 1]
    for i, tpl in enumerate((layout['tpl'], tpl2)):
        same_results(res[i], P.validate_ycbv(layout['ycb'], CLASSES, tpl, **kw))


def test_full_batches_replay_their_graphs(layout, mods, file_route):
    counts = file_route[0]
    P = mods['problems']
    eng = mods['engine'].Engine(max_batch=NUM_SAMPLE * len(CLASSES))
    log = []
    inner = eng.eval_pairs

    def eval_pairs(*a, **kw):
        out = inner(*a, **kw)
        log.append((int(kw['weight_ids_host'][0]), kw['precision'], int(a[0].shape[0]), eng.last_step_was_graph()))
        return out

    eng.eval_pairs = eval_pairs
    modes = ['bf16', 'tf32']
    res = P.validate_ycbv(layout['ycb'], CLASSES, layout['tpl'], num_sample=NUM_SAMPLE, seed=SEED, batch_size=BATCH,
                          max_batch=MAX_BATCH, precisions=modes, engine=eng, augmentations=_chain(), augment_seed=AUG_SEED)
    for c in CLASSES:
        assert res[c]['bf16']['pairs'] == counts[c]
        plan = P.batch_plan(counts[c], BATCH, MAX_BATCH)
        for m in modes:
            calls = [x for x in log if x[:2] == (c, m)]
            assert [n for _, _, n, _ in calls] == [e - s for _, s, e in plan]
            for (b, s, e), (_, _, _, graph) in zip(plan, calls):
                if b > 0 and (b + 1) * BATCH <= counts[c]:
                    assert graph, (c, m, b, s)


def test_no_kept_pair(layout, mods, file_route):
    P = mods['problems']
    res = P.validate_ycbv(layout['ycb'], (3, 7), layout['tpl'], num_sample=NUM_SAMPLE, seed=SEED, batch_size=BATCH,
                          max_batch=MAX_BATCH, precisions=['bf16'], augmentations=_chain(), augment_seed=AUG_SEED)
    r = res[7]['bf16']
    assert r['pairs'] == 0 and r['trans'] is None and r['rot'] is None and len(r['batch_trans']) == 0
    assert res[3]['bf16']['pairs'] > 0 and np.isfinite(res[3]['bf16']['trans'])


def test_append_pairs_seg_against_numpy(mods):
    L, E = mods['_lib'], mods['engine']
    eng = E.Engine(max_batch=8)
    rng = np.random.default_rng(1)
    S = 176
    Q, cap, n = 3, 6, 7

    def dev(x):
        return torch.from_numpy(np.ascontiguousarray(x)).to(eng.device)

    p = {'rgbA': dev(rng.integers(0, 256, (n, S, S, 3), dtype=np.uint8)), 'depthA': dev(rng.integers(0, 65536, (n, S, S), dtype=np.uint16)),
         'rgbB': dev(rng.integers(0, 256, (n, S, S, 3), dtype=np.uint8)), 'depthB': dev(rng.integers(0, 65536, (n, S, S), dtype=np.uint16)),
         'segB': dev(rng.integers(0, 2, (n, S, S), dtype=np.uint8)), 'count': dev(np.array([150, 99, 100, 0, 300, 101, 50], np.int32))}
    poisoned = {'rgbA': dev(rng.integers(0, 256, (Q, cap, S, S, 3), dtype=np.uint8)),
                'depthA': dev(rng.integers(0, 65536, (Q, cap, S, S), dtype=np.uint16)),
                'rgbB': dev(rng.integers(0, 256, (Q, cap, S, S, 3), dtype=np.uint8)),
                'depthB': dev(rng.integers(0, 65536, (Q, cap, S, S), dtype=np.uint16)),
                'A_in_cam': dev(rng.standard_normal((Q, cap, 4, 4))), 'B_in_cam': dev(rng.standard_normal((Q, cap, 4, 4))),
                'segB': dev(rng.integers(2, 256, (Q, cap, S, S), dtype=np.uint8))}
    queues = {k: v.clone() for k, v in poisoned.items()}
    tails0 = np.array([1, 0, 2], np.int32)
    tails = dev(tails0)
    qids = np.array([2, 0, 2, 1, 0, 2, 2], np.int32)
    qdev = dev(qids)
    A, B = dev(rng.standard_normal((n, 4, 4))), dev(rng.standard_normal((n, 4, 4)))

    def snapshot(qs, t):
        torch.cuda.synchronize()
        return {k: v.cpu().numpy().copy() for k, v in qs.items()}, t.cpu().numpy().copy()

    before, _ = snapshot(queues, tails)

    def raw(seg, q_seg):
        return eng.lib.se3tn_append_pairs_seg(eng._ctx, *(E._ptr(p[k]) for k in ('rgbA', 'depthA', 'rgbB', 'depthB', 'count')),
                                              E._ptr(A), E._ptr(B), E._hptr(qids), E._ptr(qdev), n, Q, cap, E._hptr(tails0),
                                              E._ptr(tails), *(E._ptr(queues[k]) for k in ('rgbA', 'depthA', 'rgbB', 'depthB', 'A_in_cam', 'B_in_cam')),
                                              seg, q_seg, E._stream(eng.device))

    seg_ptr, q_seg_ptr = p['segB'].data_ptr(), queues['segB'].data_ptr()
    for seg, q_seg in ((0, q_seg_ptr), (seg_ptr, 0), (0, 0), (seg_ptr + 1, q_seg_ptr), (seg_ptr, q_seg_ptr + 8)):
        assert raw(C.c_void_p(seg), C.c_void_p(q_seg)) == L.ERR_INVALID
        q_now, t_now = snapshot(queues, tails)
        assert np.array_equal(t_now, tails0) and all(np.array_equal(q_now[k], before[k]) for k in before)
    with pytest.raises(ValueError):                                 # the queues carry segB, the pairs do not
        eng.append_pairs({k: v for k, v in p.items() if k != 'segB'}, A, B, qids, tails0, tails, queues)

    eng.append_pairs(p, A, B, qids, tails0, tails, queues)
    assert eng.last_launch_count() == 1
    after, t_after = snapshot(queues, tails)
    expect = {k: v.copy() for k, v in before.items()}
    t = tails0.copy()
    host = {k: v.cpu().numpy() for k, v in p.items()}
    An, Bn = A.cpu().numpy(), B.cpu().numpy()
    for i, q in enumerate(qids):
        if host['count'][i] < L.PAIR_MIN_SEG:
            continue
        for k in ('rgbA', 'depthA', 'rgbB', 'depthB', 'segB'):
            expect[k][q, t[q]] = host[k][i]
        expect['A_in_cam'][q, t[q]] = An[i]; expect['B_in_cam'][q, t[q]] = Bn[i]
        t[q] += 1
    assert t.tolist() == [2, 0, 5] and np.array_equal(t_after, t)
    for k in expect:
        assert np.array_equal(after[k], expect[k]), k

    # the same append without the seg plane writes the same bytes everywhere else
    plain = {k: v.clone() for k, v in poisoned.items() if k != 'segB'}
    plain_tails = dev(tails0)
    eng.append_pairs(p, A, B, qids, tails0, plain_tails, plain)
    got, t_plain = snapshot(plain, plain_tails)
    assert np.array_equal(t_plain, t_after)
    for k in got:
        assert got[k].tobytes() == after[k].tobytes(), k
