"""CPU-only: the one-pass YCB-Video scorer under the train-time augmentations (problems.PairQueues(augment=...)), driven by a
stand-in engine that appends on the host and records every augmentation, calibration and validation step:

  * each queued row carries its segB, which moves with it through appends and remainder compactions
  * a batch is augmented once, in steps of at most max_batch rows, before any variant runs; each row's pair index is its
    index in its class's count order, across frame boundaries and compactions
  * every variant and fp8 calibration reads the augmented buffer, whose address never changes
  * without augment there is no segB plane and no augmentation call
  * the CLI passes --ycb_dir --augment config.yml --seed S to validate_ycbv as the chain and the seed
"""
import importlib
import inspect

import numpy as np
import pytest
import torch
import yaml

P = importlib.import_module('iros20-6d-pose-tracking_b200.problems')
S = 176
PLANES = ('rgbA', 'depthA', 'rgbB', 'depthB')
AUG = object()                                                  # stands for a se3tn_augment


def _ids(img):
    """The pair id g a plane carries in its first two bytes (g % 251, g // 251)."""
    flat = img.reshape(img.shape[0], img[0].numel() if img.shape[0] else 2)
    return (flat[:, 0].long() + 251 * flat[:, 1].long()).tolist()


class StandIn:
    """The calls PairQueues makes, on CPU tensors.  Pair g has A_in_cam[0, 3] = g, and its rgbA, rgbB and segB start with
    (g % 251, g // 251).  The augmented rgbB keeps those bytes and marks its third byte 255."""
    device = torch.device('cpu')

    def __init__(self, max_batch):
        self.max_batch = max_batch
        self.calls = []
        self.queues = None

    def append_pairs(self, pairs, A_in_cam, B_in_cam, queue_ids, tails_host, tails_dev, queues, queue_ids_dev=None):
        self.queues = queues
        planes = PLANES + (('segB',) if 'segB' in queues else ())
        for i, q in enumerate(queue_ids.tolist()):
            if int(pairs['count'][i]) < 100:
                continue
            s = int(tails_dev[q])
            for k in planes:
                queues[k][q, s] = pairs[k][i]
            queues['A_in_cam'][q, s] = A_in_cam[i]
            queues['B_in_cam'][q, s] = B_in_cam[i]
            tails_dev[q] += 1
        self.calls.append(('append', 'segB' in queues))

    def augment_crops(self, augment, rgbB, depthB, pair_index, segB=None, out_rgbB=None, out_depthB=None):
        assert augment is AUG and rgbB.shape[0] <= self.max_batch
        assert _ids(segB) == _ids(rgbB)                             # segB is the row's own
        out_rgbB.copy_(rgbB); out_depthB.copy_(depthB)
        out_rgbB[:, 0, 0, 2] = 255
        self.calls.append(('augment', _ids(rgbB), pair_index.tolist(), out_rgbB.data_ptr()))
        return out_rgbB, out_depthB

    def calibrate_fp8_pairs(self, rgbA, depthA, rgbB, depthB, A_in_cam, weight_ids=None):
        self.calls.append(('calibrate', int(weight_ids[0]), A_in_cam[:, 0, 3].long().tolist(), _ids(rgbB),
                           rgbB[:, 0, 0, 2].tolist(), rgbB.data_ptr()))

    def eval_pairs(self, rgbA, depthA, rgbB, depthB, A_in_cam, B_in_cam, tn, rn, weight_ids_host=None, weight_ids_dev=None,
                   precision='bf16x3', out_trans=None, out_rot=None, out_sums=None):
        ids = A_in_cam[:, 0, 3].long().tolist()
        assert _ids(rgbA) == ids and _ids(rgbB) == ids
        self.calls.append(('eval', int(weight_ids_host[0]), precision, ids, rgbB[:, 0, 0, 2].tolist(), rgbB.data_ptr()))
        out_trans.copy_(A_in_cam[:, :3, 3].float()); out_rot.zero_()
        out_sums[0] = float(sum(ids)); out_sums[1] = float(len(ids))


def frames(rng, classes, n_frames, num_sample, chunk):
    """Synthetic frames as ycbv_pair_steps yields them (with segB), and {class: kept pair ids in count order}."""
    kept = {c: [] for c in classes}
    out = []
    g = 0
    for f in range(n_frames):
        owners, rows = [], []
        for c in classes:
            n = int(rng.integers(0, num_sample + 1))
            if n == 0:
                continue
            owners.append((c, np.eye(4), [None] * n, len(rows)))
            for _ in range(n):
                ok = c != 9 and rng.random() < 0.7                  # class 9 never keeps a pair
                rows.append((g, 150 if ok else int(rng.integers(0, 100))))
                if ok:
                    kept[c].append(g)
                g += 1
        if not rows:
            continue
        chunks = []
        for i0 in range(0, len(rows), chunk):
            part = rows[i0:i0 + chunk]
            n = len(part)
            res = {'rgbA': torch.zeros(n, S, S, 3, dtype=torch.uint8), 'depthA': torch.zeros(n, S, S, dtype=torch.uint16),
                   'rgbB': torch.zeros(n, S, S, 3, dtype=torch.uint8), 'depthB': torch.zeros(n, S, S, dtype=torch.uint16),
                   'segB': torch.zeros(n, S, S, dtype=torch.uint8), 'count': torch.tensor([cnt for _, cnt in part], dtype=torch.int32)}
            A = torch.zeros(n, 4, 4, dtype=torch.float64)
            for j, (gj, _) in enumerate(part):
                A[j, 0, 3] = gj
                for k in ('rgbA', 'rgbB', 'segB'):
                    res[k].view(n, -1)[j, :2] = torch.tensor([gj % 251, gj // 251], dtype=torch.uint8)
            res['A_in_cam'] = A
            chunks.append((i0, res))
        out.append((owners, chunks))
    return out, kept


def _run(batch_size, max_batch, modes, augment, ckpts=1, seed=0):
    rng = np.random.default_rng(seed)
    classes, num_sample = (3, 5, 9), 6
    eng = StandIn(max_batch=16)
    q = P.PairQueues(eng, {c: (0.01 * c, 0.1) for c in classes}, modes, batch_size, max_batch, num_sample, ckpts=ckpts,
                     augment=augment)
    fr, kept = frames(rng, classes, 14, num_sample, chunk=5)
    for owners, chunks in fr:
        q.add(owners, chunks)
    return q, eng, q.finish(), kept


@pytest.mark.parametrize('batch_size,max_batch,modes,ckpts', [(5, 3, ['bf16', 'fp8'], 1), (4, 4, ['tf32'], 2), (7, 2, ['fp8', 'fp32'], 2)])
def test_each_batch_is_augmented_once_with_count_order_indices(batch_size, max_batch, modes, ckpts):
    q, eng, res, kept = _run(batch_size, max_batch, modes, AUG, ckpts, seed=batch_size)
    step = min(batch_size, max_batch)
    assert 'segB' in q.queues and q.queues['segB'].shape == q.queues['depthB'].shape
    assert all(seg for name, seg in (c[:2] for c in eng.calls if c[0] == 'append'))
    assert sum(len(v) for v in kept.values()) > 3 * batch_size       # several batches, so the queues were compacted
    aug_ptr = q.aug_rgbB.data_ptr()
    row = S * S * 3
    augments = [c for c in eng.calls if c[0] == 'augment']
    for c in (3, 5, 9):
        ids = kept[c]
        plan = P.batch_plan(len(ids), batch_size, step)
        mine = [a for a in augments if a[1] and a[1][0] in ids]
        # one augmentation per step of each batch, not per variant; every row once, keyed by its count-order index
        assert [a[1] for a in mine] == [ids[s:e] for _, s, e in plan], c
        assert [a[2] for a in mine] == [list(range(s, e)) for _, s, e in plan], c
        assert [a[3] for a in mine] == [aug_ptr + (s % batch_size) * row for _, s, e in plan]
        evals = [x for x in eng.calls if x[0] == 'eval' and x[1] % P.CKPT_ID_STRIDE == c]
        assert len(evals) == len(plan) * len(modes) * ckpts
        for x in evals:                                             # every variant reads the augmented buffer
            assert set(x[4]) == {255} and aug_ptr <= x[5] < aug_ptr + batch_size * row
        cal = [x for x in eng.calls if x[0] == 'calibrate' and x[1] % P.CKPT_ID_STRIDE == c]
        if 'fp8' in modes and ids:
            assert [x[1] for x in cal] == [c + P.CKPT_ID_STRIDE * i for i in range(ckpts)]
            for x in cal:
                assert x[2] == x[3] == ids[:min(step, len(ids))] and set(x[4]) == {255} and x[5] == aug_ptr
        else:
            assert cal == []
        # the augmentation of a batch comes before any of its steps
        order = [i for i, x in enumerate(eng.calls) if (x[0] == 'augment' and x in mine) or x in evals]
        kinds = [eng.calls[i][0] for i in order]
        per_batch = [sum(1 for b, _, _ in plan if b == bb) for bb in range(plan[-1][0] + 1)] if plan else []
        expect = []
        for k in per_batch:
            expect += ['augment'] * k + ['eval'] * (k * len(modes) * ckpts)
        assert kinds == expect, c
    for i in range(ckpts):
        r = res[i] if ckpts > 1 else res
        for c in (3, 5):
            assert r[c][modes[0]]['pairs'] == len(kept[c])
        assert r[9][modes[0]]['pairs'] == 0


def test_segB_moves_with_its_row():
    """After every add the queued segB of each live row carries the same id as its rgbB and A_in_cam."""
    rng = np.random.default_rng(11)
    eng = StandIn(max_batch=16)
    q = P.PairQueues(eng, {3: (0.03, 0.1), 5: (0.05, 0.1)}, ['bf16'], 4, 3, 6, augment=AUG)
    fr, kept = frames(rng, (3, 5), 12, 6, chunk=4)
    for owners, chunks in fr:
        q.add(owners, chunks)
        q._drain(final=False)
        for qi in range(2):
            t = int(q.tails[qi])
            d = {k: q.queues[k][qi, :t] for k in ('rgbB', 'segB', 'A_in_cam')}
            assert _ids(d['segB']) == _ids(d['rgbB']) == d['A_in_cam'][:, 0, 3].long().tolist()
    q.finish()
    assert sum(len(v) for v in kept.values()) > 8


def test_without_augment_no_segB_plane_and_no_augment_call():
    class NoAugment(StandIn):
        def augment_crops(self, *a, **kw):
            raise AssertionError('augmented without augment')

    rng = np.random.default_rng(3)
    eng = NoAugment(max_batch=16)
    q = P.PairQueues(eng, {3: (0.03, 0.1), 5: (0.05, 0.1)}, ['bf16', 'fp8'], 5, 3, 6)
    fr, kept = frames(rng, (3, 5), 10, 6, chunk=5)
    for owners, chunks in fr:
        q.add(owners, chunks)
    res = q.finish()
    assert 'segB' not in q.queues and not hasattr(q, 'aug_rgbB')
    assert not any(seg for name, seg in (c[:2] for c in eng.calls if c[0] == 'append'))
    for x in eng.calls:
        if x[0] == 'eval':                                          # the queue's own rgbB, not marked
            assert set(x[4]) == {0}
    assert res[3]['bf16']['pairs'] == len(kept[3])


CONFIG = {'data_augmentation': {'hsv_noise': [15, 15, 15], 'bright_mag': [0.5, 1.5], 'gaussian_noise': {'rgb': 0.1, 'depth': 0.1},
                                'gaussian_blur_kernel': 7}}


def test_cli_ycb_dir_augment_reaches_validate_ycbv(tmp_path, monkeypatch, capsys):
    (tmp_path / 'CADmodels' / '001_a').mkdir(parents=True)
    (tmp_path / 'CADmodels' / '002_b').mkdir(parents=True)
    cfg = tmp_path / 'config.yml'
    yaml.safe_dump(CONFIG, open(cfg, 'w'))
    seen = {}

    def validate_ycbv(ycb_dir, ids, templates, **kw):
        seen.update(kw, ids=ids)
        r = dict(pairs=3, trans=0.5, rot=0.25, batch_trans=np.zeros(1, np.float32), batch_rot=np.zeros(1, np.float32), predictions=None)
        return {c: {'bf16': dict(r)} for c in ids}

    monkeypatch.setattr(P, 'validate_ycbv', validate_ycbv)
    monkeypatch.setattr(torch.cuda, 'current_device', lambda: 0)
    monkeypatch.setattr(torch.cuda, 'get_device_name', lambda dev=None: 'card')
    P.main(['--ycb_dir', str(tmp_path), '--class_ids', 'all', '--ckpt_dir', 'c', '--mean_std_path', 's', '--train_data_path', 't',
            '--model_path', 'm', '--precision', 'bf16', '--seed', '7', '--augment', str(cfg)])
    out = capsys.readouterr()
    assert seen['ids'] == [1, 2] and seen['seed'] == 7 and seen['augment_seed'] == 7
    chain = seen['augmentations']
    assert [type(t).__name__ for t in chain.transforms] == ['HSVJitter', 'ChangeBright', 'GaussianNoise', 'GaussianBlur', 'BlackCover']
    assert out.out.count(", augmented (train.py's chain, seed 7)") == 2
    assert 'works with --val_dir only' not in out.err
    assert 'segB for BlackCover' not in inspect.getsource(P)
    # an incomplete --ycb_dir run is refused before anything runs, naming what it lacks
    seen.clear()
    with pytest.raises(SystemExit):
        P.main(['--ycb_dir', str(tmp_path), '--class_ids', '1', '--ckpt_dir', 'c', '--augment', str(cfg)])
    err = capsys.readouterr().err
    assert 'or with a whole --ycb_dir run: --ycb_dir needs --class_ids, --ckpt_dir, --mean_std_path' in err and not seen
    # without --augment: no chain, and the header says nothing of it
    P.main(['--ycb_dir', str(tmp_path), '--class_ids', '1', '--ckpt_dir', 'c', '--mean_std_path', 's', '--train_data_path', 't',
            '--model_path', 'm', '--precision', 'bf16'])
    assert seen['augmentations'] is None and 'augmented' not in capsys.readouterr().out
