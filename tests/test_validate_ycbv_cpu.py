"""CPU-only: the one-pass YCB-Video scorer's queues and batches (problems.PairQueues), driven by a stand-in engine that appends on
the host and records every validation step:

  * each class's steps are problems.batch_plan over its kept-pair count, on its pairs in count order, across frame boundaries
  * every full batch runs in every mode before the queue moves on, and its steps read the same queue rows
  * the partial last batches are flushed at the end; a class without a kept pair is reported with 0 pairs
  * fp8 calibrates each class once, on its first step
"""
import importlib

import numpy as np
import pytest
import torch

P = importlib.import_module('iros20-6d-pose-tracking_b200.problems')
S = 176
PLANES = ('rgbA', 'depthA', 'rgbB', 'depthB')


class StandIn:
    """The calls PairQueues makes, on CPU tensors.  A pair's id g is A_in_cam[0, 3] and rgbA[0, 0, 0] = g % 251."""
    device = torch.device('cpu')

    def __init__(self, max_batch):
        self.max_batch = max_batch
        self.calls = []

    def append_pairs(self, pairs, A_in_cam, B_in_cam, queue_ids, tails_host, tails_dev, queues, queue_ids_dev=None):
        cap = queues['rgbA'].shape[1]
        assert A_in_cam.shape[0] <= self.max_batch
        assert np.all(np.asarray(tails_host) >= tails_dev.numpy())           # the host's capacity check uses a bound of the tails
        for q in set(queue_ids.tolist()):
            assert tails_host[q] + int(np.sum(queue_ids == q)) <= cap
        for i, q in enumerate(queue_ids.tolist()):
            if int(pairs['count'][i]) < 100:
                continue
            s = int(tails_dev[q])
            for k in PLANES:
                queues[k][q, s] = pairs[k][i]
            queues['A_in_cam'][q, s] = A_in_cam[i]
            queues['B_in_cam'][q, s] = B_in_cam[i]
            tails_dev[q] += 1
        self.calls.append(('append',))

    def calibrate_fp8_pairs(self, rgbA, depthA, rgbB, depthB, A_in_cam, weight_ids=None):
        self.calls.append(('calibrate', int(weight_ids[0]), A_in_cam[:, 0, 3].long().tolist()))

    def eval_pairs(self, rgbA, depthA, rgbB, depthB, A_in_cam, B_in_cam, tn, rn, weight_ids_host=None, weight_ids_dev=None,
                   precision='bf16x3', out_trans=None, out_rot=None, out_sums=None):
        ids = A_in_cam[:, 0, 3].long().tolist()
        assert rgbA[:, 0, 0, 0].tolist() == [g % 251 for g in ids]
        assert B_in_cam[:, 1, 3].long().tolist() == [g // 1000 for g in ids]   # each pair keeps its frame's B_in_cam
        assert (tn, rn) == (0.01 * weight_ids_host[0], 0.1)
        self.calls.append(('eval', int(weight_ids_host[0]), precision, ids, A_in_cam.data_ptr(), out_trans.data_ptr()))
        out_trans.copy_(A_in_cam[:, :3, 3].float()); out_rot.zero_()
        out_sums[0] = float(sum(ids)); out_sums[1] = float(len(ids))


def frames(rng, classes, n_frames, num_sample, chunk):
    """Synthetic frames as ycbv_pair_steps yields them, and {class: kept pair ids in count order}."""
    kept = {c: [] for c in classes}
    out = []
    for f in range(n_frames):
        owners, rows = [], []
        for c in classes:
            n = int(rng.integers(0, num_sample + 1))
            if n == 0:
                continue
            B = np.eye(4); B[1, 3] = f
            owners.append((c, B, [None] * n, len(rows)))
            for j in range(n):
                g = f * 1000 + len(rows)
                ok = c != 9 and rng.random() < 0.7                  # class 9 never keeps a pair
                rows.append((g, 150 if ok else int(rng.integers(0, 100))))
                if ok:
                    kept[c].append(g)
        if not rows:
            continue
        chunks = []
        for i0 in range(0, len(rows), chunk):
            part = rows[i0:i0 + chunk]
            n = len(part)
            res = {'rgbA': torch.zeros(n, S, S, 3, dtype=torch.uint8), 'depthA': torch.zeros(n, S, S, dtype=torch.uint16),
                   'rgbB': torch.zeros(n, S, S, 3, dtype=torch.uint8), 'depthB': torch.zeros(n, S, S, dtype=torch.uint16),
                   'count': torch.tensor([cnt for _, cnt in part], dtype=torch.int32)}
            A = torch.zeros(n, 4, 4, dtype=torch.float64)
            for j, (g, _) in enumerate(part):
                A[j, :3, 3] = torch.tensor([g, 1.0, 2.0], dtype=torch.float64)
                res['rgbA'][j, 0, 0, 0] = g % 251
            res['A_in_cam'] = A
            chunks.append((i0, res))
        out.append((owners, chunks))
    return out, kept


@pytest.mark.parametrize('batch_size,max_batch,modes', [(5, 3, ['bf16', 'fp8', 'fp32']), (4, 4, ['tf32']), (7, 2, ['fp8', 'bf16x3'])])
def test_batches_follow_batch_plan(batch_size, max_batch, modes):
    rng = np.random.default_rng(batch_size * 10 + max_batch)
    classes, num_sample = (3, 5, 9), 6
    eng = StandIn(max_batch=16)
    q = P.PairQueues(eng, {c: (0.01 * c, 0.1) for c in classes}, modes, batch_size, max_batch, num_sample)
    fr, kept = frames(rng, classes, 12, num_sample, chunk=5)
    for owners, chunks in fr:
        q.add(owners, chunks)
    res = q.finish()
    step = min(batch_size, max_batch)
    assert sum(len(v) for v in kept.values()) > 2 * batch_size
    for c in classes:
        ids = kept[c]
        evals = [call for call in eng.calls if call[0] == 'eval' and call[1] == c]
        expect = []
        plan = P.batch_plan(len(ids), batch_size, step)
        for b in range(plan[-1][0] + 1 if plan else 0):
            for m in modes:                                          # a batch in every mode before the next batch
                expect += [(m, ids[s:e], s) for bb, s, e in plan if bb == b]
        assert [(call[2], call[3]) for call in evals] == [(m, g) for m, g, _ in expect], c
        # a step reads the same queue rows whichever batch it belongs to
        by_offset = {}
        for call, (_, _, s) in zip(evals, expect):
            by_offset.setdefault((s - s // batch_size * batch_size, len(call[3])), set()).add(call[4])
        assert all(len(v) == 1 for v in by_offset.values())
        assert len({call[5] for call in evals}) == (1 if ids else 0)
        cal = [call for call in eng.calls if call[0] == 'calibrate' and call[1] == c]
        if 'fp8' in modes and ids:
            assert cal == [('calibrate', c, ids[:min(step, len(ids))])]
        else:
            assert cal == []
        for m in modes:
            r = res[c][m]
            assert r['pairs'] == len(ids)
            if not ids:
                assert r['trans'] is None and r['rot'] is None and r['predictions'] is None and len(r['batch_trans']) == 0
                continue
            sums = np.array([[sum(ids[s:e]), e - s] for _, s, e in plan], dtype=np.float32)
            bt, br = P.batch_means(sums, plan)
            assert np.array_equal(r['batch_trans'], bt) and np.array_equal(r['batch_rot'], br)
            assert r['trans'] == P._mean_over_batches(bt)
    assert res[9][modes[0]]['pairs'] == 0


def test_predictions_in_count_order():
    rng = np.random.default_rng(7)
    eng = StandIn(max_batch=16)
    q = P.PairQueues(eng, {3: (0.03, 0.1), 5: (0.05, 0.1)}, ['bf16', 'tf32'], 4, 3, 5, keep_predictions=True)
    fr, kept = frames(rng, (3, 5), 9, 5, chunk=16)
    for owners, chunks in fr:
        q.add(owners, chunks)
    res = q.finish()
    for c in (3, 5):
        for m in ('bf16', 'tf32'):
            p = res[c][m]['predictions']
            assert p.shape == (len(kept[c]), 6)
            assert p[:, 0].astype(np.int64).tolist() == kept[c]


def test_rejects_steps_above_the_engine():
    with pytest.raises(ValueError):
        P.PairQueues(StandIn(max_batch=2), {3: (0.03, 0.1)}, ['bf16'], 5, 3, 4)
