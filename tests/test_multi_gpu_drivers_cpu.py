"""Host logic of the one-pass drivers on several GPUs (getResultsYcbAll / getResultsYcbInEOAT with gpus=N, predict --gpus): how
sequences are shared out over ranks, where each rank calibrates the fp8 sets it cannot calibrate itself, what is refused before
any process starts, the files and return value of a split run with the tracking faked, and a failing rank's error and teardown.
CPU only; the tracked poses, scales and videos are checked on the GPU (test_gpu_multi_gpu_drivers.py)."""
import importlib, multiprocessing, os
import numpy as np
import pytest
import torch
import yaml
from test_precision_sweep_cpu import pr, no_device, refusal_trees, tree_files, K_INFO      # noqa: F401


def test_assign_ranks_longest_first():
    costs = [5, 9, 2, 9, 4, 1, 7]
    plan = importlib.import_module('iros20-6d-pose-tracking_b200.predict').assign_ranks(costs, 3)
    # 9 (#1) -> r0, 9 (#3) -> r1, 7 (#6) -> r2, 5 (#0) -> r2, 4 (#4) -> r0 (r0 and r1 tie at 9 with one each), 2 (#2) -> r1,
    # 1 (#5) -> r1
    assert plan == [[1, 4], [2, 3, 5], [0, 6]]
    assert [sum(costs[i] for i in r) for r in plan] == [13, 12, 12]


def test_assign_ranks_properties(pr):
    rng = np.random.default_rng(0)
    for n_seq in (1, 2, 5, 9, 17):
        costs = [int(c) for c in rng.integers(0, 50, n_seq)]
        for gpus in (1, 2, 3, 8, 20):
            plan = pr.assign_ranks(costs, gpus)
            assert plan == pr.assign_ranks(list(costs), gpus)                       # deterministic
            assert len(plan) == min(gpus, n_seq) and all(plan)                      # no rank without a sequence
            assert sorted(i for r in plan for i in r) == list(range(n_seq))          # each sequence exactly once
            assert all(r == sorted(r) for r in plan)                                # a rank runs its sequences in run order
            loads = [sum(costs[i] for i in r) for r in plan]
            # greedy longest first: no rank is over the lightest by more than the longest sequence it was given last
            assert max(loads) - min(loads) <= max(costs)
    assert pr.assign_ranks([], 4) == []
    assert pr.assign_ranks([3, 3, 3, 3], 2) == [[0, 2], [1, 3]]                     # ties: run order, then the lowest rank
    assert pr.assign_ranks([0, 0, 0], 3) == [[0], [1], [2]]
    assert pr.assign_ranks([10, 1, 1, 1, 1, 1], 2) == [[0], [1, 2, 3, 4, 5]]


def test_borrowed_calibration_frames(pr):
    sets = [(2, 5, 7), (2, 5, 9), (7, 9), (1,), (5, 1)]
    first = {2: 0, 5: 0, 7: 0, 9: 1, 1: 3}
    for mine in ([0, 2], [1], [3, 4], [0, 1, 2, 3, 4], [4], [2]):
        got = pr.borrowed_calibrations(sets, mine)
        need = set(w for k in mine for w in sets[k])
        want = {}
        for w in sorted(need):
            if first[w] not in mine:
                want.setdefault(first[w], []).append(sets[first[w]].index(w))
        assert got == {k: sorted(v) for k, v in sorted(want.items())}, mine
    assert pr.borrowed_calibrations(sets, [0, 2]) == {1: [2]}             # 9 starts in sequence 1
    assert pr.borrowed_calibrations(sets, [1]) == {0: [0, 1]}             # 2 and 5 start in sequence 0; 9 is calibrated at home
    assert pr.borrowed_calibrations(sets, [4]) == {0: [1], 3: [0]}
    assert pr.borrowed_calibrations(sets, [2]) == {0: [2], 1: [2]}
    assert pr.borrowed_calibrations(sets, range(5)) == {}


@pytest.fixture
def no_process(pr, monkeypatch):
    def ranks(*a, **kw):
        raise AssertionError('a process was started before the configuration was checked')
    monkeypatch.setattr(pr, '_track_on_ranks', ranks)


@pytest.mark.parametrize('gpus', [0, -1, 1.5, True])
def test_refuses_fewer_than_one_gpu(pr, tmp_path, no_device, no_process, gpus):
    ycb, ycb_tpl, data, obj_tpl = refusal_trees(tmp_path)
    with pytest.raises(ValueError, match='gpus'):
        pr.getResultsYcbAll(ycb, [2], ycb_tpl, str(tmp_path / 'out'), gpus=gpus)
    with pytest.raises(ValueError, match='gpus'):
        pr.getResultsYcbInEOAT(data, obj_tpl, str(tmp_path / 'out'), gpus=gpus)
    assert not (tmp_path / 'out').exists()


def test_refuses_more_gpus_than_devices(pr, tmp_path, no_device, no_process, monkeypatch):
    ycb, ycb_tpl, data, obj_tpl = refusal_trees(tmp_path)
    monkeypatch.setattr(torch.cuda, 'device_count', lambda: 2)
    loaded = []
    monkeypatch.setattr(pr, 'ycb_all_classes', lambda *a, **kw: loaded.append(a))
    monkeypatch.setattr(pr, 'ycbineoat_objects', lambda *a, **kw: loaded.append(a))
    with pytest.raises(ValueError, match='gpus=3, but 2 CUDA devices'):
        pr.getResultsYcbAll(ycb, [2], ycb_tpl, str(tmp_path / 'out'), gpus=3)
    with pytest.raises(ValueError, match='gpus=3, but 2 CUDA devices'):
        pr.getResultsYcbInEOAT(data, obj_tpl, str(tmp_path / 'out'), gpus=3)
    assert not loaded and not (tmp_path / 'out').exists()
    assert pr.check_gpus(2) == 2 and pr.check_gpus(1) == 1
    monkeypatch.setattr(torch.cuda, 'device_count', lambda: 0)
    assert pr.check_gpus(1) == 1                                          # one GPU asks nothing of the device here


def test_every_check_fails_before_a_process_starts(pr, tmp_path, no_device, no_process, monkeypatch):
    monkeypatch.setattr(torch.cuda, 'device_count', lambda: 8)
    ycb, ycb_tpl, data, obj_tpl = refusal_trees(tmp_path)
    out = str(tmp_path / 'out')
    with pytest.raises(ValueError, match='precision'):
        pr.getResultsYcbAll(ycb, [2], ycb_tpl, out, precision='fp16', gpus=2)
    with pytest.raises(ValueError, match='video'):
        pr.getResultsYcbAll(ycb, [2], ycb_tpl, out, precision=['bf16', 'fp8'], video=True, gpus=2)
    with pytest.raises(ValueError, match='iteration'):
        pr.getResultsYcbInEOAT(data, obj_tpl, out, iterations=[1, 1], gpus=2)
    with pytest.raises(ValueError, match='decode_ahead'):
        pr.getResultsYcbInEOAT(data, obj_tpl, out, decode_ahead=0, gpus=2)
    with pytest.raises(ValueError, match='trans_normalizer'):
        pr.getResultsYcbAll(ycb, [2], dict(ycb_tpl, trans_normalizer={3: 0.1}), out, gpus=2)
    os.remove(os.path.join(os.path.dirname(ycb_tpl['ckpt_dir'].format(class_id=2)), 'ckpt.pth.tar'))
    with pytest.raises(FileNotFoundError, match='class 2'):
        pr.getResultsYcbAll(ycb, [2], ycb_tpl, out, gpus=2)
    os.remove(os.path.join(data, 'bleach0', 'depth_filled', '0000000.png'))
    with pytest.raises(FileNotFoundError, match='depth_filled'):
        pr.getResultsYcbInEOAT(data, obj_tpl, out, gpus=2)
    assert not (tmp_path / 'out').exists()


@pytest.mark.parametrize('mode', ['ycbv', 'ycbineoat', 'class'])
def test_cli_refuses_gpus_outside_the_one_pass_modes(pr, tmp_path, monkeypatch, mode):
    def loaded(*a, **kw):
        raise AssertionError('--gpus was not checked first')
    for name in ('load_run_config', 'predictSequenceYcbInEOAT', 'predictSequenceYcb', 'getResultsYcb'):
        monkeypatch.setattr(pr, name, loaded)
    base = ['--mode', mode, '--train_data_path', 't', '--model_path', 'm', '--ckpt_dir', 'c', '--mean_std_path', 's', '--outdir',
            str(tmp_path / 'o'), '--ycb_dir', 'y', '--YCBInEOAT_dir', 'd', '--seq_id', '48']
    for gpus in ('2', '0'):
        with pytest.raises(SystemExit, match='--gpus'):
            pr.main(base + ['--gpus', gpus])


def test_cli_passes_gpus(pr, tmp_path, monkeypatch):
    (tmp_path / 'y' / 'CADmodels' / '001_obj').mkdir(parents=True)
    calls = []
    monkeypatch.setattr(pr, 'getResultsYcbAll', lambda *a, **kw: calls.append(kw) or {})
    monkeypatch.setattr(pr, 'getResultsYcbInEOAT', lambda *a, **kw: calls.append(kw) or {})
    base = ['--train_data_path', 't', '--model_path', 'm', '--ckpt_dir', 'c', '--mean_std_path', 's', '--outdir', str(tmp_path / 'o'),
            '--ycb_dir', str(tmp_path / 'y'), '--YCBInEOAT_dir', 'd', '--class_ids', '1']
    for mode in ('ycbv_all', 'ycbineoat_all'):
        pr.main(base + ['--mode', mode, '--gpus', '4'])
        pr.main(base + ['--mode', mode])
        with pytest.raises(SystemExit, match='--gpus 0'):
            pr.main(base + ['--mode', mode, '--gpus', '0'])
    assert [kw.get('gpus', '-') for kw in calls] == [4, '-', 4, '-']


class Sent:
    """The child's end of the pipe, in this process: keeps what _rank_main sends."""
    def __init__(self):
        self.msgs = []

    def send(self, msg):
        self.msgs.append(msg)

    def close(self):
        pass


def test_split_run_writes_and_returns_what_one_process_does(pr, tmp_path, monkeypatch):
    """The drivers with the tracking faked (poses that depend on the variant, the sequence's tracks and its initial poses only),
    gpus=3 against gpus=1: each rank's _rank_main runs here, ranks in reverse order, with the borrowed calibrations it was given."""
    seen = {'borrowed': []}

    class Eng:
        def fp8_scales(self, w):
            return np.full(8, float(w), np.float32)
    monkeypatch.setattr(pr, '_one_pass_trackers', lambda entries, precision, max_batch, device=None: (Eng(), {}))
    monkeypatch.setattr(pr, '_calibrate_borrowed', lambda eng, trackers, sequences, borrowed: seen['borrowed'].append(borrowed))
    monkeypatch.setattr(torch.cuda, 'set_device', lambda d: None)
    monkeypatch.setattr(torch.cuda, 'device_count', lambda: 3)

    def loop(eng, trackers, sequences, variants, depth, workers, video, opts, seq_index):
        for rgb_files, _, ids, init in sequences:
            yield {v: np.stack([init * (1 + 0.01 * (t + 1)) + sum(ids) + len(str(v)) for t in range(len(rgb_files))]) for v in variants}, None
    monkeypatch.setattr(pr, '_track_sequences', loop)

    def ranks(gpus, entries, precision, max_batch, sequences, variants, depth, workers, video, writes, opts):
        plan = pr.assign_ranks([len(s[0]) for s in sequences], gpus)
        results = {}
        for r in reversed(range(len(plan))):
            conn = Sent()
            borrowed = pr.borrowed_calibrations([s[2] for s in sequences], plan[r])
            pr._rank_main(conn, r, 0, entries, precision, max_batch, sequences, plan[r], borrowed, variants, depth, workers, video, writes,
                          opts)
            (kind, out, scales), = conn.msgs
            assert kind == 'ok' and sorted(out) == plan[r], conn.msgs
            results.update(out)
        return [results[k] for k in range(len(sequences))]
    monkeypatch.setattr(pr, '_track_on_ranks', ranks)

    ycb = tmp_path / 'ycb'
    for k in range(1, 6):
        (ycb / 'CADmodels' / ('%03d_obj' % k)).mkdir(parents=True)
    for seq, cls, nf in ((48, (2, 3), 4), (49, (3,), 6), (50, (2, 5), 3), (51, (5,), 2)):
        base = ycb / 'data_organized' / ('%04d' % seq)
        for c in cls:
            (base / 'pose_gt' / str(c)).mkdir(parents=True)
            for i in range(nf):
                np.savetxt(str(base / 'pose_gt' / str(c) / ('%06d.txt' % (i + 1))), np.eye(4) * (c + seq + i))
        for sub, name in (('color', '%06d-color.png'), ('depth_filled', '%06d-depth.png')):
            (base / sub).mkdir()
            for i in range(nf):
                (base / sub / (name % (i + 1))).write_bytes(b'')
    cfg = tmp_path / 'cfg'
    for c in (2, 3, 5):
        d = cfg / ('c%d' % c)
        (d / 'train').mkdir(parents=True)
        yaml.safe_dump({'resolution': 176, 'object_width': 200.0, 'boundingbox': 10, 'camera': dict(K_INFO)}, open(d / 'dataset_info.yml', 'w'))
        np.save(d / 'mean.npy', np.zeros(8)); np.save(d / 'std.npy', np.ones(8))
        (d / 'ckpt.pth.tar').write_bytes(b'')
        (d / 'mesh.ply').write_text('ply\n')
    tpl = {'train_data_path': str(cfg / 'c{class_id}' / 'train'), 'mean_std_path': str(cfg / 'c{class_id}'),
           'ckpt_dir': str(cfg / 'c{class_id}' / 'ckpt.pth.tar'), 'model_path': str(cfg / 'c{class_id}' / 'mesh.ply')}
    for kw in (dict(), dict(precision=['fp8', 'bf16'], iterations=[1, 2])):
        name = 'sweep' if kw else 'one'
        one = pr.getResultsYcbAll(str(ycb), [2, 3, 5], tpl, str(tmp_path / (name + '1')), **kw)
        seen['borrowed'].clear()
        three = pr.getResultsYcbAll(str(ycb), [2, 3, 5], tpl, str(tmp_path / (name + '3')), gpus=3, **kw)
        # frames tracked 3, 5, 2, 1: 0049 -> rank 0, 0048 -> rank 1, 0050 -> rank 2, 0051 -> rank 2
        # run here from rank 2 down: rank 2 borrows class 2 from 0048, rank 1 owns 0048, rank 0 borrows class 3 from 0048
        assert seen['borrowed'] == [{0: [0]}, {}, {0: [1]}]
        files = tree_files(str(tmp_path / (name + '1')))
        assert files == tree_files(str(tmp_path / (name + '3'))) and len(files) == (22 if not kw else 88)

        def same(a, b):
            if isinstance(a, dict):
                assert list(a) == list(b)
                for k in a:
                    same(a[k], b[k])
            else:
                assert np.array_equal(a, b)
        same(one, three)


def test_failing_ranks_raise_one_error_and_leave_no_process(pr):
    bad = [(['a.png'], ['a.png'], None, None)] * 3               # a weight-id tuple that is not one: each rank raises at once
    with pytest.raises(RuntimeError) as e:
        pr._track_on_ranks(2, [], 'bf16x3', 1, bad, ('bf16x3',), 1, 1, None, [None] * 3, pr.step_options())
    msg = str(e.value)
    assert msg.startswith(('rank 0 (cuda:0) failed:', 'rank 1 (cuda:1) failed:')) and 'TypeError' in msg and 'Traceback' in msg, msg
    assert multiprocessing.active_children() == []


def test_ranks_that_disagree_on_fp8_scales_are_an_error(pr):
    s = np.full(8, 2.0, np.float32)
    assert list(pr._agree_fp8_scales([{2: s, 5: None}, {2: s.copy(), 5: s * 2}])) == [2, 5]
    with pytest.raises(RuntimeError, match='ranks 0 and 1 calibrated weight set 2 differently'):
        pr._agree_fp8_scales([{2: s}, {2: s * 2}])
