"""Host logic of refinement rounds (se3tn_track_opts.iterations through Engine / Tracker / the one-pass drivers' iterations= and
predict --iterations): which counts are taken, what is refused before anything reaches a device, and where each variant's tree goes.
CPU only; the tracked poses are checked on the GPU (test_gpu_refine.py)."""
import importlib, os, re
import numpy as np
import pytest
from test_precision_sweep_cpu import pr, no_device, refusal_trees, tree_files, K_INFO      # noqa: F401

PKG = 'iros20-6d-pose-tracking_b200'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_limit_is_the_headers():
    L = importlib.import_module(PKG + '._lib')
    hdr = open(os.path.join(ROOT, 'include', 'se3tn.h')).read()
    assert int(re.search(r'SE3TN_MAX_REFINE_ITERATIONS\s+(\d+)', hdr).group(1)) == L.MAX_REFINE_ITERATIONS == 8


def test_engine_refine_iterations():
    E = importlib.import_module(PKG + '.engine').Engine
    assert [E.refine_iterations(k) for k in (1, 2, 8, np.int32(3))] == [1, 2, 8, 3]
    for bad in (0, 9, -1, 2.0, '2', None, True):
        with pytest.raises(ValueError, match='iterations'):
            E.refine_iterations(bad)


def test_refine_counts(pr):
    assert pr.refine_counts(1) == ((1,), False)
    assert pr.refine_counts(3) == ((3,), False)
    assert pr.refine_counts([1, 2, 3]) == ((1, 2, 3), True)
    assert pr.refine_counts((2,)) == ((2,), True)
    for bad, msg in (([], 'no iteration'), ([1, 1], 'listed more than once'), ([1, 9], 'iterations'), (0, 'iterations')):
        with pytest.raises(ValueError, match=msg):
            pr.refine_counts(bad)


def test_tree_paths(pr, tmp_path):
    out = str(tmp_path / 'o')
    assert pr.iterations_outdir(out, 2) == os.path.join(out, 'iter2')
    v = pr._sweep_variants(out, ('bf16x3',), False, (1,), False)
    assert v == [('bf16x3', 1, out)]                                # today's tree
    v = pr._sweep_variants(out, ('bf16x3',), False, (3,), False)
    assert v == [('bf16x3', 3, out)]
    v = pr._sweep_variants(out, ('fp8', 'fp32'), True, (1, 2), True)
    assert [r for *_, r in v] == [os.path.join(out, 'iter1', 'fp8'), os.path.join(out, 'iter1', 'fp32'),
                                  os.path.join(out, 'iter2', 'fp8'), os.path.join(out, 'iter2', 'fp32')]
    assert [(m, k) for m, k, _ in v] == [('fp8', 1), ('fp32', 1), ('fp8', 2), ('fp32', 2)]
    res = {(m, k): m + str(k) for m, k, _ in v}
    assert pr._sweep_results(res, v, True, True) == {1: {'fp8': 'fp81', 'fp32': 'fp321'}, 2: {'fp8': 'fp82', 'fp32': 'fp322'}}
    v = pr._sweep_variants(out, ('fp8',), False, (2, 1), True)
    assert pr._sweep_results({(m, k): k for m, k, _ in v}, v, False, True) == {2: 2, 1: 1}


def test_cli_parses_iterations(pr):
    assert pr.cli_iterations(None, 'ycbv') is None
    assert pr.cli_iterations('3', 'ycbv') == 3
    assert pr.cli_iterations('1,2,3', 'ycbineoat_all') == [1, 2, 3]
    assert pr.cli_iterations('2, 1', 'ycbv_all') == [2, 1]
    for text, mode in (('0', 'ycbv'), ('9', 'ycbv_all'), ('x', 'ycbv'), ('1,1', 'ycbv_all'), ('1,', 'ycbineoat_all'),
                       ('1,2', 'ycbv'), ('1,2', 'ycbineoat'), ('1,2', 'class')):
        with pytest.raises(SystemExit):
            pr.cli_iterations(text, mode)


def test_cli_passes_iterations(pr, tmp_path, monkeypatch):
    calls = []
    monkeypatch.setattr(pr, 'load_run_config', lambda *a: ({}, None, None))
    monkeypatch.setattr(pr, 'predictSequenceYcbInEOAT', lambda *a, **kw: calls.append(('eoat', kw)) or [])
    monkeypatch.setattr(pr, 'predictSequenceYcb', lambda *a, **kw: calls.append(('ycbv', kw)) or ([], None))
    monkeypatch.setattr(pr, 'getResultsYcb', lambda *a, **kw: calls.append(('class', kw)) or {})
    monkeypatch.setattr(pr, 'getResultsYcbInEOAT', lambda *a, **kw: calls.append(('eoat_all', kw)) or {})
    base = ['--train_data_path', 't', '--model_path', 'm', '--ckpt_dir', 'c', '--mean_std_path', 's', '--outdir', str(tmp_path / 'o'),
            '--ycb_dir', 'y', '--YCBInEOAT_dir', 'd', '--seq_id', '48']
    for mode in ('ycbineoat', 'ycbv', 'class'):
        pr.main(base + ['--mode', mode, '--iterations', '2'])
    pr.main(base + ['--mode', 'ycbineoat_all', '--iterations', '1,3', '--precision', 'fp8,bf16'])
    pr.main(base + ['--mode', 'ycbineoat_all', '--iterations', '1'])
    pr.main(base + ['--mode', 'ycbineoat_all'])
    assert [kw.get('iterations', '-') for _, kw in calls] == [2, 2, 2, [1, 3], 1, '-']
    assert calls[3][1]['precision'] == ['fp8', 'bf16']


@pytest.mark.parametrize('iterations', [[], [1, 1], [0, 1], 9, [2, 9]])
def test_driver_refusals(pr, tmp_path, no_device, iterations):
    ycb, ycb_tpl, data, obj_tpl = refusal_trees(tmp_path)
    with pytest.raises(ValueError, match='iteration'):
        pr.getResultsYcbAll(ycb, [2], ycb_tpl, str(tmp_path / 'out'), iterations=iterations)
    with pytest.raises(ValueError, match='iteration'):
        pr.getResultsYcbInEOAT(data, obj_tpl, str(tmp_path / 'out'), iterations=iterations)
    assert not (tmp_path / 'out').exists()


def test_video_with_two_counts_is_refused(pr, tmp_path, no_device):
    ycb, ycb_tpl, data, obj_tpl = refusal_trees(tmp_path)
    with pytest.raises(ValueError, match='video'):
        pr.getResultsYcbAll(ycb, [2], ycb_tpl, str(tmp_path / 'out'), iterations=[1, 2], video=True)
    with pytest.raises(ValueError, match='video'):
        pr.getResultsYcbInEOAT(data, obj_tpl, str(tmp_path / 'out'), iterations=[1, 2], video=True)
    assert not (tmp_path / 'out').exists()


def fake_loop(pr, monkeypatch, seen):
    """The drivers without a device: poses that depend on the variant (mode and count) and the sequence only."""
    monkeypatch.setattr(pr, '_one_pass_trackers', lambda entries, precision, max_batch: (None, {}))

    def loop(eng, trackers, sequences, variants, depth, workers, video, opts, seq_index):
        seen.append(variants)
        for j, (rgb_files, _, ids, init) in enumerate(sequences):
            out = {}
            for m, k in variants:
                out[m, k] = np.stack([init + 0.001 * (t + 1) * (pr.PRECISIONS.index(m) + 1) + 0.1 * k + j for t in range(len(rgb_files))])
            yield out, None
    monkeypatch.setattr(pr, '_track_sequences', loop)


def test_layout_of_counts_and_modes(pr, tmp_path, monkeypatch):
    import yaml
    seen = []
    fake_loop(pr, monkeypatch, seen)
    data = tmp_path / 'data'
    for v, nf in (('bleach0', 3), ('sugar_box1', 2)):
        for sub in ('rgb', 'depth_filled', 'annotated_poses'):
            (data / v / sub).mkdir(parents=True)
        for i in range(nf):
            np.savetxt(str(data / v / 'annotated_poses' / ('%07d.txt' % i)), np.eye(4) * (i + 1))
            (data / v / 'rgb' / ('%07d.png' % i)).write_bytes(b'')
            (data / v / 'depth_filled' / ('%07d.png' % i)).write_bytes(b'')
    cfg = tmp_path / 'cfg'
    for o in ('bleach', 'sugar'):
        (cfg / o / 'train').mkdir(parents=True)
        yaml.safe_dump({'resolution': 176, 'object_width': 200.0, 'boundingbox': 10, 'camera': dict(K_INFO)}, open(cfg / o / 'dataset_info.yml', 'w'))
        np.save(cfg / o / 'mean.npy', np.zeros(8)); np.save(cfg / o / 'std.npy', np.ones(8))
        (cfg / o / 'ckpt.pth.tar').write_bytes(b'')
        (cfg / o / 'mesh.ply').write_text('ply\n')
    tpl = {'train_data_path': str(cfg / '{object}' / 'train'), 'mean_std_path': str(cfg / '{object}'),
           'ckpt_dir': str(cfg / '{object}' / 'ckpt.pth.tar'), 'model_path': str(cfg / '{object}' / 'mesh.ply')}
    run = lambda out, **kw: pr.getResultsYcbInEOAT(str(data), tpl, str(tmp_path / out), **kw)
    both = run('both', precision=['fp8', 'bf16x3'], iterations=[1, 2])
    assert seen[-1] == (('fp8', 1), ('bf16x3', 1), ('fp8', 2), ('bf16x3', 2))
    assert list(both) == [1, 2] and all(list(both[k]) == ['fp8', 'bf16x3'] for k in both)
    assert sorted(os.listdir(tmp_path / 'both')) == ['iter1', 'iter2']
    assert all(sorted(os.listdir(tmp_path / 'both' / k)) == ['bf16x3', 'fp8'] for k in ('iter1', 'iter2'))
    for k in (1, 2):
        for m in ('fp8', 'bf16x3'):
            one = run('%s%d' % (m, k), precision=m, iterations=k)
            assert seen[-1] == ((m, k),)
            assert all(np.array_equal(one[v], both[k][m][v]) for v in one)
            files = tree_files(str(tmp_path / ('%s%d' % (m, k))))
            assert files == tree_files(str(tmp_path / 'both' / ('iter%d' % k) / m)) and len(files) == 5
    counts = run('counts', precision='fp8', iterations=[2, 1])
    assert list(counts) == [2, 1] and sorted(os.listdir(tmp_path / 'counts')) == ['iter1', 'iter2']
    assert tree_files(str(tmp_path / 'counts' / 'iter1')) == tree_files(str(tmp_path / 'fp81'))
    run('default', precision='fp8')
    assert seen[-1] == (('fp8', 1),) and tree_files(str(tmp_path / 'default')) == tree_files(str(tmp_path / 'fp81'))
