"""Precision sweeps of the one-pass drivers (predict.getResultsYcbInEOAT / getResultsYcbAll with a list of modes or 'all') on small
synthetic data sets in the YCBInEOAT and YCB-Video layouts, against single-mode runs of each mode on the same trees.

  * every mode's returned poses and pose files bit for bit a single-mode run of that mode (YCBInEOAT: all six modes; YCB-Video:
    bf16x3, bf16, fp8, fp32), and every weight set's fp8 scales those of a single-mode fp8 run
  * each frame decoded once per sweep, exactly one step per mode and frame, and in every captured mode a CUDA graph replay on
    every step after a track set's first
  * predict.score_precisions: the reference mode's drift row is 0, every other row a numpy restatement of ADD / ADD-S between
    the two modes' poses (oracle/se3_oracle.py), and the AUCs those the scorers give each mode's tree
  * the CLI's --precision all --score: one tree per mode, the per-mode score headers and the table
"""
import argparse, contextlib, importlib, io, os, shutil, threading
import numpy as np
import pytest
import torch
import yaml
import se3_oracle as O

pytestmark = pytest.mark.gpu

PKG = 'iros20-6d-pose-tracking_b200'
NFRAMES = 4
VIDEOS = {'bleach0': 'bleach', 'sugar_box1': 'sugar', 'bleach_hard_00_03': 'bleach', 'cracker_box_reorient': 'cracker'}
CAD = {'cracker': '003_cracker_box', 'sugar': '004_sugar_box', 'bleach': '021_bleach_cleanser'}
CLASSES = (2, 5, 7)
SEQS = {48: (2, 5, 7), 49: (2, 5)}
KEYFRAMES = ['0048/000001', '0048/000003', '0049/000002', '0049/000004']
YCB_MODES = ('bf16x3', 'bf16', 'fp8', 'fp32')


@pytest.fixture(scope='module')
def pr():
    return importlib.import_module(PKG + '.predict')


def camera(synth):
    K = synth.CAMERA_K
    return {'focalX': float(K[0, 0]), 'focalY': float(K[1, 1]), 'centerX': float(K[0, 2]), 'centerY': float(K[1, 2]), 'height': 480, 'width': 640}


def write_config(d, synth, seed, width):
    """dataset_info.yml, mean / std, checkpoint and mesh of one class or object under d."""
    mio = importlib.import_module(PKG + '.mesh_io')
    (d / 'train').mkdir(parents=True)
    yaml.safe_dump({'resolution': 176, 'object_width': width, 'boundingbox': 10, 'camera': camera(synth)}, open(d / 'dataset_info.yml', 'w'))
    mean, std = synth.default_mean_std()
    np.save(d / 'mean.npy', mean + seed); np.save(d / 'std.npy', std * (1 + 0.05 * seed))
    torch.save({'epoch': 1, 'state_dict': synth.make_state_dict(seed), 'best_prec': 0.0}, str(d / 'model_best_val.pth.tar'))
    mio.save_ply_mesh(str(d / 'textured.ply'), synth.mesh(3, seed=seed))


def gliding(synth, seed):
    p = synth.raw_poses(NFRAMES, seed=seed)
    p[1:, :3, 3] = p[0, :3, 3] + 0.002 * np.arange(1, NFRAMES)[:, None]
    p[1:, :3, :3] = p[0, :3, :3]
    return p


@pytest.fixture(scope='module')
def eoat(tmp_path_factory, synth):
    """A YCBInEOAT tree: 4 videos (two of the bleach bottle) of 3 objects -> (tmp, templates)."""
    import cv2
    tmp = tmp_path_factory.mktemp('sweep_eoat')
    for j, obj in enumerate(CAD):
        write_config(tmp / 'cfg' / obj, synth, j + 1, 180.0 + 20 * j)
        (tmp / 'ycb' / 'CADmodels' / CAD[obj]).mkdir(parents=True)
        np.savetxt(str(tmp / 'ycb' / 'CADmodels' / CAD[obj] / 'points.xyz'), synth.mesh(3, seed=j + 1)['pos'].astype(np.float64))
    for v_i, v in enumerate(VIDEOS):
        base = tmp / 'data' / v
        for sub in ('rgb', 'depth_filled', 'annotated_poses'):
            (base / sub).mkdir(parents=True)
        p = gliding(synth, 10 + v_i)
        for i in range(NFRAMES):
            rgb, depth = synth.raw_frame(seed=100 * v_i + i)
            cv2.imwrite(str(base / 'rgb' / ('%07d.png' % i)), rgb[..., ::-1])
            cv2.imwrite(str(base / 'depth_filled' / ('%07d.png' % i)), depth)
            np.savetxt(str(base / 'annotated_poses' / ('%07d.txt' % i)), p[i])
    templates = {'train_data_path': str(tmp / 'cfg' / '{object}' / 'train'), 'mean_std_path': str(tmp / 'cfg' / '{object}'),
                 'ckpt_dir': str(tmp / 'cfg' / '{object}' / 'model_best_val.pth.tar'), 'model_path': str(tmp / 'cfg' / '{object}' / 'textured.ply')}
    return tmp, templates


@pytest.fixture(scope='module')
def ycbv(tmp_path_factory, synth):
    """A YCB-Video tree: sequences 0048 (classes 2, 5, 7) and 0049 (2, 5), 21 CADmodels folders with points, key frames ->
    (tmp, templates)."""
    import cv2
    tmp = tmp_path_factory.mktemp('sweep_ycbv')
    ycb = tmp / 'ycb'
    for c in CLASSES:
        write_config(tmp / 'cfg' / ('c%d' % c), synth, c, 150.0 + 10 * c)
    for k in range(1, 22):
        (ycb / 'CADmodels' / ('%03d_obj' % k)).mkdir(parents=True)
        np.savetxt(str(ycb / 'CADmodels' / ('%03d_obj' % k) / 'points.xyz'),
                   synth.mesh(3, seed=k if k in CLASSES else 2)['pos'].astype(np.float64))
    for seq, cls in SEQS.items():
        base = ycb / 'data_organized' / ('%04d' % seq)
        for d in ['color', 'depth_filled'] + ['pose_gt/%d' % c for c in cls]:
            (base / d).mkdir(parents=True)
        for i in range(NFRAMES):
            rgb, depth = synth.raw_frame(seed=100 * seq + i)
            cv2.imwrite(str(base / 'color' / ('%06d-color.png' % (i + 1))), rgb[..., ::-1])
            cv2.imwrite(str(base / 'depth_filled' / ('%06d-depth.png' % (i + 1))), depth)
        for c in cls:
            p = gliding(synth, 10 * seq + c)
            for i in range(NFRAMES):
                np.savetxt(str(base / 'pose_gt' / str(c) / ('%06d.txt' % (i + 1))), p[i])
    (ycb / 'YCB_Video_toolbox').mkdir()
    (ycb / 'YCB_Video_toolbox' / 'keyframe.txt').write_text('\n'.join(KEYFRAMES) + '\n')
    templates = {'train_data_path': str(tmp / 'cfg' / 'c{class_id}' / 'train'), 'mean_std_path': str(tmp / 'cfg' / 'c{class_id}'),
                 'ckpt_dir': str(tmp / 'cfg' / 'c{class_id}' / 'model_best_val.pth.tar'),
                 'model_path': str(tmp / 'cfg' / 'c{class_id}' / 'textured.ply')}
    return tmp, templates


@contextlib.contextmanager
def recording(pr):
    """-> (steps, decodes): every Engine.track_render call as (engine, precision, first weight id, n, last_step_was_graph), and
    the number of read_rgb / read_depth calls, while the block runs."""
    E = pr.Engine
    orig, rgb, depth = E.track_render, pr.read_rgb, pr.read_depth
    steps, decodes, lock = [], {'rgb': 0, 'depth': 0}, threading.Lock()

    def track_render(self, *a, **kw):
        out = orig(self, *a, **kw)
        wh = kw.get('weight_ids_host')
        steps.append((self, kw.get('precision', 'bf16x3'), None if wh is None else int(wh[0]), int(a[3].shape[0]), self.last_step_was_graph()))
        return out

    def count(name, fn):
        def read(path):
            with lock:                                                # the decode jobs run on a thread pool
                decodes[name] += 1
            return fn(path)
        return read
    E.track_render, pr.read_rgb, pr.read_depth = track_render, count('rgb', rgb), count('depth', depth)
    try:
        yield steps, decodes
    finally:
        E.track_render, pr.read_rgb, pr.read_depth = orig, rgb, depth


def fp8_scales(steps, wids):
    eng = steps[-1][0]
    return {w: eng.fp8_scales(w) for w in wids}


@pytest.fixture(scope='module')
def eoat_runs(pr, eoat):
    tmp, templates = eoat
    data = str(tmp / 'data')
    wids = sorted(set(importlib.import_module(PKG + '.eval_ycbineoat').OBJECTS.index(o) for o in VIDEOS.values()))
    runs = {}
    with recording(pr) as (steps, decodes):
        runs['sweep'] = pr.getResultsYcbInEOAT(data, templates, str(tmp / 'sweep'), precision='all')
        runs['sweep_steps'], runs['sweep_decodes'] = list(steps), dict(decodes)
        runs['sweep_scales'] = fp8_scales(steps, wids)
    for m in pr.PRECISIONS:
        with recording(pr) as (steps, _):
            runs[m] = pr.getResultsYcbInEOAT(data, templates, str(tmp / 'single' / m), precision=m)
        if m == 'fp8':
            runs['fp8_scales'] = fp8_scales(steps, wids)
    return runs


@pytest.fixture(scope='module')
def ycbv_runs(pr, ycbv):
    tmp, templates = ycbv
    ycb = str(tmp / 'ycb')
    runs = {}
    with recording(pr) as (steps, decodes):
        runs['sweep'] = pr.getResultsYcbAll(ycb, list(CLASSES), templates, str(tmp / 'sweep'), precision=list(YCB_MODES))
        runs['sweep_steps'], runs['sweep_decodes'] = list(steps), dict(decodes)
        runs['sweep_scales'] = fp8_scales(steps, CLASSES)
    for m in YCB_MODES:
        with recording(pr) as (steps, _):
            runs[m] = pr.getResultsYcbAll(ycb, list(CLASSES), templates, str(tmp / 'single' / m), precision=m)
        if m == 'fp8':
            runs['fp8_scales'] = fp8_scales(steps, CLASSES)
    return runs


def same_tree(a, b):
    """Both trees hold the same files, and every pose file the same float64 values."""
    fa = sorted(os.path.relpath(os.path.join(d, f), a) for d, _, fs in os.walk(a) for f in fs)
    fb = sorted(os.path.relpath(os.path.join(d, f), b) for d, _, fs in os.walk(b) for f in fs)
    assert fa == fb and fa
    for f in fa:
        assert np.array_equal(np.loadtxt(os.path.join(a, f)), np.loadtxt(os.path.join(b, f))), f
        with open(os.path.join(a, f), 'rb') as x, open(os.path.join(b, f), 'rb') as y:
            assert x.read() == y.read(), f


def test_ycbineoat_sweep_bit_identical_to_single_mode_runs(pr, eoat, eoat_runs):
    tmp, _ = eoat
    sweep = eoat_runs['sweep']
    assert list(sweep) == list(pr.PRECISIONS) and sorted(os.listdir(tmp / 'sweep')) == sorted(pr.PRECISIONS)
    for m in pr.PRECISIONS:
        assert sorted(sweep[m]) == sorted(eoat_runs[m]) == sorted(VIDEOS)
        for v in VIDEOS:
            assert np.array_equal(sweep[m][v], eoat_runs[m][v]), (m, v, np.abs(sweep[m][v] - eoat_runs[m][v]).max())
        same_tree(str(tmp / 'sweep' / m), str(tmp / 'single' / m))
    assert not np.array_equal(sweep['fp8']['bleach0'], sweep['fp32']['bleach0'])        # the modes really differ


def test_ycbv_sweep_bit_identical_to_single_mode_runs(pr, ycbv, ycbv_runs):
    tmp, _ = ycbv
    sweep = ycbv_runs['sweep']
    assert list(sweep) == list(YCB_MODES) and sorted(os.listdir(tmp / 'sweep')) == sorted(YCB_MODES)
    for m in YCB_MODES:
        assert sorted(sweep[m]) == list(CLASSES)
        for c in CLASSES:
            assert sorted(sweep[m][c]) == sorted(ycbv_runs[m][c])
            for seq in sweep[m][c]:
                assert np.array_equal(sweep[m][c][seq], ycbv_runs[m][c][seq]), (m, c, seq)
        same_tree(str(tmp / 'sweep' / m), str(tmp / 'single' / m))


@pytest.mark.parametrize('driver', ['eoat', 'ycbv'])
def test_sweep_fp8_scales_equal_a_single_fp8_run(eoat_runs, ycbv_runs, driver):
    runs = eoat_runs if driver == 'eoat' else ycbv_runs
    assert runs['sweep_scales'].keys() == runs['fp8_scales'].keys()
    for w, s in runs['sweep_scales'].items():
        assert s is not None and np.array_equal(s, runs['fp8_scales'][w]), w


@pytest.mark.parametrize('driver', ['eoat', 'ycbv'])
def test_sweep_decodes_each_frame_once_and_steps_once_per_mode(pr, eoat_runs, ycbv_runs, driver):
    runs, modes = (eoat_runs, pr.PRECISIONS) if driver == 'eoat' else (ycbv_runs, YCB_MODES)
    frames = NFRAMES * len(VIDEOS) if driver == 'eoat' else (NFRAMES - 1) * len(SEQS)        # YCB-Video tracks from frame 1
    assert runs['sweep_decodes'] == {'rgb': frames, 'depth': frames}
    rec = runs['sweep_steps']
    assert len(rec) == len(modes) * frames
    assert [r[1] for r in rec] == list(modes) * frames                                    # M steps per frame, the modes in order
    seen = set()
    for _, m, wid, n, graph in rec:
        key = (m, wid, n)
        if m != 'fp32' and key in seen:
            assert graph, (m, wid, n)
        if m == 'fp32':
            assert not graph
        seen.add(key)


def cloud(pr, path):
    return np.asarray(pr.object_cloud(path).points, dtype=np.float64)


@pytest.mark.parametrize('driver', ['eoat', 'ycbv'])
def test_scores_and_drift_against_numpy(pr, eoat, ycbv, eoat_runs, ycbv_runs, driver):
    ev = importlib.import_module(PKG + '.eval_ycbineoat')
    ey = importlib.import_module(PKG + '.eval_ycb')
    if driver == 'eoat':
        tmp, templates = eoat
        sweep = eoat_runs['sweep']
        kw = dict(YCBInEOAT_dir=str(tmp / 'data'))
        tracks = {v: (sweep, lambda r, v=v: r[v], templates['model_path'].format(object=o)) for v, o in VIDEOS.items()}
    else:
        tmp, templates = ycbv
        sweep = ycbv_runs['sweep']
        kw = {}
        tracks = {(c, s): (sweep, lambda r, c=c, s=s: r[c][s], templates['model_path'].format(class_id=c)) for s, cls in SEQS.items() for c in cls}
    ycb = str(tmp / 'ycb')
    with contextlib.redirect_stdout(io.StringIO()) as buf:
        ref, rows = pr.score_precisions(sweep, str(tmp / 'sweep'), ycb, templates, **kw)
    printed = buf.getvalue().splitlines()
    assert ref == 'fp32' and list(rows) == list(sweep)
    assert [l for l in printed if l.startswith('precision ')] == ['precision %s' % m for m in sweep]
    assert rows[ref]['add_max'] == rows[ref]['add_mean'] == rows[ref]['adds_max'] == rows[ref]['adds_mean'] == 0.0
    points = {p: cloud(pr, p) for p in set(t[2] for t in tracks.values())}
    for m in sweep:
        add, adds = [], []
        for _, get, path in tracks.values():
            for a, b in zip(get(sweep[m]), get(sweep[ref])):
                add.append(O.add(a, b, points[path]) * 1000)
                adds.append(O.adi(a, b, points[path]) * 1000)
        want = dict(add_max=max(add), add_mean=np.mean(add), adds_max=max(adds), adds_mean=np.mean(adds))
        for k, w in want.items():
            assert abs(rows[m][k] - w) <= 1e-9 * max(1.0, abs(w)), (m, k, rows[m][k], w)
        if m != ref:
            assert rows[m]['adds_max'] > 0, m
        with contextlib.redirect_stdout(io.StringIO()):
            if driver == 'eoat':
                _, adi_auc, add_auc, _ = ev.eval_all(argparse.Namespace(res_dir=str(tmp / 'sweep' / m) + '/', YCBInEOAT_dir=str(tmp / 'data'),
                                                                        ycb_dir=ycb))
            else:
                names = pr.ycb_class_names(ycb)
                errs = [ey.eval_one_class(argparse.Namespace(ycb_dir=ycb, class_id=c, res_dir=pr.ycb_all_res_dir(str(tmp / 'sweep' / m), names[c - 1]) + '/'))
                        for c in CLASSES]
                adi_auc = ey.VOCap(np.concatenate([e[0] for e in errs])) * 100
                add_auc = ey.VOCap(np.concatenate([e[1] for e in errs])) * 100
        assert rows[m]['add'] == add_auc and rows[m]['adds'] == adi_auc, m


def test_cli_precision_all_writes_a_tree_per_mode_and_prints_the_table(pr, eoat, capsys):
    tmp, templates = eoat
    out = tmp / 'cli'
    res = pr.main(['--mode', 'ycbineoat_all', '--YCBInEOAT_dir', str(tmp / 'data'), '--ycb_dir', str(tmp / 'ycb'), '--outdir', str(out),
                   '--precision', 'all', '--score'] + sum([['--' + k, v] for k, v in templates.items()], []))
    printed = capsys.readouterr().out.splitlines()
    assert list(res) == list(pr.PRECISIONS) and sorted(os.listdir(out)) == sorted(pr.PRECISIONS)
    for m in pr.PRECISIONS:
        assert sorted(os.listdir(out / m)) == sorted(VIDEOS)
        for v in VIDEOS:
            assert sorted(os.listdir(out / m / v)) == ['%07d.txt' % i for i in range(NFRAMES)]
    heads = [i for i, l in enumerate(printed) if l.startswith('precision ')]
    assert [printed[i] for i in heads][:len(pr.PRECISIONS)] == ['precision %s' % m for m in pr.PRECISIONS]
    for i in heads[:len(pr.PRECISIONS)]:                                # each header is followed by eval_ycbineoat's lines
        assert printed[i + 1] in VIDEOS
    title = heads[len(pr.PRECISIONS)]
    assert printed[title].startswith('precision sweep:') and 'fp32' in printed[title]
    table = printed[title + 2:title + 2 + len(pr.PRECISIONS)]
    assert [l.split()[0] for l in table] == list(pr.PRECISIONS)
    assert [float(x) for x in table[pr.PRECISIONS.index('fp32')].split()[3:]] == [0.0] * 4
    shutil.rmtree(out)
