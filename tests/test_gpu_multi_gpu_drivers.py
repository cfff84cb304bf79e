"""The one-pass drivers on two GPUs (predict.getResultsYcbAll / getResultsYcbInEOAT with gpus=2, one spawned process per rank)
against gpus=1 runs on the same small synthetic YCB-Video and YCBInEOAT trees.

  * every returned array equal and in the same key order, every pose file byte for byte: ycbv_all in bf16x3, a ycbv_all sweep of
    bf16x3, bf16, fp8 and fp32, a ycbineoat_all sweep with fp16 and fp8, an iteration sweep [1, 2]
  * each rank's fp8 scales of every weight set it tracked equal the single-GPU run's, including the sets whose first sequence
    belongs to the other rank
  * with video=True, every decoded frame of every mp4 equal
  * the CLI's --gpus 2 --score prints the score lines of --gpus 1
  * an unreadable depth PNG of a rank-1 video: one RuntimeError naming the file, and no process left behind

The sequences all have the same number of frames, so assign_ranks deals them out in order: YCB-Video 0048 and 0050 to rank 0,
0049 to rank 1 (classes 2 and 5 start in 0048 and recur in 0049; class 9 starts in 0049 and recurs in 0050); YCBInEOAT bleach0
and cracker_box_reorient to rank 0, bleach_hard_00_03 and sugar_box1 to rank 1 (the bleach bottle starts on rank 0).

Every case runs twice: on two GPUs (skipped with fewer), and as two ranks sharing cuda:0 (the same processes, split and pipes,
only the devices differ), so a one-GPU machine runs the multi-process path too.
"""
import contextlib, importlib, io, multiprocessing, os, shutil
import numpy as np
import pytest
import torch
import yaml

pytestmark = pytest.mark.gpu

PKG = 'iros20-6d-pose-tracking_b200'
NFRAMES = 4
CLASSES = (2, 5, 7, 9)
SEQS = {48: (2, 5, 7), 49: (2, 5, 9), 50: (7, 9)}
RANK_SEQS = ([48, 50], [49])
KEYFRAMES = ['0048/000001', '0048/000003', '0049/000002', '0050/000004']
VIDEOS = {'bleach0': 'bleach', 'bleach_hard_00_03': 'bleach', 'cracker_box_reorient': 'cracker', 'sugar_box1': 'sugar'}
RANK_VIDEOS = (['bleach0', 'cracker_box_reorient'], ['bleach_hard_00_03', 'sugar_box1'])
CAD = {'cracker': '003_cracker_box', 'sugar': '004_sugar_box', 'bleach': '021_bleach_cleanser'}
YCB_SWEEP = ['bf16x3', 'bf16', 'fp8', 'fp32']
EOAT_SWEEP = ['bf16x3', 'fp16', 'fp8']


@pytest.fixture(scope='module')
def pr():
    return importlib.import_module(PKG + '.predict')


def camera(synth):
    K = synth.CAMERA_K
    return {'focalX': float(K[0, 0]), 'focalY': float(K[1, 1]), 'centerX': float(K[0, 2]), 'centerY': float(K[1, 2]), 'height': 480, 'width': 640}


def write_config(d, synth, seed, width):
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
def ycbv(tmp_path_factory, synth):
    """-> (tmp, ycb dir, templates): sequences SEQS, 21 CADmodels folders with points, key frames."""
    import cv2
    tmp = tmp_path_factory.mktemp('multi_ycbv')
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
    return tmp, str(ycb), templates


@pytest.fixture(scope='module')
def eoat(tmp_path_factory, synth):
    """-> (tmp, data dir, templates): the videos VIDEOS of 3 objects, CADmodels folders with points."""
    import cv2
    tmp = tmp_path_factory.mktemp('multi_eoat')
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
    return tmp, str(tmp / 'data'), templates


@contextlib.contextmanager
def single_engine(pr):
    """-> [Engine]: the Engine of the gpus=1 run made in the block, kept to read its fp8 scales."""
    got, orig = [], pr._one_pass_trackers

    def make(*a, **kw):
        eng, trackers = orig(*a, **kw)
        got.append(eng)
        return eng, trackers
    with pytest.MonkeyPatch.context() as m:
        m.setattr(pr, '_one_pass_trackers', make)
        yield got


@pytest.fixture(scope='module', params=['two_gpus', 'two_ranks_on_cuda0'])
def multi(request, pr):
    """-> a context manager for the block that makes gpus=2 runs; it yields the list that collects each run's per-rank fp8 scales."""
    if request.param == 'two_gpus' and torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs')

    @contextlib.contextmanager
    def ranks():
        got, orig = [], pr._agree_fp8_scales
        with pytest.MonkeyPatch.context() as m:
            m.setattr(pr, '_agree_fp8_scales', lambda per_rank: got.append(per_rank) or orig(per_rank))
            if request.param == 'two_ranks_on_cuda0':
                m.setattr(torch.cuda, 'device_count', lambda: 2)
                m.setattr(pr, '_rank_devices', lambda n: [0] * n)
            yield got
    ranks.name = request.param
    return ranks


def ycbv_runs(pr, ycbv, out, **kw):
    tmp, ycb, templates = ycbv
    return pr.getResultsYcbAll(ycb, list(CLASSES), templates, str(tmp / out), **kw)


def eoat_runs(pr, eoat, out, **kw):
    tmp, data, templates = eoat
    return pr.getResultsYcbInEOAT(data, templates, str(tmp / out), **kw)


CASES = {'ycbv_bf16x3': (ycbv_runs, {}), 'ycbv_sweep': (ycbv_runs, dict(precision=YCB_SWEEP)),
         'ycbv_iterations': (ycbv_runs, dict(iterations=[1, 2])), 'eoat_sweep': (eoat_runs, dict(precision=EOAT_SWEEP)),
         'ycbv_video': (ycbv_runs, dict(video=True)), 'eoat_video': (eoat_runs, dict(video=True))}


@pytest.fixture(scope='module')
def single(pr, ycbv, eoat):
    """Every case at gpus=1 -> {case: (result, tree, fp8 scales {weight id: scales} of its Engine)}."""
    objects = importlib.import_module(PKG + '.eval_ycbineoat').OBJECTS
    out = {}
    for name, (run, kw) in CASES.items():
        tree = eoat if run is eoat_runs else ycbv
        with single_engine(pr) as engines:
            res = run(pr, tree, 'one_' + name, **kw)
            wids = CLASSES if tree is ycbv else sorted(set(objects.index(o) for o in VIDEOS.values()))
            scales = {w: engines[0].fp8_scales(w) for w in wids}
        out[name] = (res, str(tree[0] / ('one_' + name)), scales)
    return out


@pytest.fixture(scope='module')
def multi_runs(pr, ycbv, eoat, multi):
    """Every case at gpus=2 -> {case: (result, tree, [per-rank fp8 scales])}."""
    out = {}
    for name, (run, kw) in CASES.items():
        tree = eoat if run is eoat_runs else ycbv
        with multi() as scales:
            res = run(pr, tree, '%s_%s' % (multi.name, name), gpus=2, **kw)
        assert multiprocessing.active_children() == []
        out[name] = (res, str(tree[0] / ('%s_%s' % (multi.name, name))), scales[0])
    return out


def same_results(a, b, path=()):
    """Equal nested dicts, keys in the same order, arrays equal."""
    if isinstance(a, dict):
        assert isinstance(b, dict) and list(a) == list(b), (path, list(a), list(b))
        for k in a:
            same_results(a[k], b[k], path + (k,))
    else:
        assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b), (path, np.abs(a - b).max())


def video_frames(path):
    import cv2
    cap = cv2.VideoCapture(path)
    frames = []
    while True:
        ok, f = cap.read()
        if not ok:
            break
        frames.append(f)
    cap.release()
    return frames


def same_tree(a, b):
    """The same files; pose files byte for byte, videos frame for frame."""
    fa = sorted(os.path.relpath(os.path.join(d, f), a) for d, _, fs in os.walk(a) for f in fs)
    fb = sorted(os.path.relpath(os.path.join(d, f), b) for d, _, fs in os.walk(b) for f in fs)
    assert fa == fb and fa
    for f in fa:
        if f.endswith('.mp4'):
            x, y = video_frames(os.path.join(a, f)), video_frames(os.path.join(b, f))
            assert len(x) == len(y) > 0 and all(np.array_equal(p, q) for p, q in zip(x, y)), f
            continue
        with open(os.path.join(a, f), 'rb') as x, open(os.path.join(b, f), 'rb') as y:
            assert x.read() == y.read(), f
    return fa


@pytest.mark.parametrize('case', list(CASES))
def test_two_ranks_equal_one_gpu(single, multi_runs, case):
    res1, tree1, _ = single[case]
    res2, tree2, _ = multi_runs[case]
    same_results(res1, res2)
    files = same_tree(tree1, tree2)
    if case.endswith('video'):
        assert sum(f.endswith('.mp4') for f in files) == (sum(len(c) for c in SEQS.values()) if case.startswith('ycbv') else len(VIDEOS))


@pytest.mark.parametrize('case', ['ycbv_sweep', 'eoat_sweep'])
def test_each_ranks_fp8_scales_equal_one_gpu(pr, single, multi_runs, case):
    _, _, want = single[case]
    _, _, per_rank = multi_runs[case]
    assert len(per_rank) == 2
    ev = importlib.import_module(PKG + '.eval_ycbineoat')
    if case == 'ycbv_sweep':
        tracked = [sorted(set(c for s in seqs for c in SEQS[s])) for seqs in RANK_SEQS]
        assert tracked == [[2, 5, 7, 9], [2, 5, 9]]            # rank 1 borrows 2 and 5 from 0048, rank 0 borrows 9 from 0049
    else:
        tracked = [sorted(set(ev.OBJECTS.index(VIDEOS[v]) for v in vs)) for vs in RANK_VIDEOS]
    for r, scales in enumerate(per_rank):
        assert sorted(scales) == tracked[r]
        for w, s in scales.items():
            assert s is not None and want[w] is not None and np.array_equal(s, want[w]), (r, w, s, want[w])


def test_cli_gpus_2_prints_the_scores_of_gpus_1(pr, eoat, multi, capsys):
    tmp, data, templates = eoat
    base = ['--mode', 'ycbineoat_all', '--YCBInEOAT_dir', data, '--ycb_dir', str(tmp / 'ycb'), '--score'] + \
        sum([['--' + k, v] for k, v in templates.items()], [])
    printed = {}
    for gpus in (1, 2):
        out = str(tmp / ('cli_%s_%d' % (multi.name, gpus)))
        with multi():
            pr.main(base + ['--outdir', out, '--gpus', str(gpus)])
        lines = capsys.readouterr().out.splitlines()
        printed[gpus] = [l for l in lines if l != '-> %s' % out]
    assert printed[1] == printed[2] and any(l.startswith('Total pose') for l in printed[1])


def test_a_failing_rank_names_the_file_and_leaves_no_process(pr, eoat, multi):
    tmp, data, templates = eoat
    broken = tmp / ('broken_%s' % multi.name)
    shutil.copytree(data, str(broken))
    bad = broken / 'sugar_box1' / 'depth_filled' / ('%07d.png' % 2)          # sugar_box1 is rank 1's
    bad.write_bytes(b'not a png')
    with multi():
        with pytest.raises(RuntimeError) as e:
            pr.getResultsYcbInEOAT(str(broken), templates, str(tmp / ('broken_out_%s' % multi.name)), gpus=2)
    msg = str(e.value)
    assert msg.startswith('rank 1 ') and str(bad) in msg and 'Traceback' in msg, msg
    assert multiprocessing.active_children() == []
