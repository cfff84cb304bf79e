"""The YCBInEOAT evaluation in one pass on the device: ADD / ADD-S over many model point sets (se3tn_add_adi_sets), VOCap of
many error sets at once (se3tn_vocap_sets), the eval_ycbineoat drop-in against its CPU restatement (oracle/ycbineoat_oracle.py),
and predict.getResultsYcbInEOAT on a synthetic data set in the YCBInEOAT layout: four videos (two of the bleach bottle) of three
objects with their own weights, statistics, meshes and widths, five frames each.

  * add_adi_sets bit for bit what one add_adi call per model computes, and within 1e-12 of the cKDTree oracle
  * vocap_sets bit for bit what one vocap call per set (and one on all errors) computes; its scratch only grows
  * the drop-in's printed lines and AUCs against the CPU restatement
  * the driver's poses bit for bit a frame-by-frame Tracker.on_track_batch loop (bf16x3, bf16), the same for every decode-ahead
    depth, within test_headless_sequence_driver's tolerance of per-video predictSequenceYcbInEOAT runs, and a CUDA graph replay
    on every step after each object's first
"""
import argparse, importlib, io, os, contextlib
import numpy as np
import pytest
import torch
import yaml
import se3_oracle as O
import ycbineoat_oracle as YO

pytestmark = pytest.mark.gpu

PKG = 'iros20-6d-pose-tracking_b200'
VIDEOS = {'bleach0': 'bleach', 'bleach_hard_00_03': 'bleach', 'sugar_box1': 'sugar', 'cracker_box_reorient': 'cracker'}
CAD = {'cracker': '003_cracker_box', 'sugar': '004_sugar_box', 'bleach': '021_bleach_cleanser'}
WIDTHS = {'cracker': 180.0, 'sugar': 200.0, 'bleach': 230.0}
NFRAMES = 5
POSE_ATOL = 1e-4                    # test_gpu_parity.py: the bf16x3 gate on the network's 6-vector, carried to a pose entry


@pytest.fixture(scope='module')
def eng(pkg):
    e = pkg.Engine(max_batch=1)
    yield e
    e.close()


def t64(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(dev)


def pose_pairs(n, seed):
    rng = np.random.default_rng(seed)
    from scipy.spatial.transform import Rotation
    pred = np.tile(np.eye(4), (n, 1, 1)); gt = pred.copy()
    if n == 0:
        return pred, gt
    gt[:, :3, :3] = Rotation.random(n, random_state=seed).as_matrix()
    gt[:, :3, 3] = rng.normal(0, 0.2, (n, 3)) + [0, 0, 1]
    pred[:, :3, :3] = Rotation.from_rotvec(rng.normal(0, 0.1, (n, 3))).as_matrix() @ gt[:, :3, :3]
    pred[:, :3, 3] = gt[:, :3, 3] + rng.normal(0, 0.02, (n, 3))
    return pred, gt


SET_SIZES = (1, 255, 256, 257, 511, 513, 2620)


@pytest.mark.parametrize('n', [0, 1, 3001])
def test_add_adi_sets_bit_identical_to_per_model_calls(eng, n):
    dev = eng.device
    rng = np.random.default_rng(n)
    models = [rng.normal(0, 0.05, (m, 3)) for m in SET_SIZES]
    pose_set = (np.arange(n) * 5 + n) % len(SET_SIZES)                    # interleaved set order
    pred, gt = pose_pairs(n, seed=n)
    add, adi = eng.add_adi_sets(models, pose_set.astype(np.int32), t64(pred.reshape(-1, 4, 4), dev), t64(gt.reshape(-1, 4, 4), dev))
    add, adi = add.cpu().numpy(), adi.cpu().numpy()
    assert add.shape == adi.shape == (n,)
    for s, m in enumerate(models):
        idx = np.nonzero(pose_set == s)[0]
        if len(idx) == 0:
            continue
        a1, b1 = eng.add_adi(t64(m, dev), t64(pred[idx], dev), t64(gt[idx], dev))
        assert np.array_equal(add[idx], a1.cpu().numpy()) and np.array_equal(adi[idx], b1.cpu().numpy()), 'set %d' % s
    for i in range(0, n, max(1, n // 60)):                                # the cKDTree oracle on a sample of the poses
        m = models[pose_set[i]]
        assert abs(add[i] - O.add(pred[i], gt[i], m)) <= 1e-12 * abs(O.add(pred[i], gt[i], m))
        assert abs(adi[i] - O.adi(pred[i], gt[i], m)) <= 1e-12 * abs(O.adi(pred[i], gt[i], m))


def test_add_adi_sets_refuses_invalid_offsets_and_ids(eng):
    L = importlib.import_module(PKG + '._lib')
    dev = eng.device
    table = t64(np.zeros((10, 3)), dev)
    pred, gt = (t64(p, dev) for p in pose_pairs(2, seed=1))
    for offs, ids in (([1, 4, 10], [0, 1]), ([0, 4, 9], [0, 1]), ([0, 4, 4, 10], [0, 2]), ([0, 6, 4, 10], [0, 2]),
                      ([0, 4, 10], [0, 2]), ([0, 4, 10], [-1, 0]), ([0], [0, 0])):
        with pytest.raises(ValueError if len(offs) < 2 else L.Se3tnError) as e:
            eng.add_adi_sets(table, np.array(ids, np.int32), pred, gt, set_offsets=offs)
        if len(offs) >= 2:
            assert e.value.code == L.ERR_INVALID, (offs, ids)


def test_vocap_sets_bit_identical_to_per_set_calls(eng):
    dev = eng.device
    rng = np.random.default_rng(5)
    n_sets = 6
    sizes = {0: 700, 1: 1, 2: 0, 3: 2500, 4: 300, 5: 40}                  # set 2 is empty; set 4 has nothing below 0.1 m
    errs = np.concatenate([rng.uniform(0.1, 0.3, sz) if s == 4 else np.abs(rng.normal(0, 0.06, sz)) for s, sz in sizes.items()])
    ids = np.concatenate([np.full(sz, s, np.int32) for s, sz in sizes.items()])
    perm = rng.permutation(len(errs))
    errs, ids = errs[perm], ids[perm]
    errs[:20] = np.round(errs[:20], 2)                                    # ties
    ap = eng.vocap_sets(t64(errs, dev), torch.from_numpy(ids).to(dev), n_sets)
    assert ap.shape == (n_sets + 1,)
    for s in range(n_sets):
        assert ap[s] == eng.vocap(t64(errs[ids == s], dev)), s
    assert ap[2] == 0.0 and ap[4] == 0.0 and ap[n_sets] == eng.vocap(t64(errs, dev))
    assert abs(ap[n_sets] - O.vocap(errs)) < 1e-12 and abs(ap[0] - O.vocap(errs[ids == 0])) < 1e-12

    # context scratch grows only when a call needs more, and repeated calls allocate nothing
    sizes_seen = []
    for n in (10, 100, 1000, 5000, 100, 5000, 2000):
        e = np.abs(rng.normal(0, 0.05, n))
        s = rng.integers(0, n_sets, n).astype(np.int32)
        got = eng.vocap_sets(t64(e, dev), torch.from_numpy(s).to(dev), n_sets)
        assert got[n_sets] == eng.vocap(t64(e, dev))
        sizes_seen.append(eng.metrics_scratch_bytes())
    assert all(b >= a for a, b in zip(sizes_seen, sizes_seen[1:])) and sizes_seen[3:] == [sizes_seen[3]] * 4, sizes_seen

    L = importlib.import_module(PKG + '._lib')
    with pytest.raises(L.Se3tnError) as e:
        eng.vocap_sets(t64([0.01, 0.02], dev), torch.tensor([0, n_sets], dtype=torch.int32, device=dev), n_sets)
    assert e.value.code == L.ERR_INVALID
    assert list(eng.vocap_sets(t64([], dev), torch.zeros(0, dtype=torch.int32, device=dev), 3)) == [0.0] * 4


# ---------------------------------------------------------------------------------------------------------- a YCBInEOAT tree
@pytest.fixture(scope='module')
def tree(tmp_path_factory, synth):
    """<tmp>/data/<video>/{rgb,depth_filled,annotated_poses}, <tmp>/ycb/CADmodels/<folder>/points.xyz, <tmp>/cfg/<object>/... ->
    (tmp, templates, gt poses {video: (NFRAMES,4,4)})."""
    import cv2
    mio = importlib.import_module(PKG + '.mesh_io')
    tmp = tmp_path_factory.mktemp('ycbineoat_all')
    K = synth.CAMERA_K
    cam = {'focalX': float(K[0, 0]), 'focalY': float(K[1, 1]), 'centerX': float(K[0, 2]), 'centerY': float(K[1, 2]), 'height': 480, 'width': 640}
    mean, std = synth.default_mean_std()
    for j, obj in enumerate(CAD):
        d = tmp / 'cfg' / obj
        (d / 'train').mkdir(parents=True)
        yaml.safe_dump({'resolution': 176, 'object_width': WIDTHS[obj], 'boundingbox': 10, 'camera': cam}, open(d / 'dataset_info.yml', 'w'))
        np.save(d / 'mean.npy', mean + j); np.save(d / 'std.npy', std * (1 + 0.05 * j))
        torch.save({'epoch': 1, 'state_dict': synth.make_state_dict(j + 1), 'best_prec': 0.0}, str(d / 'model_best_val.pth.tar'))
        mio.save_ply_mesh(str(d / 'textured.ply'), synth.mesh(3, seed=j + 1))
        (tmp / 'ycb' / 'CADmodels' / CAD[obj]).mkdir(parents=True)
        np.savetxt(str(tmp / 'ycb' / 'CADmodels' / CAD[obj] / 'points.xyz'), synth.mesh(3, seed=j + 1)['pos'].astype(np.float64))
    gt = {}
    for v_i, v in enumerate(VIDEOS):
        base = tmp / 'data' / v
        for sub in ('rgb', 'depth_filled', 'annotated_poses'):
            (base / sub).mkdir(parents=True)
        p = synth.raw_poses(NFRAMES, seed=10 + v_i)
        p[1:, :3, 3] = p[0, :3, 3] + 0.002 * np.arange(1, NFRAMES)[:, None]
        p[1:, :3, :3] = p[0, :3, :3]
        gt[v] = p
        for i in range(NFRAMES):
            rgb, depth = synth.raw_frame(seed=100 * v_i + i)
            cv2.imwrite(str(base / 'rgb' / ('%07d.png' % i)), rgb[..., ::-1])
            cv2.imwrite(str(base / 'depth_filled' / ('%07d.png' % i)), depth)
            np.savetxt(str(base / 'annotated_poses' / ('%07d.txt' % i)), p[i])
    (tmp / 'data' / 'bleach0.tar.gz').write_bytes(b'')
    templates = {'train_data_path': str(tmp / 'cfg' / '{object}' / 'train'), 'mean_std_path': str(tmp / 'cfg' / '{object}'),
                 'ckpt_dir': str(tmp / 'cfg' / '{object}' / 'model_best_val.pth.tar'), 'model_path': str(tmp / 'cfg' / '{object}' / 'textured.ply')}
    return tmp, templates, gt


def test_eval_all_against_the_cpu_restatement(pkg, tree):
    ev = importlib.import_module(PKG + '.eval_ycbineoat')
    tmp, _, gt = tree
    res = tmp / 'eval_res'
    rng = np.random.default_rng(3)
    from scipy.spatial.transform import Rotation
    for v in VIDEOS:                                                      # estimates from a few mm to some cm off the truth
        os.makedirs(res / v)
        for i, p in enumerate(gt[v]):
            q = p.copy()
            q[:3, :3] = Rotation.from_rotvec(rng.normal(0, 0.05, 3)).as_matrix() @ p[:3, :3]
            q[:3, 3] += rng.normal(0, 0.01 * (1 + i), 3)
            np.savetxt(str(res / v / ('%07d.txt' % i)), q)
    (res / 'old.tar.gz').write_bytes(b'')
    args = argparse.Namespace(res_dir=str(res) + '/', YCBInEOAT_dir=str(tmp / 'data'), ycb_dir=str(tmp / 'ycb'))
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        per_object, adi, add, n = ev.eval_all(args)
    lines = buf.getvalue().splitlines()
    ref_lines, ref_obj, ref_adi, ref_add, ref_n = YO.eval_all(args.res_dir, args.YCBInEOAT_dir, args.ycb_dir)
    assert n == ref_n == NFRAMES * len(VIDEOS) and len(lines) == len(ref_lines)
    for got, want in zip(lines, ref_lines):
        gw, ww = got.replace('=', ' ').split(), want.replace('=', ' ').split()
        assert len(gw) == len(ww)
        for a, b in zip(gw, ww):
            try:
                assert abs(float(a) - float(b)) <= 1e-9, (got, want)
            except ValueError:
                assert a == b, (got, want)
    assert abs(adi - ref_adi) <= 1e-9 and abs(add - ref_add) <= 1e-9
    for o in ev.OBJECTS:
        assert np.allclose(per_object[o], ref_obj[o], rtol=0, atol=1e-9), o
    assert 0 < add < 100 and per_object['tomato'] == (0.0, 0.0)
    os.remove(res / 'sugar_box1' / ('%07d.txt' % (NFRAMES - 1)))
    with pytest.raises(AssertionError, match='#pred_files:%d, #gt_files:%d' % (NFRAMES - 1, NFRAMES)):
        with contextlib.redirect_stdout(io.StringIO()):
            ev.eval_all(args)


@pytest.fixture(scope='module')
def steps(pkg):
    """Every Engine.track_render call of the module: (first weight id, last_step_was_graph)."""
    E = pkg.Engine
    orig = E.track_render
    rec = []

    def track_render(self, *a, **kw):
        out = orig(self, *a, **kw)
        wh = kw.get('weight_ids_host')
        rec.append((None if wh is None else int(wh[0]), self.last_step_was_graph()))
        return out
    E.track_render = track_render
    yield rec
    E.track_render = orig


@pytest.fixture(scope='module')
def driver_runs(tree, steps):
    pr = importlib.import_module(PKG + '.predict')
    tmp, templates, _ = tree
    runs = {}
    for name, kw in (('bf16x3_d1', dict(decode_ahead=1)), ('bf16x3_d2', dict(decode_ahead=2)), ('bf16x3_d4', dict(decode_ahead=4)),
                     ('bf16_d4', dict(precision='bf16', decode_ahead=4))):
        n0 = len(steps)
        runs[name] = pr.getResultsYcbInEOAT(str(tmp / 'data'), templates, str(tmp / ('out_' + name)), **kw)
        runs[name + '_steps'] = steps[n0:]
    return runs


@pytest.mark.parametrize('precision', ['bf16x3', 'bf16'])
def test_driver_bit_identical_to_an_on_track_batch_loop(pkg, tree, driver_runs, precision):
    pr = importlib.import_module(PKG + '.predict')
    ev = importlib.import_module(PKG + '.eval_ycbineoat')
    tmp, templates, gt = tree
    res = driver_runs[precision + '_d4']
    assert sorted(res) == sorted(VIDEOS)
    objs = pr.ycbineoat_objects(sorted(set(VIDEOS.values())), templates, precision=precision)
    eng = pkg.Engine(max_batch=1)
    trk = {o: pkg.Tracker(k['dataset_info'], k['mean'], k['std'], k['ckpt_dir'], model_path=k['model_path'], engine=eng,
                          weight_id=ev.OBJECTS.index(o), precision=precision, trans_normalizer=0.03, rot_normalizer=30 * np.pi / 180)
           for o, k in objs.items()}
    dev = eng.device
    for v, o in VIDEOS.items():
        ids = np.array([ev.OBJECTS.index(o)], dtype=np.int32)
        widths = torch.tensor([WIDTHS[o]], dtype=torch.float64, device=dev)
        poses = torch.from_numpy(gt[v][:1].copy()).to(dev)
        loop = []
        for i in range(NFRAMES):
            rgb = pr.read_rgb(str(tmp / 'data' / v / 'rgb' / ('%07d.png' % i)))
            depth = pr.read_depth(str(tmp / 'data' / v / 'depth_filled' / ('%07d.png' % i)))
            poses = trk[o].on_track_batch(poses, torch.from_numpy(rgb).to(dev), torch.from_numpy(depth).to(dev), weight_ids=ids, object_width=widths)
            loop.append(poses[0].cpu().numpy())
        loop = np.stack(loop)
        assert np.array_equal(res[v], loop), '%s: max |diff| %.3g' % (v, np.abs(res[v] - loop).max())
        files = np.stack([np.loadtxt(str(tmp / ('out_%s_d4' % precision) / v / ('%07d.txt' % i))) for i in range(NFRAMES)])
        assert np.array_equal(files, loop)
    eng.close()


def test_driver_same_for_every_decode_depth_and_close_to_per_video_runs(tree, driver_runs):
    pr = importlib.import_module(PKG + '.predict')
    tmp, templates, _ = tree
    for d in ('d1', 'd2'):
        for v in VIDEOS:
            assert np.array_equal(driver_runs['bf16x3_' + d][v], driver_runs['bf16x3_d4'][v]), (d, v)
    objs = pr.ycbineoat_objects(sorted(set(VIDEOS.values())), templates)
    worst = 0.0
    for v, o in VIDEOS.items():
        k = objs[o]
        one = pr.predictSequenceYcbInEOAT(str(tmp / 'data' / v), k['dataset_info'], k['mean'], k['std'], k['ckpt_dir'], k['model_path'],
                                          str(tmp / 'per_video' / v), max_batch=1)
        d = np.abs(one - driver_runs['bf16x3_d4'][v]).max()
        worst = max(worst, float(d))
        assert one.shape == (NFRAMES, 4, 4) and d < 6 * POSE_ATOL, '%s: %.3g' % (v, d)
    print('one pass vs per-video runs: max |pose diff| %.3g' % worst)


def test_every_step_after_an_objects_first_is_a_graph_replay(driver_runs):
    ev = importlib.import_module(PKG + '.eval_ycbineoat')
    for name in ('bf16x3_d1', 'bf16x3_d2', 'bf16x3_d4', 'bf16_d4'):
        rec = driver_runs[name + '_steps']
        assert len(rec) == NFRAMES * len(VIDEOS)
        seen = set()
        for wid, graph in rec:
            if wid in seen:
                assert graph, (name, rec)
            seen.add(wid)
        assert seen == {ev.OBJECTS.index(o) for o in VIDEOS.values()}


def test_cli_writes_the_tree_and_prints_the_scores(tree, capsys):
    pr = importlib.import_module(PKG + '.predict')
    tmp, templates, _ = tree
    out = tmp / 'cli'
    pr.main(['--mode', 'ycbineoat_all', '--YCBInEOAT_dir', str(tmp / 'data'), '--ycb_dir', str(tmp / 'ycb'), '--outdir', str(out),
             '--score', '--decode_ahead', '3'] + sum([['--' + k, v] for k, v in templates.items()], []))
    printed = capsys.readouterr().out.splitlines()
    assert sorted(os.listdir(out)) == sorted(VIDEOS)
    for v in VIDEOS:
        assert sorted(os.listdir(out / v)) == ['%07d.txt' % i for i in range(NFRAMES)]
    ref_lines = YO.eval_all(str(out) + '/', str(tmp / 'data'), str(tmp / 'ycb'))[0]
    tail = printed[-len(ref_lines):]
    assert [l.split('=')[0] for l in tail] == [l.split('=')[0] for l in ref_lines]
    assert tail[-3] == 'Total pose: %d' % (NFRAMES * len(VIDEOS))
