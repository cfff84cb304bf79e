"""The drivers of the start from boxes on a synthetic data set in the YCB-Video layout with seg/ label images (the layout of
test_gpu_init_drivers): each class's box is the tight box of its pixels in the label image.  --mode ycbv_all --init box writes
the tree a run started from Engine.init_boxes' poses writes, on one GPU or two; --mode ycbv_init --init box returns the poses
direct init_boxes calls give."""
import filecmp
import importlib
import os
import shutil
import sys
import numpy as np
import pytest
import torch
import yaml

pytestmark = pytest.mark.gpu
PKG = 'iros20-6d-pose-tracking_b200'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import init_box_ref as ibr  # noqa: E402
import init_ref  # noqa: E402

CLASSES = (2, 5)
SEQS = {48: (2, 5), 49: (5,)}
NFRAMES = 3
WIDTHS = {2: 180.0, 5: 200.0}
INIT = dict(viewpoints=12, inplane=4, keep=2, icp=2)


@pytest.fixture(scope='module')
def pr():
    return importlib.import_module(PKG + '.predict')


@pytest.fixture(scope='module')
def tree(tmp_path_factory, synth):
    import cv2
    mio = importlib.import_module(PKG + '.mesh_io')
    tmp = tmp_path_factory.mktemp('init_box_drivers')
    ycb, cfg = tmp / 'ycb', tmp / 'cfg'
    K = synth.CAMERA_K
    cam = {'focalX': float(K[0, 0]), 'focalY': float(K[1, 1]), 'centerX': float(K[0, 2]), 'centerY': float(K[1, 2]), 'height': 480, 'width': 640}
    mean, std = synth.default_mean_std()
    meshes = {c: synth.mesh(3, seed=c) for c in CLASSES}
    for c in CLASSES:
        d = cfg / ('c%d' % c)
        (d / 'train').mkdir(parents=True)
        yaml.safe_dump({'resolution': 176, 'object_width': WIDTHS[c], 'boundingbox': 10, 'camera': cam}, open(d / 'dataset_info.yml', 'w'))
        np.save(d / 'mean.npy', mean); np.save(d / 'std.npy', std)
        torch.save({'epoch': 1, 'state_dict': synth.make_state_dict(c), 'best_prec': 0.0}, str(d / 'model_best_val.pth.tar'))
        mio.save_ply_mesh(str(d / 'textured.ply'), meshes[c])
    for k in range(1, 22):
        (ycb / 'CADmodels' / ('%03d_obj' % k)).mkdir(parents=True)
    keyframes = []
    for seq, cls in SEQS.items():
        base = ycb / 'data_organized' / ('%04d' % seq)
        for d in ['color', 'depth_filled', 'seg'] + ['pose_gt/%d' % c for c in cls]:
            (base / d).mkdir(parents=True)
        for i in range(NFRAMES):
            D, L = np.zeros((480, 640), np.uint16), np.zeros((480, 640), np.uint8)
            for j, c in enumerate(cls):
                P = np.eye(4)
                P[:3, :3] = synth._random_rotations(np.random.default_rng(100 * seq + 10 * c), 1)[0]
                P[:3, 3] = (-0.12 + 0.24 * j + 0.002 * i, 0.03, 0.75 + 0.05 * j)
                np.savetxt(str(base / 'pose_gt' / str(c) / ('%06d.txt' % (i + 1))), P)
                d = init_ref.full_depth(P, K, meshes[c], 480, 640)
                win = (d > 0) & ((D == 0) | (d < D))
                D, L = np.where(win, d, D), np.where(win, np.uint8(c), L)
            cv2.imwrite(str(base / 'color' / ('%06d-color.png' % (i + 1))), synth.raw_frame(seed=seq + i)[0][..., ::-1])
            cv2.imwrite(str(base / 'depth_filled' / ('%06d-depth.png' % (i + 1))), D)
            cv2.imwrite(str(base / 'seg' / ('%06d-label.png' % (i + 1))), L)
            keyframes.append('%04d/%06d' % (seq, i + 1))
    (ycb / 'image_sets').mkdir()
    (ycb / 'image_sets' / 'keyframe.txt').write_text('\n'.join(keyframes) + '\n')
    templates = {'train_data_path': str(cfg / 'c{class_id}' / 'train'), 'mean_std_path': str(cfg / 'c{class_id}'),
                 'ckpt_dir': str(cfg / 'c{class_id}' / 'model_best_val.pth.tar'), 'model_path': str(cfg / 'c{class_id}' / 'textured.ply')}
    return tmp, ycb, templates


def _same_tree(a, b):
    for root, _, files in os.walk(a):
        for f in files:
            p = os.path.join(root, f)
            q = os.path.join(b, os.path.relpath(p, a))
            assert os.path.isfile(q) and filecmp.cmp(p, q, shallow=False), q
    return True


def test_label_boxes_are_the_tight_boxes(pr, tree):
    _, ycb, _ = tree
    L = pr.read_seg(os.path.join(str(ycb), 'data_organized', '0048', 'seg', '000001-label.png'))
    boxes = pr.label_boxes(L, [2, 5, 7])
    assert np.array_equal(boxes, np.stack([ibr.tight_box(L, c) for c in (2, 5, 7)]))
    assert list(boxes[2]) == [0, 0, 0, 0]


def test_init_box_tree_equals_a_run_from_the_init_boxes(pr, tree):
    tmp, ycb, templates = tree
    argv = ['--mode', 'ycbv_all', '--ycb_dir', str(ycb), '--class_ids', '2,5', '--outdir', str(tmp / 'box'), '--init', 'box',
            '--init_depths', '2', '--init_viewpoints', '12', '--init_inplane', '4', '--init_keep', '2', '--init_icp', '2'] + \
        sum([['--' + k, v] for k, v in templates.items()], [])
    pr.main(argv)
    classes = pr.ycb_all_classes(str(ycb), list(CLASSES), templates)
    starts = pr.MaskStarts(classes, 2, INIT)
    copy = tmp / 'ycb_from_box_starts'
    shutil.copytree(str(ycb), str(copy))
    try:
        for seq, cls in SEQS.items():
            base = os.path.join(str(ycb), 'data_organized', '%04d' % seq)
            D = pr.read_depth(os.path.join(base, 'depth_filled', '000001-depth.png'))
            L = pr.read_seg(os.path.join(base, 'seg', '000001-label.png'))
            ow = torch.tensor([WIDTHS[c] for c in cls], dtype=torch.float64, device=starts.eng.device)
            ids = np.asarray(cls, np.int32)
            P, R = starts.eng.init_boxes(torch.from_numpy(D).to(starts.eng.device), [ibr.tight_box(L, c) for c in cls], starts.K, ow,
                                         weight_ids=ids, init=INIT, depths=2, **starts.render)
            assert (R[:, 0] == 0).all()
            for j, c in enumerate(cls):
                np.savetxt(os.path.join(str(copy), 'data_organized', '%04d' % seq, 'pose_gt', str(c), '000001.txt'), P[j].cpu().numpy())
    finally:
        starts.close()
    pr.getResultsYcbAll(str(copy), list(CLASSES), templates, str(tmp / 'gt_box'), initialize_method='gt')
    assert _same_tree(str(tmp / 'box'), str(tmp / 'gt_box')) and _same_tree(str(tmp / 'gt_box'), str(tmp / 'box'))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs two GPUs')
def test_init_box_on_two_gpus_writes_the_one_gpu_tree(pr, tree):
    tmp, ycb, templates = tree
    one = pr.getResultsYcbAll(str(ycb), list(CLASSES), templates, str(tmp / 'b1'), initialize_method='box', init=INIT, depths=2)
    two = pr.getResultsYcbAll(str(ycb), list(CLASSES), templates, str(tmp / 'b2'), initialize_method='box', init=INIT, depths=2, gpus=2)
    assert _same_tree(str(tmp / 'b1'), str(tmp / 'b2'))
    for c in one:
        for s in one[c]:
            assert np.array_equal(one[c][s], two[c][s])


def test_init_box_refuses_a_class_without_a_start(pr, tree):
    tmp, ycb, templates = tree
    copy = tmp / 'ycb_no_box'
    shutil.copytree(str(ycb), str(copy))
    import cv2
    p = os.path.join(str(copy), 'data_organized', '0049', 'seg', '000001-label.png')
    cv2.imwrite(p, np.zeros((480, 640), np.uint8))
    with pytest.raises(ValueError, match='sequence 0049, class 5.*box is empty'):
        pr.getResultsYcbAll(str(copy), list(CLASSES), templates, str(tmp / 'none'), initialize_method='box', init=INIT)


def test_ycbv_init_box_rows_equal_direct_calls(pr, tree, capsys):
    tmp, ycb, templates = tree
    res = pr.main(['--mode', 'ycbv_init', '--ycb_dir', str(ycb), '--class_ids', '2,5', '--train_data_path', templates['train_data_path'],
                   '--model_path', templates['model_path'], '--init_viewpoints', '12', '--init_inplane', '4', '--init_keep', '2',
                   '--init_icp', '2', '--init', 'box', '--init_depths', '2'])
    out = capsys.readouterr().out
    assert 'best of K' in out and 'boxes from the labels, D 2' in out
    jobs = importlib.import_module(PKG + '.produce_train_pair_data').ycbv_keyframe_jobs(str(ycb), list(CLASSES))
    starts = pr.MaskStarts(pr.init_classes(str(ycb), list(CLASSES), templates), 2, INIT)
    try:
        direct = []
        for _, depth_path, seg_path, rows in jobs:
            cls = [c for c, _ in rows]
            L = pr.read_seg(seg_path)
            ow = torch.tensor([WIDTHS[c] for c in cls], dtype=torch.float64, device=starts.eng.device)
            P, R = starts.eng.init_boxes(torch.from_numpy(pr.read_depth(depth_path)).to(starts.eng.device),
                                         [ibr.tight_box(L, c) for c in cls], starts.K, ow, weight_ids=np.asarray(cls, np.int32),
                                         init=INIT, depths=2, **starts.render)
            assert (R[:, 0] == 0).all()
            direct.append(P.cpu().numpy())
    finally:
        starts.close()
    assert res['all']['failed'] == 0
    assert np.array_equal(res['all']['icp']['poses'], np.concatenate(direct))
