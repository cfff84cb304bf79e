"""Re-initialisation in the one-pass YCB-Video driver (--mode ycbv_all --reinit_below, getResultsYcbAll(reinit=)) on the
synthetic data set of the start-from-mask driver tests (two test sequences, classes 2 and 5, seg/ label images): a run in which
nothing is lost writes the pose and fit files of a run without re-initialisation byte for byte, and reinit.npy holds 0 or 1 as
each fit row says (the checkpoints are random, so a track may drift below the threshold without being lost); a run in
which every track is lost every frame writes the codes of the rule, and each restarted pose file holds the start MaskStarts
finds on that frame; score_reinit counts what the files say; several GPUs write the one-GPU tree; a missing label image is
refused before anything is loaded."""
import os
import shutil
import numpy as np
import pytest
import torch
from test_gpu_init_drivers import CLASSES, INIT, NFRAMES, SEQS, _same_tree, pr, tree      # noqa: F401

pytestmark = pytest.mark.gpu
TAU = 10


def _files(root, name):
    return sorted(os.path.join(dp, f) for dp, _, fs in os.walk(root) for f in fs if f == name)


def _without(root, name, dest):
    """A copy of the tree `root` without its `name` files."""
    shutil.copytree(root, dest, ignore=shutil.ignore_patterns(name))
    return dest


def test_nothing_lost_writes_the_run_without_reinit(pr, tree):
    tmp, ycb, templates = tree
    pr.getResultsYcbAll(str(ycb), list(CLASSES), templates, str(tmp / 'plain'), fit=TAU)
    # below 0.001 for 1000 frames in a row: nothing is lost in three frames
    argv = ['--mode', 'ycbv_all', '--ycb_dir', str(ycb), '--class_ids', '2,5', '--outdir', str(tmp / 'quiet'), '--fit', str(TAU),
            '--reinit_below', '0.001', '--reinit_after', '1000'] + sum([['--' + k, v] for k, v in templates.items()], [])
    pr.main(argv)
    files = _files(str(tmp / 'quiet'), pr.REINIT_FILE)
    assert len(files) == sum(len(c) for c in SEQS.values())
    for f in files:
        e, rows = np.load(f), np.load(os.path.join(os.path.dirname(f), pr.FIT_FILE)).astype(np.int64)
        assert e.dtype == np.int32 and e.shape == (NFRAMES,) and e[0] == -1
        # no track is lost; a frame is below (1) exactly when the rule says so for its fit row
        below = (rows[1:, 0] == 0) | (1000 * rows[1:, 2] < 1 * rows[1:, 0])
        assert np.array_equal(e[1:], below.astype(np.int32))
    rest = _without(str(tmp / 'quiet'), pr.REINIT_FILE, str(tmp / 'quiet_rest'))
    assert _same_tree(str(tmp / 'plain'), rest) and _same_tree(rest, str(tmp / 'plain'))


def test_restarts_follow_the_rule_and_equal_mask_starts(pr, tree):
    tmp, ycb, templates = tree
    # below 1.0 after 1: a track is lost in every frame whose model pixels are not all inliers
    reinit = dict(below=1.0, after=1, init=INIT)
    pr.getResultsYcbAll(str(ycb), list(CLASSES), templates, str(tmp / 'busy'), fit=TAU, reinit=reinit)
    classes = pr.ycb_all_classes(str(ycb), list(CLASSES), templates)
    starts = pr.MaskStarts(classes, 2, INIT)          # the driver's Engine holds 2 tracks x keep, as this one
    names = pr.ycb_class_names(str(ycb))
    restarts = 0
    try:
        for seq, cls in SEQS.items():
            base = os.path.join(str(ycb), 'data_organized', '%04d' % seq)
            for c in cls:
                sdir = os.path.join(pr.ycb_all_res_dir(str(tmp / 'busy'), names[c - 1]), 'seq%d' % seq)
                e, rows = np.load(os.path.join(sdir, pr.REINIT_FILE)), np.load(os.path.join(sdir, pr.FIT_FILE))
                for i in range(1, NFRAMES):
                    assert e[i] in (0, 2, 3, 4)
                    if e[i] != 2:                    # the step's own row: not below only when every model pixel fits
                        assert (e[i] == 0) == (rows[i, 2] == rows[i, 0] and rows[i, 0] > 0)
                        continue
                    restarts += 1
                    D = pr.read_depth(os.path.join(base, 'depth_filled', '%06d-depth.png' % (i + 1)))
                    L = pr.read_seg(os.path.join(base, 'seg', '%06d-label.png' % (i + 1)))
                    P, R = starts(D, L, [c])
                    assert R[0, 0] == 0
                    assert np.array_equal(np.loadtxt(os.path.join(sdir, '%07d.txt' % i)),
                                          np.loadtxt(_saved(tmp, P[0].cpu().numpy())))
    finally:
        starts.close()
    assert restarts > 0
    # score_reinit counts what the files say; restarts are compared with the annotations on points.xyz
    for k, name in enumerate(names):                 # eval_ycb reads class k's points from the k-th points.xyz
        c = k + 1 if k + 1 in CLASSES else CLASSES[0]
        np.savetxt(os.path.join(str(ycb), 'CADmodels', name, 'points.xyz'), np.asarray(
            pr.object_cloud(templates['model_path'].format(class_id=c)).points, np.float64))
    r = pr.score_reinit(str(tmp / 'busy'), str(ycb), list(CLASSES))
    e = np.concatenate([np.load(f)[1:] for f in _files(str(tmp / 'busy'), pr.REINIT_FILE)])
    assert r['tracked'] == len(e) and r['restarted'] == restarts == (e == 2).sum()
    assert r['attempts'] == r['restarted'] + r['rejected'] + r['failed'] == (e >= 2).sum() and 0 <= r['restarts_near'] <= 1


def _saved(tmp, P):
    """P through np.savetxt, as the driver writes a pose file."""
    p = os.path.join(str(tmp), 'start.txt')
    np.savetxt(p, P)
    return p


def test_a_missing_label_image_is_refused_first(pr, tree):
    tmp, ycb, templates = tree
    copy = tmp / 'ycb_no_label'
    shutil.copytree(str(ycb), str(copy))
    os.remove(os.path.join(str(copy), 'data_organized', '0049', 'seg', '%06d-label.png' % NFRAMES))
    with pytest.raises(FileNotFoundError, match='sequence 0049 have no label image'):
        pr.getResultsYcbAll(str(copy), list(CLASSES), templates, str(tmp / 'nolabel'), reinit=dict(below=0.5))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs two GPUs')
def test_reinit_on_two_gpus_writes_the_one_gpu_tree(pr, tree):
    tmp, ycb, templates = tree
    reinit = dict(below=1.0, after=1, init=INIT)
    pr.getResultsYcbAll(str(ycb), list(CLASSES), templates, str(tmp / 'r1'), fit=TAU, reinit=reinit)
    pr.getResultsYcbAll(str(ycb), list(CLASSES), templates, str(tmp / 'r2'), fit=TAU, reinit=reinit, gpus=2)
    assert _same_tree(str(tmp / 'r1'), str(tmp / 'r2')) and _same_tree(str(tmp / 'r2'), str(tmp / 'r1'))
