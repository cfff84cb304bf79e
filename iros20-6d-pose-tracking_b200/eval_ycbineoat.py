"""Drop-in for the reference's eval_ycbineoat.py (eval_all, eval_ycbineoat.py:49-109): scoring of tracked YCBInEOAT videos.

Same file conventions and printed lines: result poses from <res_dir>/<video>/%07d.txt (what predict.getResultsYcbInEOAT writes),
ground truth from <YCBInEOAT_dir>/<video>/annotated_poses/*.txt, model points from <ycb_dir>/CADmodels/*/points.xyz; every
video folder in os.listdir order, then '<obj>: adi=.. add=..' for each of OBJECTS, 'Total pose:' and 'Overall, adi=.. add=..'
(AUCs in percent).  The reference calls Utils.add and Utils.adi once per pose and VOCap once per object and once on all poses;
here ADD and ADD-S of every pose of every video are one se3tn_add_adi_sets launch, and each metric's AUCs are one
se3tn_vocap_sets call.  A video whose pose counts differ raises the reference's AssertionError.

Two inputs the reference accepts silently are refused with a ValueError that names the folder or path:
  * a video folder that names none of OBJECTS.  The reference's loop (eval_ycbineoat.py:80-86) then keeps the previous folder's
    gt_files and scores this folder's poses against another video's ground truth (or fails on an unbound name).
  * a points.xyz whose object name occurs in its path only through ycb_dir, not in the CADmodels/ folder name.  The reference
    (eval_ycbineoat.py:65-67) tests `obj in t` on the whole path, so a ycb_dir such as /data/sugar_runs makes every model the
    sugar model.

    python -m <package>.eval_ycbineoat --YCBInEOAT_dir .. --ycb_dir .. --res_dir ..
"""
import argparse, glob, os
import numpy as np
import torch
from . import Utils as U
from .eval_ycb import _read_points

OBJECTS = ['cracker', 'bleach', 'sugar', 'tomato', 'mustard']


def video_object(folder):
    """The object a video folder shows: the first of OBJECTS whose name is part of the folder name, or None."""
    for o in OBJECTS:
        if o in folder:
            return o
    return None


def model_points(ycb_dir):
    """{object: (m,3) float64 points} from <ycb_dir>/CADmodels/*/points.xyz; a later glob match replaces an earlier one, as in
    the reference."""
    models = {}
    for t in glob.glob('{}/CADmodels/*/points.xyz'.format(ycb_dir)):
        folder = os.path.basename(os.path.dirname(t))
        pts = None
        for obj in OBJECTS:
            if obj not in t:
                continue
            if obj not in folder:
                raise ValueError('%s: the object name %r occurs only in ycb_dir, not in the CADmodels/ folder name %r' % (t, obj, folder))
            if pts is None:
                pts = _read_points(t)
            models[obj] = pts
    return models


def eval_all(args):
    """args.res_dir (ending in '/'), args.YCBInEOAT_dir, args.ycb_dir -> ({object: (adi_auc, add_auc)}, adi_auc, add_auc, n poses)."""
    res_dir = args.res_dir
    data_dir = '{}/'.format(args.YCBInEOAT_dir)
    models = model_points(args.ycb_dir)
    preds, gts, objs = [], [], []
    for folder in os.listdir(res_dir):
        if '.tar.gz' in folder:
            continue
        print(folder)
        pred_files = sorted(glob.glob(res_dir + folder + '/*.txt'))
        obj = video_object(folder)
        if obj is None:
            raise ValueError('%s: the folder name contains none of %s, so no ground truth or model belongs to it' % (res_dir + folder, OBJECTS))
        gt_files = sorted(glob.glob(data_dir + folder + '/annotated_poses/*.txt'))
        assert len(pred_files) == len(gt_files), '#pred_files:{}, #gt_files:{}'.format(len(pred_files), len(gt_files))
        if pred_files and obj not in models:
            raise ValueError('%s: no CADmodels/*%s*/points.xyz under %s' % (res_dir + folder, obj, args.ycb_dir))
        for i in range(len(pred_files)):
            preds.append(np.loadtxt(pred_files[i]))
            gts.append(np.loadtxt(gt_files[i]))
            objs.append(OBJECTS.index(obj))

    eng = U._eng()
    dev = eng.device
    used = [o for o in OBJECTS if o in models]
    obj_ids = np.asarray(objs, dtype=np.int32)
    if preds:
        table_id = np.asarray([used.index(OBJECTS[k]) for k in objs], dtype=np.int32)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(np.stack(a).reshape(-1, 4, 4), dtype=np.float64)).to(dev)
        add_d, adi_d = eng.add_adi_sets([models[o] for o in used], table_id, t(preds), t(gts))
    else:
        add_d = adi_d = torch.empty(0, dtype=torch.float64, device=dev)
    ids_d = torch.from_numpy(obj_ids).to(dev)
    adi_ap = eng.vocap_sets(adi_d, ids_d, len(OBJECTS)) * 100
    add_ap = eng.vocap_sets(add_d, ids_d, len(OBJECTS)) * 100
    per_object = {}
    for k, obj in enumerate(OBJECTS):
        per_object[obj] = (float(adi_ap[k]), float(add_ap[k]))
        print('{}: adi={} add={}'.format(obj, per_object[obj][0], per_object[obj][1]))
    adi_auc, add_auc = float(adi_ap[-1]), float(add_ap[-1])
    print('Total pose:', len(objs))
    print('\nOverall, adi={} add={}'.format(adi_auc, add_auc))
    return per_object, adi_auc, add_auc, len(objs)


def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument('--YCBInEOAT_dir', required=True)
    parser.add_argument('--ycb_dir', required=True)
    parser.add_argument('--res_dir', type=str, required=True, help='the folder with <video>/%%07d.txt')
    args = parser.parse_args(argv)
    if not args.res_dir.endswith('/'):
        args.res_dir += '/'
    return eval_all(args)


if __name__ == '__main__':
    main()
