"""eval_ycbineoat.eval_all (reference eval_ycbineoat.py:49-109) restated on the CPU: the same folders, files, printed lines and AUCs,
with se3_oracle's add / adi (scipy cKDTree, as Utils.adi) and vocap (eval_ycb.py VOCap).  The GPU drop-in is tested against it.

A VOCap of errors none of which is below 0.1 m (or of no errors) is 0 here, as on the device; the reference raises there."""
import glob, os
import numpy as np
import se3_oracle as O

OBJECTS = ['cracker', 'bleach', 'sugar', 'tomato', 'mustard']


def _vocap(errs):
    errs = np.asarray(errs, dtype=np.float64)
    return O.vocap(errs) if (errs < 0.1).any() else 0.0


def eval_all(res_dir, YCBInEOAT_dir, ycb_dir):
    """-> (lines printed, {object: (adi_auc, add_auc)}, adi_auc, add_auc, n poses)."""
    lines = []
    data_dir = '{}/'.format(YCBInEOAT_dir)
    models = {}
    for t in glob.glob('{}/CADmodels/*/points.xyz'.format(ycb_dir)):
        pts = np.loadtxt(t, dtype=np.float64).reshape(-1, 3)
        for obj in OBJECTS:
            if obj in t:
                models[obj] = pts
    class_res = {obj: {'add': [], 'add-s': []} for obj in OBJECTS}
    for folder in os.listdir(res_dir):
        if '.tar.gz' in folder:
            continue
        lines.append(folder)
        pred_files = sorted(glob.glob(res_dir + folder + '/*.txt'))
        obj = next(o for o in OBJECTS if o in folder)
        gt_files = sorted(glob.glob(data_dir + folder + '/annotated_poses/*.txt'))
        assert len(pred_files) == len(gt_files), '#pred_files:{}, #gt_files:{}'.format(len(pred_files), len(gt_files))
        for i in range(len(pred_files)):
            pred, gt = np.loadtxt(pred_files[i]), np.loadtxt(gt_files[i])
            class_res[obj]['add'].append(O.add(pred, gt, models[obj]))
            class_res[obj]['add-s'].append(O.adi(pred, gt, models[obj]))
    adds, adis, per_object = [], [], {}
    for k in class_res:
        adis += class_res[k]['add-s']
        adds += class_res[k]['add']
        per_object[k] = (_vocap(class_res[k]['add-s']) * 100, _vocap(class_res[k]['add']) * 100)
        lines.append('{}: adi={} add={}'.format(k, *per_object[k]))
    adi_auc, add_auc = _vocap(adis) * 100, _vocap(adds) * 100
    lines.append('Total pose: {}'.format(len(adis)))
    lines += ['', 'Overall, adi={} add={}'.format(adi_auc, add_auc)]
    return lines, per_object, adi_auc, add_auc, len(adis)
