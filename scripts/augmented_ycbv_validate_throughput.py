"""Validation on perturbed YCB-Video key frames under the train-time augmentations, three routes on the synthetic layout of
perturbed_validate_throughput.build_layout:

  * augmented file route: `produce_train_pair_data --mode ycbv` (produce_ycbv: PNG / npz pair files), then problems.evaluate on
    each class's folder through TrackDataset(augmentations=...) -- what `problems --val_dir <class folder> --augment` runs;
  * augmented one pass: problems.validate_ycbv with the chain -- `problems --ycb_dir --augment`;
  * plain one pass: problems.validate_ycbv without it.

The chain is train.py:85-92's, built by data_augmentation.from_config from the reference's config.yml block; the generator and
augmentation seeds are both --seed.  The routes alternate `--rounds` times in one process; the script checks that both augmented
routes give the same pair counts and losses and prints pairs/s as one JSON line (also to `--out`), with the card's name and power
limit read in the same run.

    python scripts/augmented_ycbv_validate_throughput.py [--frames 200] [--num_sample 10] [--rounds 2] [--precision bf16x3] [--out FILE]
"""
import argparse, importlib, json, os, shutil, subprocess, sys, tempfile, time
import numpy as np
import torch
import yaml
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.dirname(__file__))
PKG = 'iros20-6d-pose-tracking_b200'
from perturbed_validate_throughput import build_layout, CLASSES, H, W          # noqa: E402

CONFIG = {'data_augmentation': {'hsv_noise': [15, 15, 15], 'bright_mag': [0.5, 1.5], 'gaussian_noise': {'rgb': 2, 'depth': 5},
                                'gaussian_blur_kernel': 6}}                  # the reference's config.yml block


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=200)
    ap.add_argument('--num_sample', type=int, default=10)
    ap.add_argument('--batch_size', type=int, default=200)
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--precision', default='bf16x3')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    pkg = importlib.import_module(PKG)
    PP, P, D, E, A = (importlib.import_module(PKG + '.' + m) for m in ('produce_train_pair_data', 'problems', 'datasets', 'engine',
                                                                       'data_augmentation'))
    mesh_io = importlib.import_module(PKG + '.mesh_io')
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    chain = A.from_config(CONFIG)
    mode = args.precision
    with tempfile.TemporaryDirectory() as root:
        tpl = build_layout(root, pkg.synth, mesh_io, args.frames)
        ycb = os.path.join(root, 'ycb')

        def file_route():
            out = os.path.join(root, 'pairs')
            shutil.rmtree(out, ignore_errors=True)
            counts = PP.produce_ycbv(ycb, CLASSES, tpl, out, num_sample=args.num_sample, seed=args.seed)
            eng = E.Engine(max_batch=args.batch_size)
            res = {}
            for c in CLASSES:
                d = tpl['mean_std_path'].format(class_id=c)
                info = yaml.safe_load(open(os.path.join(d, 'dataset_info.yml')))
                ds = D.TrackDataset(os.path.join(out, '%03d_obj' % c), 'val', np.load(os.path.join(d, 'mean.npy')),
                                    np.load(os.path.join(d, 'std.npy')), None, chain, None, dataset_info=info,
                                    trans_normalizer=info['max_translation'], rot_normalizer=info['max_rotation'] * np.pi / 180,
                                    augment_seed=args.seed)
                model = pkg.Se3TrackNet(engine=eng, weight_id=0)
                model.load_state_dict(torch.load(tpl['ckpt_dir'].format(class_id=c), map_location='cpu')['state_dict'])
                r = P.evaluate(model, ds, args.batch_size, precision=mode)
                res[c] = (counts[c], r['trans'], r['rot'])
            eng.close()
            return res

        def one_pass(augmentations):
            r = P.validate_ycbv(ycb, CLASSES, tpl, num_sample=args.num_sample, seed=args.seed, batch_size=args.batch_size,
                                max_batch=args.batch_size, precisions=[mode], augmentations=augmentations)
            return {c: (r[c][mode]['pairs'], r[c][mode]['trans'], r[c][mode]['rot']) for c in CLASSES}

        routes = (('augmented_file_route', file_route), ('augmented_one_pass', lambda: one_pass(chain)),
                  ('plain_one_pass', lambda: one_pass(None)))
        times = {name: [] for name, _ in routes}
        results = {}
        for _ in range(args.rounds):
            for name, fn in routes:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                results[name] = fn()
                torch.cuda.synchronize()
                times[name].append(time.perf_counter() - t0)
    pairs = sum(n for n, _, _ in results['augmented_one_pass'].values())
    out = dict(gpu=gpu, frames=args.frames, frame_hw=[H, W], classes=len(CLASSES), num_sample=args.num_sample,
               batch_size=args.batch_size, precision=mode, seed=args.seed, pairs=pairs,
               identical=results['augmented_file_route'] == results['augmented_one_pass'],
               augmentation_changes_loss=results['augmented_one_pass'] != results['plain_one_pass'])
    for name, ts in times.items():
        out[name] = dict(seconds=[round(t, 3) for t in ts], pairs_per_s=[round(pairs / t, 1) for t in ts])
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')
    if not out['identical']:
        raise SystemExit('the augmented one pass and the augmented file route disagree')


if __name__ == '__main__':
    main()
