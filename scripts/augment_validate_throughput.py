"""Validation pairs/s with and without the reference's train-time augmentations (problems --augment), alternating in one process:
Problem.validate end to end (PNG decoding included) and the device step alone (eval_pairs on a batch already on the device), plus
the augmentation launches' own device time (se3tn_augment_crops, the step's two augmentation kernels, timed with CUDA events).
The card's name and power limit are printed with the numbers.

    python scripts/augment_validate_throughput.py [--pairs 1000] [--batch_size 200] [--rounds 4] [--precision bf16x3]
"""
import argparse, importlib, json, os, subprocess, sys, tempfile, time
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from validate_throughput import write_pairs
PKG = 'iros20-6d-pose-tracking_b200'
REF_CONFIG = {'hsv_noise': [15, 15, 15], 'bright_mag': [0.5, 1.5], 'gaussian_noise': {'rgb': 2, 'depth': 5}, 'gaussian_blur_kernel': 6}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--pairs', type=int, default=1000)
    ap.add_argument('--batch_size', type=int, default=200)
    ap.add_argument('--rounds', type=int, default=4)
    ap.add_argument('--precision', default='bf16x3')
    args = ap.parse_args()
    pkg = importlib.import_module(PKG)
    D = importlib.import_module(PKG + '.datasets'); P = importlib.import_module(PKG + '.problems')
    A = importlib.import_module(PKG + '.data_augmentation')
    synth = pkg.synth
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    mean, std = synth.default_mean_std()
    info = {'resolution': 176, 'camera': {'focalX': 1066.778, 'focalY': 1067.487, 'centerX': 312.9869, 'centerY': 241.3109}}
    with tempfile.TemporaryDirectory() as d:
        write_pairs(d, args.pairs)
        model = pkg.Se3TrackNet(max_batch=args.batch_size, precision=args.precision)
        model.load_state_dict(synth.make_state_dict(0))
        eng = model.engine
        probs = {}
        for name, augs in (('plain', None), ('augmented', A.from_config(REF_CONFIG))):
            ds = D.TrackDataset(d, 'val', mean, std, None, augs, dataset_info=info, trans_normalizer=0.02,
                                rot_normalizer=15 * np.pi / 180, engine=eng, precision=args.precision)
            loader = torch.utils.data.DataLoader(ds, batch_size=args.batch_size, shuffle=False, drop_last=False)
            probs[name] = P.Problem(model, None, loader, config={'loss_weights': {'trans': 1, 'rot': 1}})
        dev = eng.device
        bs = min(args.batch_size, args.pairs)
        batch = [D.read_pair(f) for f in sorted(probs['plain'].valid_data.dataset.rgbA_files)[:bs]]
        st = lambda k, dt: torch.from_numpy(np.stack([p[k] for p in batch]).astype(dt)).to(dev)
        dev_args = (st('rgbA', np.uint8), st('depthA', np.uint16), st('rgbB', np.uint8), st('depthB', np.uint16),
                    st('A_in_cam', np.float64), st('B_in_cam', np.float64), 0.02, 15 * np.pi / 180)
        seg = (st('depthB', np.int32) > 100).to(torch.uint8)
        idx = torch.arange(bs, dtype=torch.int64, device=dev)
        cfg = A.chain_config(A.from_config(REF_CONFIG), 0)
        outs = dict(out_trans=torch.empty(bs, 3, device=dev), out_rot=torch.empty(bs, 3, device=dev), out_sums=torch.empty(2, device=dev))
        steps = -(-args.pairs // bs)
        aug_out = (torch.empty_like(dev_args[2]), torch.empty_like(dev_args[3]))

        legs = {'problem_validate_plain': lambda: probs['plain'].validate(0),
                'problem_validate_augmented': lambda: probs['augmented'].validate(0),
                'device_step_plain': lambda: [eng.eval_pairs(*dev_args, precision=args.precision, **outs) for _ in range(steps)],
                'device_step_augmented': lambda: [eng.eval_pairs(*dev_args, precision=args.precision, augment=cfg, segB=seg, pair_index=idx,
                                                                 **outs) for _ in range(steps)]}
        for f in legs.values():                                # warm-up: graphs captured, pinned buffers allocated, page cache filled
            f(); torch.cuda.synchronize()
        rates = {k: [] for k in legs}
        for _ in range(args.rounds):
            for k, f in legs.items():
                torch.cuda.synchronize(); t0 = time.perf_counter()
                f(); torch.cuda.synchronize()
                rates[k].append(args.pairs / (time.perf_counter() - t0))
        # the augmentation launches alone: draws + pixels for one batch
        reps = 50
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ms = []
        for _ in range(args.rounds):
            e0.record()
            for _ in range(reps):
                eng.augment_crops(cfg, dev_args[2], dev_args[3], idx, segB=seg, out_rgbB=aug_out[0], out_depthB=aug_out[1])
            e1.record(); torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1) / reps)
    res = {'gpu': gpu, 'pairs': args.pairs, 'batch_size': args.batch_size, 'precision': args.precision, 'cpus': os.cpu_count(),
           'pairs_per_s': {k: [round(min(v), 1), round(max(v), 1)] for k, v in rates.items()},
           'augment_launches_ms_per_batch': [round(min(ms), 4), round(max(ms), 4)],
           'augment_min_bytes_per_pair': 176 * 176 * 11}   # rgbB | depthB read and written, maskB read
    print(json.dumps(res))


if __name__ == '__main__':
    main()
