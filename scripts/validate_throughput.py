"""Validation pairs/s end to end: Problem.validate (thread-pool PNG decoding into pinned staging, one se3tn_eval_pairs step per
batch) against the reference-style loop (the drop-in TrackDataset.__getitem__ per pair, then Se3TrackNet.forward and
Se3TrackNet.loss per batch of 200, as problems.py:106-132 drives them).  The two alternate `--rounds` times in one process; the
ranges are printed with the card's name and power limit.  Two more legs say which part sets the rate: decoding alone (the same
thread pool, no GPU) and the device step alone (eval_pairs on batches already on the device).

    python scripts/validate_throughput.py [--pairs 1000] [--batch_size 200] [--rounds 4] [--precision bf16x3]

The pair folder is written to a temporary directory (synthetic crops in the reference's on-disk format) and removed afterwards.
"""
import argparse, importlib, json, os, subprocess, sys, tempfile, time
from concurrent.futures import ThreadPoolExecutor
import cv2
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
PKG = 'iros20-6d-pose-tracking_b200'


def write_pairs(d, n, seed=0):
    rng = np.random.default_rng(seed)
    for i in range(n):
        stem = os.path.join(d, '%06d' % i)
        for name in ('rgbA', 'rgbB'):
            img = rng.integers(0, 256, (176, 176, 3), dtype=np.uint8)
            img[40:136, 40:136] //= 2                              # some structure, so the PNGs are not all incompressible noise
            cv2.imwrite(stem + name + '.png', img)
        for name in ('depthA', 'depthB'):
            cv2.imwrite(stem + name + '.png', rng.integers(300, 1800, (176, 176)).astype(np.uint16))
        B = np.eye(4); B[:3, 3] = (rng.uniform(-.1, .1), rng.uniform(-.1, .1), rng.uniform(.5, .8))
        A = B.copy(); A[:3, 3] += rng.normal(0, 0.005, 3)
        np.savez(stem + 'meta.npz', A_in_cam=A, B_in_cam=B)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--pairs', type=int, default=1000)
    ap.add_argument('--batch_size', type=int, default=200)
    ap.add_argument('--rounds', type=int, default=4)
    ap.add_argument('--precision', default='bf16x3')
    args = ap.parse_args()
    pkg = importlib.import_module(PKG)
    D = importlib.import_module(PKG + '.datasets'); P = importlib.import_module(PKG + '.problems')
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
        ds = D.TrackDataset(d, 'val', mean, std, dataset_info=info, trans_normalizer=0.02, rot_normalizer=15 * np.pi / 180,
                            engine=eng, precision=args.precision)
        loader = torch.utils.data.DataLoader(ds, batch_size=args.batch_size, shuffle=False, drop_last=False)
        prob = P.Problem(model, None, loader, config={'loss_weights': {'trans': 1, 'rot': 1}})

        def fused():
            return prob.validate(0)

        def reference_style():
            losses_t, losses_r = [], []
            for b0 in range(0, len(ds), args.batch_size):
                items = [ds[i] for i in range(b0, min(len(ds), b0 + args.batch_size))]
                dataA = torch.stack([it[0][0] for it in items]); dataB = torch.stack([it[0][1] for it in items])
                target = [torch.from_numpy(np.stack([it[1][k] for it in items])).cuda() for k in (0, 1)]
                pred = model(dataA.cuda(), dataB.cuda(), return_feature=False)
                out = model.loss((pred['trans'], pred['rot']), target)
                losses_t.append(out['trans'].cpu().item()); losses_r.append(out['rot'].cpu().item())
            return np.mean(losses_t) + np.mean(losses_r)

        def decode_only():
            with ThreadPoolExecutor(max_workers=min(16, os.cpu_count() or 4)) as pool:
                list(pool.map(D.read_pair, ds.rgbA_files))

        dev = eng.device
        bs = min(args.batch_size, len(ds))
        batch = [D.read_pair(f) for f in ds.rgbA_files[:bs]]
        st = lambda k, dt: torch.from_numpy(np.stack([p[k] for p in batch]).astype(dt)).to(dev)
        dev_args = (st('rgbA', np.uint8), st('depthA', np.uint16), st('rgbB', np.uint8), st('depthB', np.uint16),
                    st('A_in_cam', np.float64), st('B_in_cam', np.float64), 0.02, 15 * np.pi / 180)
        outs = dict(out_trans=torch.empty(bs, 3, device=dev), out_rot=torch.empty(bs, 3, device=dev), out_sums=torch.empty(2, device=dev))

        def step_only():
            for _ in range(-(-len(ds) // bs)):
                eng.eval_pairs(*dev_args, precision=args.precision, **outs)

        legs = {'problem_validate': fused, 'reference_style_loop': reference_style, 'decode_only_threads': decode_only, 'device_step_only': step_only}
        for f in legs.values():                                # warm-up: graphs captured, pinned buffers allocated, page cache filled
            f(); torch.cuda.synchronize()
        rates = {k: [] for k in legs}
        vals = {}
        for _ in range(args.rounds):
            for k, f in legs.items():
                torch.cuda.synchronize(); t0 = time.perf_counter()
                v = f(); torch.cuda.synchronize()
                rates[k].append(len(ds) / (time.perf_counter() - t0))
                if v is not None:
                    vals[k] = v
    res = {'gpu': gpu, 'pairs': len(ds), 'batch_size': args.batch_size, 'precision': args.precision, 'cpus': os.cpu_count(),
           'pairs_per_s': {k: [round(min(v), 1), round(max(v), 1)] for k, v in rates.items()},
           'validation_loss': {k: float(v) for k, v in vals.items()}}
    print(json.dumps(res))


if __name__ == '__main__':
    main()
