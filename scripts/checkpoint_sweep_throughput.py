"""Wall time of `problems --val_dir` over N checkpoints: one pass (problems.evaluate with N models on one Engine, each step's
pairs decoded once) against N separate single-checkpoint evaluate calls, for N = 1, 2, 4, the two alternating `--rounds` times in
one process.  Prints one JSON line per N with both ranges, and the card's name and power limit.

    python scripts/checkpoint_sweep_throughput.py [--pairs 1000] [--batch_size 200] [--rounds 3] [--precision bf16x3]

The pair folder is written to a temporary directory (validate_throughput.write_pairs) and removed afterwards.
"""
import argparse, importlib, json, os, subprocess, sys, tempfile, time
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.dirname(__file__))
PKG = 'iros20-6d-pose-tracking_b200'
from validate_throughput import write_pairs          # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--pairs', type=int, default=1000)
    ap.add_argument('--batch_size', type=int, default=200)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--precision', default='bf16x3')
    args = ap.parse_args()
    pkg = importlib.import_module(PKG)
    D, P, E = (importlib.import_module(PKG + '.' + m) for m in ('datasets', 'problems', 'engine'))
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    mean, std = pkg.synth.default_mean_std()
    info = {'resolution': 176, 'camera': {'focalX': 1066.778, 'focalY': 1067.487, 'centerX': 312.9869, 'centerY': 241.3109}}
    sds = [pkg.synth.make_state_dict(s) for s in range(4)]
    with tempfile.TemporaryDirectory() as d:
        write_pairs(d, args.pairs)
        ds = D.TrackDataset(d, 'val', mean, std, dataset_info=info, trans_normalizer=0.02, rot_normalizer=15 * np.pi / 180)
        eng = E.Engine(max_batch=args.batch_size)
        models = []
        for i, sd in enumerate(sds):
            models.append(pkg.Se3TrackNet(engine=eng, weight_id=i))
            models[-1].load_state_dict(sd)
        stats = [(mean, std)] * len(models)

        def one_pass(n):
            return P.evaluate(models[:n], ds, args.batch_size, False, [args.precision], stats=stats[:n])

        def separate(n):
            return {(i, args.precision): P.evaluate(models[i], ds, args.batch_size, precision=args.precision) for i in range(n)}

        for n in (1, 2, 4):
            one_pass(n); separate(n)                          # warm: graphs captured, files in the page cache
            times = {'one_pass': [], 'separate': []}
            for _ in range(args.rounds):
                for name, fn in (('one_pass', one_pass), ('separate', separate)):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    fn(n)
                    torch.cuda.synchronize()
                    times[name].append(time.perf_counter() - t0)
            print(json.dumps(dict(checkpoints=n, pairs=args.pairs, batch_size=args.batch_size, precision=args.precision,
                                  one_pass_s=[round(min(times['one_pass']), 3), round(max(times['one_pass']), 3)],
                                  separate_s=[round(min(times['separate']), 3), round(max(times['separate']), 3)],
                                  gpu=gpu, cpus=os.cpu_count())))
        eng.close()


if __name__ == '__main__':
    main()
