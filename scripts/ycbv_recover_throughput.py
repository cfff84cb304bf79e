"""Pose recovery on perturbed YCB-Video key frames (predict.recoverYcbKeyframes), on the synthetic layout of
perturbed_validate_throughput.build_layout (480 x 640 key frames, its classes, one checkpoint each):

  * rounds in one step: one pass at K = 4, every frame one se3tn_track_render step that records rounds 1..4;
  * separate steps: the passes at K = 1, 2, 3 and 4, the 1 + 2 + 3 + 4 = 10 rounds per frame a sweep of K costs without the
    round output.

The two alternate `--rounds` times in one process; the script checks that round k of the K = 4 pass equals the K = k pass bit for
bit and prints key frames/s and scored rows/s as one JSON line (also to `--out`), with the card's name and power limit read in the
same run.

    python scripts/ycbv_recover_throughput.py [--frames 100] [--num_sample 10] [--rounds 2] [--precision bf16x3] [--out FILE]
"""
import argparse, importlib, json, os, subprocess, sys, tempfile, time
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.dirname(__file__))
PKG = 'iros20-6d-pose-tracking_b200'
from perturbed_validate_throughput import build_layout, CLASSES, H, W          # noqa: E402

KMAX = 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=100)
    ap.add_argument('--num_sample', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--precision', default='bf16x3')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    pkg = importlib.import_module(PKG)
    P = importlib.import_module(PKG + '.predict')
    mesh_io = importlib.import_module(PKG + '.mesh_io')
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    m = args.precision
    with tempfile.TemporaryDirectory() as root:
        tpl = build_layout(root, pkg.synth, mesh_io, args.frames)
        tpl = dict(tpl, pair_model_path=tpl['model_path'])
        ycb = os.path.join(root, 'ycb')

        def run(k):
            return P.recoverYcbKeyframes(ycb, CLASSES, tpl, num_sample=args.num_sample, seed=args.seed, precision=m, iterations=k)[m, k]

        routes = (('rounds_in_one_step', lambda: {KMAX: run(KMAX)}), ('separate_steps', lambda: {k: run(k) for k in range(1, KMAX + 1)}))
        times = {name: [] for name, _ in routes}
        results = {}
        for _ in range(args.rounds):
            for name, fn in routes:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                results[name] = fn()
                torch.cuda.synchronize()
                times[name].append(time.perf_counter() - t0)
    one, sep = results['rounds_in_one_step'][KMAX], results['separate_steps']
    identical = all(np.array_equal(one[c]['poses'][k - 1], sep[k][c]['poses'][k - 1]) for c in CLASSES for k in range(1, KMAX + 1))
    rows = one['all']['rows']
    frames = args.frames
    out = dict(gpu=gpu, frames=frames, frame_hw=[H, W], classes=len(CLASSES), num_sample=args.num_sample, precision=m, K=KMAX,
               scored_rows=rows, identical=identical,
               add_auc_by_round=[one['all']['summary'][r]['add_auc'] for r in range(KMAX + 1)])
    for name, ts in times.items():
        out[name] = dict(seconds=[round(t, 3) for t in ts], keyframes_per_s=[round(frames / t, 2) for t in ts],
                         rows_per_s=[round(rows / t, 1) for t in ts])
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')
    if not identical:
        raise SystemExit('round k of the K = %d pass differs from the K = k pass' % KMAX)


if __name__ == '__main__':
    main()
