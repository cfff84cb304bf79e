"""Tracking pairs/s of the precision modes on the full track_batch path (preprocess, conv stack, head and pose update in one
captured step per frame), at 64 and 256 tracks.  The modes (default 'bf16', 'fp8', 'bf16x3') alternate `--rounds` times in
one process; the pairs/s ranges, the trunk launch's device time (conv_trunk_kernel) and every launch's time (the profile
slots of include/se3tn.h, from the last profiled step of each mode) are printed with the card's name and power limit, read
in the same run.

    python scripts/fp8_throughput.py [--rounds 4] [--steps 50] [--modes bf16x3 tf32 bf16 fp16 fp8]

Synthetic weights and a synthetic raw-regime frame: the rates do not depend on the values (no data-dependent work on the path).
"""
import argparse, importlib, json, os, subprocess, sys, time
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
PKG = 'iros20-6d-pose-tracking_b200'
MODES = ['bf16', 'fp8', 'bf16x3']
TRUNK_SLOT = 8                                           # include/se3tn.h profile slot of the trunk launch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=4)
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--tracks', type=int, nargs='+', default=[64, 256])
    ap.add_argument('--modes', nargs='+', default=MODES)
    args = ap.parse_args()
    modes = args.modes
    pkg = importlib.import_module(PKG)
    synth = pkg.synth
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    eng = pkg.Engine(max_batch=max(args.tracks))
    eng.load_state_dict(synth.make_state_dict(0), 0)
    mean, std = synth.default_mean_std()
    eng.set_stats(mean, std, 0)
    dev = eng.device
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    res = {'gpu': gpu, 'torch_device': torch.cuda.get_device_name(0), 'steps': args.steps, 'rounds': args.rounds, 'modes': modes, 'tracks': {}}
    for n in args.tracks:
        rgb, depth = synth.raw_frame(3)
        poses = synth.raw_poses(n, seed=3)
        rgbA, depthA = synth.rendered_views(n, poses, seed=3)
        targs = (t(rgb), t(depth), synth.CAMERA_K, t(poses), t(np.full(n, 200.0)), t(rgbA), t(depthA), 0.03, 5 * np.pi / 180)
        a, b, _, _ = eng.preprocess(*targs[:7], want_tensors=True)
        if 'fp8' in modes:
            eng.calibrate_fp8(a, b, weight_id=0)
        outs = dict(out_poses=torch.empty_like(targs[3]), out_trans=torch.empty(n, 3, device=dev), out_rot=torch.empty(n, 3, device=dev))

        def run(prec, steps):
            for _ in range(steps):
                eng.track_batch(*targs, precision=prec, **outs)

        for m in modes:                                  # warm-up: each mode's step graph captured
            run(m, 3)
        torch.cuda.synchronize()
        rates = {m: [] for m in modes}
        trunk_ms = {m: [] for m in modes}
        slots_ms = {}
        for _ in range(args.rounds):
            for m in modes:
                torch.cuda.synchronize(); t0 = time.perf_counter()
                run(m, args.steps)
                torch.cuda.synchronize()
                rates[m].append(n * args.steps / (time.perf_counter() - t0))
            for m in modes:                              # one profiled step (plain launches) per mode for the launch times
                eng.set_profiling(True)
                run(m, 1)
                prof = [float(x) for x in eng.get_profile()]
                trunk_ms[m].append(prof[TRUNK_SLOT])
                slots_ms[m] = [round(x, 4) for x in prof]
                eng.set_profiling(False)
        res['tracks'][n] = {'pairs_per_s': {m: [round(min(v), 1), round(max(v), 1)] for m, v in rates.items()},
                            'pairs_per_s_rounds': {m: [round(x, 1) for x in v] for m, v in rates.items()},
                            'trunk_ms': {m: [round(min(v), 3), round(max(v), 3)] for m, v in trunk_ms.items()},
                            'slot_ms': slots_ms}
    eng.close()
    print('card (name, power limit, max SM clock): %s' % gpu)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
