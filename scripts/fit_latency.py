"""Per-frame time of a tracking step with and without the fit check (Tracker(fit=tau)), bf16x3, n = 1 and 64 tracks, k = 1 and 4
refinement rounds, through Tracker.on_track_batch on numpy inputs (the host route: one synchronous se3tn_track_render_host call
per frame).  The two Trackers share one Engine and alternate frame by frame in one process, so both see the same card state.
The fit check leaves the poses bit for bit unchanged (tests/test_gpu_fit.py); this checks it again on every timed frame.  The
card's name and power limit are printed first: the numbers belong to them.

    python scripts/fit_latency.py [--frames 200] [--tau 10] [--out result.json]
"""
import argparse, importlib, json, os, sys, tempfile, time
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))
pkg = importlib.import_module('iros20-6d-pose-tracking_b200')
synth, mio = pkg.synth, importlib.import_module('iros20-6d-pose-tracking_b200.mesh_io')
from refine_latency import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=200)
    ap.add_argument('--tau', type=int, default=10)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'fit_latency measures on a CUDA device'
    print('device: %s' % card(), flush=True)
    path = os.path.join(tempfile.mkdtemp(), 'model.ply')
    mio.save_ply_mesh(path, synth.mesh(3, seed=1))                  # 20,480 faces
    K = synth.CAMERA_K
    info = {'resolution': 176, 'object_width': 200.0, 'boundingbox': 10,
            'camera': {'focalX': K[0, 0], 'focalY': K[1, 1], 'centerX': K[0, 2], 'centerY': K[1, 2], 'height': 480, 'width': 640}}
    mean, std = synth.default_mean_std()
    rgb, depth = synth.raw_frame(0)
    eng = pkg.Engine(max_batch=64)
    rows = []
    for n in (1, 64):
        start = synth.raw_poses(n, seed=n)
        for k in (1, 4):
            trk = {fit: pkg.Tracker(info, mean, std, {'state_dict': synth.make_state_dict(0)}, model_path=path, renderer='cuda',
                                    engine=eng, precision='bf16x3', iterations=k, fit=fit) for fit in (None, args.tau)}
            for _ in range(10):                                     # warm-up: capture and first launches of both steps
                for t in trk.values():
                    t.on_track_batch(start, rgb, depth)
            ms = {fit: 0.0 for fit in trk}
            for _ in range(args.frames):                            # alternate: each call ends in a synchronise
                got = {}
                for fit, t in trk.items():
                    t0 = time.perf_counter()
                    got[fit] = t.on_track_batch(start, rgb, depth)
                    ms[fit] += (time.perf_counter() - t0) * 1e3
                assert np.array_equal(got[None], got[args.tau])
            row = dict(precision='bf16x3', n=n, k=k, tau=args.tau, off_ms=ms[None] / args.frames, on_ms=ms[args.tau] / args.frames)
            rows.append(row)
            print('n=%2d k=%d  fit off %.3f ms  fit on %.3f ms  (+%.3f ms per frame)' % (n, k, row['off_ms'], row['on_ms'],
                                                                                         row['on_ms'] - row['off_ms']), flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(dict(device=card(), frames=args.frames, rows=rows), f, indent=1)
    eng.close()


if __name__ == '__main__':
    main()
