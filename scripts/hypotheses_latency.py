"""Per-frame time of multi-hypothesis tracking (Tracker(hypotheses=S)), bf16x3, S in {1, 4, 8, 16} x n in {1, 8} tracks x k in {1, 2}
refinement rounds, through Tracker.on_track_batch on numpy inputs (the host route: one synchronous se3tn_track_render_host
call per frame, with opts->hyp for S > 1; S = 1 is the plain step with the fit check).  For each (n, k) the Trackers of every S
share one Engine and alternate frame by frame in one process, so all see the same card state.  The card's name and power limit
are printed first: the numbers belong to them.

    python scripts/hypotheses_latency.py [--frames 200] [--out result.json]
"""
import argparse, importlib, json, os, sys, tempfile, time
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))
pkg = importlib.import_module('iros20-6d-pose-tracking_b200')
synth, mio = pkg.synth, importlib.import_module('iros20-6d-pose-tracking_b200.mesh_io')
from refine_latency import card  # noqa: E402

HYPOTHESES = (1, 4, 8, 16)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=200)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'hypotheses_latency measures on a CUDA device'
    print('device: %s' % card(), flush=True)
    path = os.path.join(tempfile.mkdtemp(), 'model.ply')
    mio.save_ply_mesh(path, synth.mesh(3, seed=1))                  # 20,480 faces
    K = synth.CAMERA_K
    info = {'resolution': 176, 'object_width': 200.0, 'boundingbox': 10, 'max_translation': 0.02, 'max_rotation': 15,
            'camera': {'focalX': K[0, 0], 'focalY': K[1, 1], 'centerX': K[0, 2], 'centerY': K[1, 2], 'height': 480, 'width': 640}}
    mean, std = synth.default_mean_std()
    rgb, depth = synth.raw_frame(0)
    eng = pkg.Engine(max_batch=8 * max(HYPOTHESES))
    rows = []
    for n in (1, 8):
        start = synth.raw_poses(n, seed=n)
        for k in (1, 2):
            trk = {S: pkg.Tracker(info, mean, std, {'state_dict': synth.make_state_dict(0)}, model_path=path, renderer='cuda',
                                  engine=eng, precision='bf16x3', iterations=k, fit=10, hypotheses=S) for S in HYPOTHESES}
            for _ in range(10):                                     # warm-up: capture and first launches of every step
                for t in trk.values():
                    t.on_track_batch(start, rgb, depth)
            ms = {S: 0.0 for S in trk}
            for _ in range(args.frames):                            # alternate: each call ends in a synchronise
                for S, t in trk.items():
                    t0 = time.perf_counter()
                    t.on_track_batch(start, rgb, depth)
                    ms[S] += (time.perf_counter() - t0) * 1e3
            for S in HYPOTHESES:
                row = dict(precision='bf16x3', n=n, k=k, S=S, ms=ms[S] / args.frames)
                rows.append(row)
                print('n=%d k=%d S=%2d  %.3f ms per frame' % (n, k, S, row['ms']), flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(dict(device=card(), frames=args.frames, rows=rows), f, indent=1)
    eng.close()


if __name__ == '__main__':
    main()
