"""Per-frame latency of k refinement rounds (Tracker(iterations=k)) against k separate tracking calls per frame, for k = 1..4 at
n = 1 and n = 64 tracks, in bf16x3 and fp8.  Both cases go through Tracker.on_track_batch on numpy inputs (the host route: one
synchronous se3tn_track_render_host call per step, the reference's calling pattern):

    fused     one Tracker(iterations=k) call per frame: k rounds inside one step and one CUDA graph
    separate  k calls of a Tracker(iterations=1) per frame, each from the poses the previous call returned

Both give the same poses bit for bit (tests/test_gpu_refine.py); only the time differs.  The card's name and power limit are
printed first: the numbers belong to them.

    python scripts/refine_latency.py [--frames 200] [--out result.json]
"""
import argparse, importlib, json, os, subprocess, sys, time
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module('iros20-6d-pose-tracking_b200')
synth, mio = pkg.synth, importlib.import_module('iros20-6d-pose-tracking_b200.mesh_io')


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[torch.cuda.current_device()]
        return q
    except Exception as e:                                          # the name alone, and why the power limit is missing
        return '%s, power limit unknown (%s)' % (torch.cuda.get_device_name(), e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=200)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'refine_latency measures on a CUDA device'
    print('device: %s' % card(), flush=True)
    import tempfile
    tmp = tempfile.mkdtemp()
    path = os.path.join(tmp, 'model.ply')
    mio.save_ply_mesh(path, synth.mesh(3, seed=1))                  # 20,480 faces
    K = synth.CAMERA_K
    info = {'resolution': 176, 'object_width': 200.0, 'boundingbox': 10,
            'camera': {'focalX': K[0, 0], 'focalY': K[1, 1], 'centerX': K[0, 2], 'centerY': K[1, 2], 'height': 480, 'width': 640}}
    mean, std = synth.default_mean_std()
    rgb, depth = synth.raw_frame(0)
    rows = []
    for prec in ('bf16x3', 'fp8'):
        eng = pkg.Engine(max_batch=64)
        make = lambda k: pkg.Tracker(info, mean, std, {'state_dict': synth.make_state_dict(0)}, model_path=path, renderer='cuda',
                                     engine=eng, precision=prec, iterations=k)
        single = make(1)
        for n in (1, 64):
            start = synth.raw_poses(n, seed=n)
            for k in range(1, 5):
                fused = make(k)

                def run_fused(p):
                    return fused.on_track_batch(p, rgb, depth)

                def run_separate(p):
                    for _ in range(k):
                        p = single.on_track_batch(p, rgb, depth)
                    return p
                res = {}
                for name, fn in (('fused', run_fused), ('separate', run_separate)):
                    p = start
                    for _ in range(10):                             # warm-up: calibration, capture, first launches
                        p = fn(start)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    p = start
                    for _ in range(args.frames):                    # each call returns numpy poses: it ends in a synchronise
                        p = fn(start)
                    res[name] = (time.perf_counter() - t0) * 1e3 / args.frames
                    res[name + '_poses'] = p
                assert np.array_equal(res['fused_poses'], res['separate_poses'])
                row = dict(precision=prec, n=n, k=k, fused_ms=res['fused'], separate_ms=res['separate'])
                rows.append(row)
                print('%-6s n=%-2d k=%d  one %d-round step %7.3f ms/frame   %d separate calls %7.3f ms/frame' %
                      (prec, n, k, k, row['fused_ms'], k, row['separate_ms']), flush=True)
        eng.close()
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(dict(device=card(), frames=args.frames, rows=rows), f, indent=1)


if __name__ == '__main__':
    main()
