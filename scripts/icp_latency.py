"""Per-frame cost of the depth refinement through Tracker.on_track_batch (device route, bf16x3, fit check on): M = 0 / 1 / 3 / 5
ICP iterations at n = 1, 8 and 64 tracks that sit on their objects: the 480 x 640 depth frame is drawn at 8 poses
(oracle/icp_ref.py synthetic_scene), the tracks start 5-10 mm and 2-5 degrees off them (repeated to n), and the head outputs 0,
so every iteration associates and solves as on a track that follows its object.  Prints the card's name and power limit read in the same run,
then one JSON line per (n, M) with the mean ms per frame over `--frames` frames after `--warmup`.

    python scripts/icp_latency.py [--frames 200] [--warmup 20]"""
import argparse, importlib, json, os, subprocess, sys, tempfile
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import icp_ref  # noqa: E402
PKG = 'iros20-6d-pose-tracking_b200'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=20)
    args = ap.parse_args()
    print(subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip())
    pkg = importlib.import_module(PKG)
    synth, mio = pkg.synth, importlib.import_module(PKG + '.mesh_io')
    K = synth.CAMERA_K
    path = os.path.join(tempfile.mkdtemp(), 'model.ply')
    mesh, _, starts, depth = icp_ref.synthetic_scene(synth, 8)
    mio.save_ply_mesh(path, mesh)
    sd = synth.make_state_dict(0)
    for k in ('trans_out.0.weight', 'trans_out.0.bias', 'rot_out.0.weight', 'rot_out.0.bias'):
        sd[k] = torch.zeros_like(sd[k])
    info = {'resolution': 176, 'object_width': 200.0, 'boundingbox': 10,
            'camera': {'focalX': K[0, 0], 'focalY': K[1, 1], 'centerX': K[0, 2], 'centerY': K[1, 2], 'height': 480, 'width': 640}}
    mean, std = synth.default_mean_std()
    engine = pkg.Engine(max_batch=64)
    rgb = synth.raw_frame(0)[0]
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    R, D = dev(rgb), dev(depth)
    for n in (1, 8, 64):
        P0 = dev(np.concatenate([starts] * ((n + 7) // 8))[:n])
        for M in (0, 1, 3, 5):
            t = pkg.Tracker(info, mean, std, {'state_dict': sd}, model_path=path, renderer='cuda', engine=engine,
                            fit=10, icp=M or None)
            P = P0.clone()
            for _ in range(args.warmup):
                t.on_track_batch(P0, R, D)
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.frames):
                P = t.on_track_batch(P0, R, D)
            b.record()
            torch.cuda.synchronize()
            print(json.dumps({'n': n, 'icp_iterations': M, 'ms_per_frame': a.elapsed_time(b) / args.frames,
                              'launches': engine.last_launch_count(),
                              'mean_inliers': None if t.last_icp is None else float(t.last_icp[:, 0].mean())}))
    engine.close()


if __name__ == '__main__':
    main()
