"""Time per se3tn_init_poses call (Engine.init_poses) with Engine.init_spec's defaults (300 x 24 candidates, 8 kept, 5 ICP
iterations) at n = 1, 8 and 21 objects of one synthetic 480 x 640 frame (oracle/init_ref.py labelled_scene), on contexts of
max_batch 64 and 168: the candidates are drawn in chunks of max_batch rows, so max_batch sets the number of launches.  Prints
the card's name and power limit read in the same run, then one JSON line per (max_batch, n) with the mean ms per call over
`--calls` calls after `--warmup`, with and without ICP.  Then the same for se3tn_init_boxes (Engine.init_boxes, the tight box of
each object's label) at D = 1 and D = 4 depth candidates, D x 7,200 candidates per object.

    python scripts/init_latency.py [--calls 5] [--warmup 1]"""
import argparse, importlib, itertools, json, os, subprocess, sys
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import init_box_ref  # noqa: E402
import init_ref  # noqa: E402
PKG = 'iros20-6d-pose-tracking_b200'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--calls', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=1)
    args = ap.parse_args()
    print(subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip())
    pkg = importlib.import_module(PKG)
    synth = pkg.synth
    K = synth.CAMERA_K
    mesh, _, _, depth, seg = init_ref.labelled_scene(synth, 21, seed=0)
    boxes = np.stack([init_box_ref.tight_box(seg, k) for k in range(1, 22)])
    for mb in (64, 168):
        e = pkg.Engine(max_batch=mb)
        e.set_mesh(mesh, 0)
        D, S = torch.from_numpy(depth).cuda(), torch.from_numpy(seg).cuda()
        for n in (1, 8, 21):
            if n * 8 > mb:
                continue
            ow = torch.full((n,), 200.0, dtype=torch.float64, device='cuda')
            calls = [('mask', lambda init: e.init_poses(D, S, K, list(range(1, n + 1)), ow, init=init))]
            calls += [('box D=%d' % d, lambda init, d=d: e.init_boxes(D, boxes[:n], K, ow, init=init, depths=d)) for d in (1, 4)]
            for (start, call), icp in itertools.product(calls, (5, 0)):
                init = dict(icp=icp)
                for _ in range(args.warmup):
                    call(init)
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(args.calls):
                    _, rows = call(init)
                b.record()
                torch.cuda.synchronize()
                print(json.dumps({'start': start, 'max_batch': mb, 'n': n, 'icp_iterations': icp, 'ms_per_call': a.elapsed_time(b) / args.calls,
                                  'launches': e.last_launch_count(), 'failed': int((rows[:, 0] != 0).sum())}))
        e.close()


if __name__ == '__main__':
    main()
