"""Small start-pose calls for compute-sanitizer (memcheck / racecheck): se3tn_init_poses on a 120 x 160 frame with three objects
(one whose mask runs over the frame's edge, one without depth under its mask, one label absent), both render modes, with and
without ICP, several chunks per call (max_batch 4), and every optional output; then se3tn_init_boxes on the same frame with
overlapping boxes, a box on the frame's corner, one without depth and an empty one, at D = 1 and 3.

    compute-sanitizer --tool memcheck python scripts/sanitize_init.py
"""
import importlib, os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
pkg = importlib.import_module('iros20-6d-pose-tracking_b200'); synth = pkg.synth
eng = pkg.Engine(max_batch=4)
eng.set_mesh(synth.mesh(1, seed=0), 0)
_, depth = synth.raw_frame(0, h=120, w=160)
K = synth.CAMERA_K.copy(); K[:2] /= 4                               # the same field of view on a 120 x 160 frame
seg = np.zeros((120, 160), np.uint8)
seg[40:80, 60:100] = 1
seg[0:30, 140:160] = 2                                              # over the frame's edge
seg[90:110, 10:30] = 3
depth[90:110, 10:30] = 0                                            # label 3 has no depth; label 4 has no pixels
D, S = torch.from_numpy(depth).cuda(), torch.from_numpy(seg).cuda()
n = 2
ow = torch.full((n,), 200.0, dtype=torch.float64, device='cuda')
for mode in ('vispy', 'pyrender'):
    for icp in (None, 2):
        for labels in ([1, 2], [3, 4]):
            init = dict(viewpoints=3, inplane=2, keep=2, min_pixels=10, icp=icp)
            out = dict(stats=torch.empty(n, 6, dtype=torch.int64, device='cuda'), t0=torch.empty(n, 3, dtype=torch.float64, device='cuda'),
                       cand_rows=torch.empty(n, 6, 8, dtype=torch.int32, device='cuda'),
                       kept_rows=torch.empty(n, 2, 8, dtype=torch.int32, device='cuda'),
                       kept_poses=torch.empty(n, 2, 4, 4, dtype=torch.float64, device='cuda'))
            if icp:
                out.update(icp_poses=torch.empty(n, 2, 4, 4, dtype=torch.float64, device='cuda'),
                           icp_rows=torch.empty(n, 2, 8, dtype=torch.int32, device='cuda'),
                           icp_stats=torch.empty(n, 2, 4, dtype=torch.float64, device='cuda'))
            P, R = eng.init_poses(D, S, K, labels, ow, mode=mode, image_hw=(120, 160) if mode == 'pyrender' else None, init=init, out=out)
boxes = np.array([[50, 30, 110, 90], [60, 40, 100, 80], [130, 0, 160, 30], [10, 90, 30, 110], [5, 5, 5, 50]], np.int32)
for mode in ('vispy', 'pyrender'):
    for icp in (None, 2):
        for sel, nd in (([0, 1], 1), ([2, 3], 3), ([4, 0], 3)):          # overlapping; corner and no depth; empty
            init = dict(viewpoints=3, inplane=2, keep=2, min_pixels=10, icp=icp)
            out = dict(stats=torch.empty(n, 6, dtype=torch.int64, device='cuda'), t0=torch.empty(n, nd, 3, dtype=torch.float64, device='cuda'),
                       cand_rows=torch.empty(n, 6 * nd, 8, dtype=torch.int32, device='cuda'),
                       kept_rows=torch.empty(n, 2, 8, dtype=torch.int32, device='cuda'),
                       kept_poses=torch.empty(n, 2, 4, 4, dtype=torch.float64, device='cuda'))
            if icp:
                out.update(icp_poses=torch.empty(n, 2, 4, 4, dtype=torch.float64, device='cuda'),
                           icp_rows=torch.empty(n, 2, 8, dtype=torch.int32, device='cuda'),
                           icp_stats=torch.empty(n, 2, 4, dtype=torch.float64, device='cuda'))
            Pb, Rb = eng.init_boxes(D, boxes[sel], K, ow, mode=mode, image_hw=(120, 160) if mode == 'pyrender' else None, init=init,
                                    depths=nd, out=out)
torch.cuda.synchronize()
print('ok', R.cpu().numpy().tolist(), Rb.cpu().numpy().tolist())
eng.close()
