"""Small re-initialisation calls for compute-sanitizer (memcheck / racecheck): se3tn_lost_tracks over n = 1, 3 and 1100 tracks
(more than one scan tile), se3tn_fit_poses in both render modes with a pose whose window runs over the frame's edge and one
with a NaN entry, se3tn_accept_starts with a failed start, and Engine.reinit on a 120 x 160 frame with one track lost.

    compute-sanitizer --tool memcheck python scripts/sanitize_reinit.py
"""
import importlib, os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
pkg = importlib.import_module('iros20-6d-pose-tracking_b200'); synth = pkg.synth
eng = pkg.Engine(max_batch=1100)
eng.set_mesh(synth.mesh(1, seed=0), 0)
_, depth = synth.raw_frame(0, h=120, w=160)
K = synth.CAMERA_K.copy(); K[:2] /= 4                               # the same field of view on a 120 x 160 frame
D = torch.from_numpy(depth).cuda()
for n in (1, 3, 1100):
    rows = torch.randint(0, 50, (n, 6), dtype=torch.int32, device='cuda')
    streak = torch.zeros(n, dtype=torch.int32, device='cuda')
    for _ in range(3):
        event, lost = eng.lost_tracks(rows, streak, 0.5, 2)
P = torch.eye(4, dtype=torch.float64, device='cuda').repeat(3, 1, 1).contiguous()
P[:, 2, 3] = 0.6
P[1, 0, 3] = 0.25                                                   # over the frame's right edge
P[2, 1, 3] = float('nan')
ow = torch.full((3,), 200.0, dtype=torch.float64, device='cuda')
for mode in ('vispy', 'pyrender'):
    rows = eng.fit_poses(D, K, P, ow, 10, mode=mode, image_hw=(120, 160) if mode == 'pyrender' else None)
init_rows = torch.zeros(2, 8, dtype=torch.int32, device='cuda'); init_rows[1, 0] = 1
streak, event = torch.zeros(3, dtype=torch.int32, device='cuda'), torch.zeros(3, dtype=torch.int32, device='cuda')
eng.accept_starts([2, 0], P[:2].clone(), init_rows, rows[:2].clone(), P, rows, streak, event)
seg = np.zeros((120, 160), np.uint8); seg[40:80, 60:100] = 1
fit = torch.zeros(1, 6, dtype=torch.int32, device='cuda')           # model 0: below, lost at after = 1
ev = eng.reinit(D, seg, K, [1], ow[:1], P[:1].clone(), fit, torch.zeros(1, dtype=torch.int32, device='cuda'), 10, 0.5, 1,
                init=dict(viewpoints=3, inplane=2, keep=2, min_pixels=10, icp=2))
torch.cuda.synchronize()
print('ok', ev.cpu().numpy().tolist(), event.cpu().numpy().tolist())
eng.close()
