"""Small tracking steps with ICP for compute-sanitizer (memcheck / racecheck): M = 1 and 3 inside track_render with and without
the depth fill and the fit check, in a graph and as plain launches (fp32), both render modes, a window over the frame's edge,
and through track_render_host.

    compute-sanitizer --tool memcheck python scripts/sanitize_icp.py
"""
import importlib, os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
pkg = importlib.import_module('iros20-6d-pose-tracking_b200'); synth = pkg.synth
n = 3
eng = pkg.Engine(max_batch=4)
mean, std = synth.default_mean_std()
eng.load_state_dict(synth.make_state_dict(0), 0); eng.set_stats(mean, std, 0)
eng.set_mesh(synth.mesh(1, seed=0), 0)
TN, RN = 0.03, 5 * np.pi / 180
rgb, depth = synth.raw_frame(0, h=120, w=160)
K = synth.CAMERA_K.copy(); K[:2] /= 4                               # the same field of view on a 120 x 160 frame
poses = synth.raw_poses(n, seed=0)
poses[0, :3, 3] = (0.3, -0.19, 0.5)                                 # a window over the frame's edge
P = torch.from_numpy(poses).cuda(); ow = torch.full((n,), 200.0, dtype=torch.float64, device='cuda')
R, D = torch.from_numpy(rgb).cuda(), torch.from_numpy(depth).cuda()
for mode in ('vispy', 'pyrender'):
    for fill in (False, True):
        for prec in ('bf16x3', 'fp32'):
            for M in (1, 3):
                slots = torch.empty(M, n, 4, 4, dtype=torch.float64, device='cuda')
                out = eng.track_render(R, D, K, P, ow, TN, RN, precision=prec, mode=mode, image_hw=(120, 160) if mode == 'pyrender' else None,
                                       fill_depth=fill, fit=10 if fill else None, icp={'iterations': M, 'tau_mm': 200}, out_icp_poses=slots)
host = eng.track_render_host(rgb, depth, K, poses, ow.cpu().numpy(), TN, RN, iterations=2, fit=10, icp=3)
torch.cuda.synchronize()
print('ok', out[-1].cpu().numpy().tolist(), host[-1].tolist())
eng.close()
