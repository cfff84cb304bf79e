"""Small filled tracking steps for compute-sanitizer (memcheck / racecheck): every fill branch inside track_batch and
track_render, in a graph and without one, and both host entry points, which upload the whole depth frame.

    compute-sanitizer --tool memcheck python scripts/sanitize_fill_track.py
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
K = synth.CAMERA_K
TN, RN = 0.03, 5 * np.pi / 180
rgb, depth = synth.raw_frame(0, h=120, w=160)
K = K.copy(); K[:2] /= 4                                         # the same field of view on a 120 x 160 frame
poses = synth.raw_poses(n, seed=0)
P = torch.from_numpy(poses).cuda(); ow = torch.full((n,), 200.0, dtype=torch.float64, device='cuda')
R, D = torch.from_numpy(rgb).cuda(), torch.from_numpy(depth).cuda()
rgbA, depA = eng.render(K, P, ow)
for fill in (True, dict(extrapolate=True), dict(blur_type='gaussian'), dict(extrapolate=True, blur_type='gaussian', max_depth=1.5)):
    for prec in ('bf16x3', 'fp32'):
        out, _, _ = eng.track_batch(R, D, K, P, ow, rgbA, depA, TN, RN, precision=prec, fill_depth=fill)
        eng.track_render(R, D, K, P, ow, TN, RN, precision=prec, fill_depth=fill)
host = eng.track_host(rgb, depth, K, poses, ow.cpu().numpy(), rgbA.cpu().numpy(), depA.cpu().numpy(), TN, RN, fill_depth=True)
host_r = eng.track_render_host(rgb, depth, K, poses, ow.cpu().numpy(), TN, RN, fill_depth=True)
torch.cuda.synchronize()
print('ok', float(out.abs().sum()), float(np.abs(host).sum()), float(np.abs(host_r).sum()))
eng.close()
