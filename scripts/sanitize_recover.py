"""One pose-recovery step with the round output and one se3tn_pose_errors_sets call with a keep mask, for compute-sanitizer
(memcheck / racecheck): k = 3 rounds recorded by se3tn_track_render's round_poses in a graph (bf16x3) and as plain launches (fp32).

    compute-sanitizer --tool memcheck python scripts/sanitize_recover.py
"""
import importlib, os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
pkg = importlib.import_module('iros20-6d-pose-tracking_b200'); synth = pkg.synth
n, k = 3, 3
eng = pkg.Engine(max_batch=4)
mean, std = synth.default_mean_std()
eng.load_state_dict(synth.make_state_dict(0), 0); eng.set_stats(mean, std, 0)
mesh = synth.mesh(1, seed=0)
eng.set_mesh(mesh, 0)
TN, RN = 0.03, 5 * np.pi / 180
rgb, depth = synth.raw_frame(0, h=120, w=160)
K = synth.CAMERA_K.copy(); K[:2] /= 4
P = torch.from_numpy(synth.raw_poses(n, seed=0)).cuda(); ow = torch.full((n,), 200.0, dtype=torch.float64, device='cuda')
R, D = torch.from_numpy(rgb).cuda(), torch.from_numpy(depth).cuda()
rounds = torch.empty((k, n, 4, 4), dtype=torch.float64, device='cuda')
for prec in ('bf16x3', 'fp32'):
    out, _, _ = eng.track_render(R, D, K, P, ow, TN, RN, precision=prec, iterations=k, out_rounds=rounds)
keep = torch.tensor([1, 0, 1], dtype=torch.uint8, device='cuda')
errs, sets = eng.pose_errors_sets([mesh['pos'].astype(np.float64)], np.zeros(n, np.int32), rounds[k - 1], P, keep=keep)
torch.cuda.synchronize()
print('ok', float(out.abs().sum()), errs.cpu().numpy().tolist(), sets.cpu().numpy().tolist())
eng.close()
