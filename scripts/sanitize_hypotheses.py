"""Small hypothesis steps for compute-sanitizer (memcheck / racecheck): the expansion alone, S = 1 and 4 hypotheses at k = 1 and 3
inside track_hypotheses, with and without the depth fill, in a graph and as plain launches (fp32), a window over the frame's edge,
and through track_hypotheses_host.

    compute-sanitizer --tool memcheck python scripts/sanitize_hypotheses.py
    compute-sanitizer --tool racecheck python scripts/sanitize_hypotheses.py
"""
import importlib, os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
pkg = importlib.import_module('iros20-6d-pose-tracking_b200'); synth = pkg.synth
n, S = 3, 4
eng = pkg.Engine(max_batch=n * S)
mean, std = synth.default_mean_std()
eng.load_state_dict(synth.make_state_dict(0), 0); eng.set_stats(mean, std, 0)
eng.set_mesh(synth.mesh(1, seed=0), 0)
TN, RN = 0.03, 5 * np.pi / 180
SPREAD = dict(max_translation=0.02, max_rotation_deg=15.0)
rgb, depth = synth.raw_frame(0, h=120, w=160)
K = synth.CAMERA_K.copy(); K[:2] /= 4                               # the same field of view on a 120 x 160 frame
poses = synth.raw_poses(n, seed=0)
poses[0, :3, 3] = (0.3, -0.19, 0.5)                                 # a window over the frame's edge
P = torch.from_numpy(poses).cuda(); ow = torch.full((n,), 200.0, dtype=torch.float64, device='cuda')
R, D = torch.from_numpy(rgb).cuda(), torch.from_numpy(depth).cuda()
keys = torch.arange(n, dtype=torch.int64, device='cuda') + 77
starts, draws = eng.draw_hypotheses(P, keys, S, want_draws=True, **SPREAD)
for fill in (False, True):
    for prec in ('bf16x3', 'fp32'):
        for hyps in (1, S):
            for k in (1, 3):
                hp = torch.empty(n, hyps, 4, 4, dtype=torch.float64, device='cuda')
                rounds = torch.empty(k, n, hyps, 4, 4, dtype=torch.float64, device='cuda')
                out = eng.track_hypotheses(R, D, K, P, ow, TN, RN, keys, hyps, fit=10, precision=prec, fill_depth=fill, iterations=k,
                                           out_hyp_poses=hp, out_rounds=rounds, **SPREAD)
host = eng.track_hypotheses_host(rgb, depth, K, poses, ow.cpu().numpy(), TN, RN, keys.cpu().numpy(), S, fit=10, iterations=3, **SPREAD)
torch.cuda.synchronize()
print('ok', out[1].cpu().numpy().tolist(), host[1].tolist())
eng.close()
