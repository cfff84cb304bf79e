"""Small augmented validation steps for compute-sanitizer (memcheck / racecheck): se3tn_eval_pairs_augmented with every stage
taken (captured and replayed as a graph, with segB and without, into context scratch and into caller outputs), then
se3tn_augment_draws with the noise fields and se3tn_augment_crops.

    compute-sanitizer --tool memcheck python scripts/sanitize_augment.py
    compute-sanitizer --tool racecheck python scripts/sanitize_augment.py
"""
import importlib, os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
pkg = importlib.import_module('iros20-6d-pose-tracking_b200'); synth = pkg.synth
n = 3
eng = pkg.Engine(max_batch=4)
mean, std = synth.default_mean_std()
eng.load_state_dict(synth.make_state_dict(0), 0); eng.set_stats(mean, std, 0)
TN, RN = 0.02, 15 * np.pi / 180
B = synth.raw_poses(n, seed=0)
A = B.copy(); A[:, :3, 3] += 0.01
rng = np.random.default_rng(0)
rgbB = rng.integers(0, 256, (n, 176, 176, 3), dtype=np.uint8)
rgbA, depA = synth.rendered_views(n, A, seed=0)
depB = rng.integers(0, 2000, (n, 176, 176)).astype(np.uint16)
seg = (depB > 500).astype(np.uint8)
t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
args = (t(rgbA), t(depA), t(rgbB), t(depB), t(A), t(B), TN, RN)
cfg = eng.augment_config(seed=1, hsv=dict(h=15, s=15, v=15, prob=1.0), bright=dict(lo=0.5, hi=1.5), noise=dict(rgb=2, depth=5, prob=1.0),
                         blur=dict(max_kernel=6, prob=1.0), cover=dict(prob=1.0))
idx = torch.arange(n, dtype=torch.int64, device='cuda')
out_r, out_d = torch.empty_like(args[2]), torch.empty_like(args[3])
tot = 0.0
for s in (t(seg), None):
    for outs in ({}, dict(out_rgbB=out_r, out_depthB=out_d)):
        for rep in range(2):                                   # the second call replays the captured graph
            sums = eng.eval_pairs(*args, precision='bf16x3', augment=cfg, segB=s, pair_index=idx, **outs)[2]
            tot += float(sums.sum())
params, nr, nd = eng.augment_draws(cfg, args[3], idx, segB=t(seg), want_noise=True)
r, d = eng.augment_crops(cfg, args[2], args[3], idx, segB=t(seg))
torch.cuda.synchronize()
print('ok', tot, float(params.sum()), int(r.sum()))
eng.close()
