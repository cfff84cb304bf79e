"""Small validation steps for compute-sanitizer (memcheck / racecheck): se3tn_eval_pairs in a tensor-core mode (captured and
replayed as a graph, with and without the optional outputs, two weight sets in one step), in the fp32 mode (FFMA forwards and the
stand-alone loss launch) and se3tn_pair_loss.

    compute-sanitizer --tool memcheck python scripts/sanitize_eval_pairs.py
    compute-sanitizer --tool racecheck python scripts/sanitize_eval_pairs.py
"""
import importlib, os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
pkg = importlib.import_module('iros20-6d-pose-tracking_b200'); synth = pkg.synth
n = 3
eng = pkg.Engine(max_batch=4)
mean, std = synth.default_mean_std()
for w in (0, 1):
    eng.load_state_dict(synth.make_state_dict(w), w); eng.set_stats(mean, std, w)
TN, RN = 0.02, 15 * np.pi / 180
B = synth.raw_poses(n, seed=0)
A = B.copy(); A[:, :3, 3] += 0.01
rgbB = np.random.default_rng(0).integers(0, 256, (n, 176, 176, 3), dtype=np.uint8)
rgbA, depA = synth.rendered_views(n, A, seed=0)
depB = depA[::-1].copy()
t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
args = (t(rgbA), t(depA), t(rgbB), t(depB), t(A), t(B), TN, RN)
tot = 0.0
for prec in ('bf16x3', 'fp32'):
    for ids in (None, np.array([0, 1, 0], np.int32)):
        for rep in range(2):                                   # the second tensor-core call replays the captured graph
            tr, ro, sums, sq, lab = eng.eval_pairs(*args, weight_ids_host=ids, precision=prec, want_terms=rep == 0, want_labels=rep == 0)
            tot += float(sums.sum())
s2 = eng.pair_loss(tr, ro, t(np.zeros((n, 3))), t(np.ones((n, 3))))
torch.cuda.synchronize()
print('ok', tot, float(s2.sum()))
eng.close()
