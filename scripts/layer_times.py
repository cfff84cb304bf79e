"""Per-layer conv times (ms) for a precision and batch size.   python scripts/layer_times.py [precision] [n]"""
import importlib, os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
pkg = importlib.import_module('iros20-6d-pose-tracking_b200'); synth = pkg.synth
prec = sys.argv[1] if len(sys.argv) > 1 else 'bf16x3'
nb = int(sys.argv[2]) if len(sys.argv) > 2 else 64
eng = pkg.Engine(max_batch=nb); eng.load_state_dict(synth.make_state_dict(0), 0)
A, B = synth.tensor_pairs(nb, seed=1); A = A.cuda(); B = B.cuda()
for _ in range(3): eng.forward(A, B, precision=prec)
eng.set_profiling(True); acc = []
for _ in range(10):
    eng.forward(A, B, precision=prec); acc.append(eng.get_profile())
m = np.mean(np.stack(acc), 0)
print('%s n=%d: conv %s sum %.4f' % (prec, nb, ' '.join('%.4f' % x for x in m[:14]), m[:14].sum()))
