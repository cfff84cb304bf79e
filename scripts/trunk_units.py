"""Per-unit timeline of the trunk launch at a small batch (SE3TN_TRACE=1): for every layer, when its units' dependencies were met, when
their MMAs ran and when their epilogues finished, and the fraction of SM time with an MMA group in flight (per layer: inside the
window from the layer's first MMA to its last epilogue; whole launch: from the first CTA's entry to the last CTA's exit).
   python scripts/trunk_units.py [precision] [n]"""
import importlib, os, sys
os.environ['SE3TN_TRACE'] = '1'; os.environ['SE3TN_GRAPH'] = '0'
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
pkg = importlib.import_module('iros20-6d-pose-tracking_b200'); synth = pkg.synth
prec = sys.argv[1] if len(sys.argv) > 1 else 'bf16x3'
nb = int(sys.argv[2]) if len(sys.argv) > 2 else 1
eng = pkg.Engine(max_batch=max(nb, 4)); eng.load_state_dict(synth.make_state_dict(0), 0)
A, B = synth.tensor_pairs(nb, seed=1); A = A.cuda(); B = B.cuda()
for _ in range(4): eng.forward(A, B, precision=prec)
torch.cuda.synchronize()
tr = eng.get_trace().astype(np.int64)
trunk = tr[8]                               # per-CTA stamps of the trunk launch
live = trunk[:, 0] > 0
t0 = trunk[live, 0].min()
t_end = (trunk[live, 7] & ~0xff).max()
n_cta = int(live.sum())
units = tr[9:14].reshape(-1)[:2048 * 5].reshape(2048, 5)
used = units[:, 4] > 0
idx = np.nonzero(used)[0]
cta = units[:, 4] & 0xff                    # the epilogue-done stamp carries the CTA index in its low 8 bits
units = units.copy(); units[:, 4] &= ~0xff


def busy(lo, hi):
    """SM time with an MMA group in flight inside [lo, hi], summed over the CTAs: union of the [first A unit, last MMA] intervals."""
    tot = 0
    for b in range(n_cta):
        iv = sorted((max(s, lo), min(e, hi)) for s, e in units[idx[cta[idx] == b]][:, 1:3] if min(e, hi) > max(s, lo))
        cur_s = cur_e = None
        for s, e in iv:
            if cur_e is None or s > cur_e:
                if cur_e is not None: tot += cur_e - cur_s
                cur_s, cur_e = s, e
            else:
                cur_e = max(cur_e, e)
        if cur_e is not None: tot += cur_e - cur_s
    return tot


print('%s n=%d: %d work units on %d CTAs; times in us from the first trunk CTA entry' % (prec, nb, len(idx), n_cta))
# layer boundaries: infer from unit counts (n * units_per_image * ksplit per layer) -- print in groups of equal size
per_layer = len(idx) // 6
for l in range(6):
    u = units[idx[l * per_layer:(l + 1) * per_layer]]
    f = lambda a: '%7.1f..%7.1f' % ((a.min() - t0) / 1e3, (a.max() - t0) / 1e3)
    lo, hi = u[:, 1].min(), u[:, 4].max()
    print('layer %d: dep met %s | first A %s | last MMA commit %s | acc seen %s | epilogue done %s | mma %.1f us, epi %.1f us (medians) | mma busy %.3f' % (
        l, f(u[:, 0]), f(u[:, 1]), f(u[:, 2]), f(u[:, 3]), f(u[:, 4]), np.median(u[:, 2] - u[:, 1]) / 1e3, np.median(u[:, 4] - u[:, 3]) / 1e3,
        busy(lo, hi) / (n_cta * (hi - lo))))
print('whole launch: %.1f us, mma busy %.3f' % ((t_end - t0) / 1e3, busy(t0, t_end) / (n_cta * (t_end - t0))))
