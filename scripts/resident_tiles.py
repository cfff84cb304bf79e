"""Per-tile timeline of the 8 resident-weight conv launches (SE3TN_TRACE=1): for each launch, the median MMA time and epilogue
time of a tile, the gap from a tile's epilogue end to the first MMA of the CTA's next tile (negative: the next tile's MMAs
started under this epilogue), and the fraction of SM time with an MMA group in flight (union over a CTA's tiles of [first A
unit, last MMA completed], inside the window from the launch's first CTA entry to its last CTA exit).
   python scripts/resident_tiles.py [precision] [n]"""
import importlib, os, sys
os.environ['SE3TN_TRACE'] = '1'; os.environ['SE3TN_GRAPH'] = '0'
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
pkg = importlib.import_module('iros20-6d-pose-tracking_b200'); synth = pkg.synth
prec = sys.argv[1] if len(sys.argv) > 1 else 'bf16x3'
nb = int(sys.argv[2]) if len(sys.argv) > 2 else 64
eng = pkg.Engine(max_batch=max(nb, 4)); eng.load_state_dict(synth.make_state_dict(0), 0)
A, B = synth.tensor_pairs(nb, seed=1); A = A.cuda(); B = B.cuda()
for _ in range(4): eng.forward(A, B, precision=prec)
torch.cuda.synchronize()
cta_tr = eng.get_trace().astype(np.int64)
tile_tr = eng.get_tile_trace().astype(np.int64)
NAMES = ['convA1 (stem)', 'convB1 (stem)', 'convA2.conv1', 'convA2.conv2', 'convB2.conv1', 'convB2.conv2', 'convB3.conv1', 'convB3.conv2']


def union(iv):
    tot, cur_s, cur_e = 0, None, None
    for s, e in sorted(iv):
        if cur_e is None or s > cur_e:
            if cur_e is not None: tot += cur_e - cur_s
            cur_s, cur_e = s, e
        else:
            cur_e = max(cur_e, e)
    return tot + (cur_e - cur_s if cur_e is not None else 0)


print('%s n=%d; medians per tile in us' % (prec, nb))
print('%-14s %6s %5s %8s %8s %9s %9s %10s' % ('launch', 'tiles', 'CTAs', 'mma', 'epilogue', 'gap', 'launch', 'mma busy'))
for l in range(8):
    ct = cta_tr[l]
    live = ct[:, 0] > 0
    t0, t1 = ct[live, 0].min(), (ct[live, 7] & ~0xff).max()
    t = tile_tr[l]
    used = np.nonzero(t[:, 3] > 0)[0]
    u = t[used].copy()
    cta = u[:, 3] & 0xff
    u[:, 3] &= ~0xff
    mma = np.median(u[:, 1] - u[:, 0]) / 1e3
    epi = np.median(u[:, 3] - u[:, 2]) / 1e3
    gaps, busy = [], 0
    for b in np.unique(cta):
        tb = u[cta == b]                          # a CTA's tiles in tile order (its contiguous range)
        gaps += list(tb[1:, 0] - tb[:-1, 3])
        busy += union([(max(s, t0), min(e, t1)) for s, e in tb[:, 0:2] if min(e, t1) > max(s, t0)])
    n_cta = int(live.sum())
    gap = '%9.2f' % (np.median(gaps) / 1e3) if gaps else '%9s' % '-'
    print('%-14s %6d %5d %8.2f %8.2f %s %9.1f %10.3f' % (NAMES[l], len(used), n_cta, mma, epi, gap, (t1 - t0) / 1e3, busy / (n_cta * (t1 - t0))))
