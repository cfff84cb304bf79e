#!/usr/bin/env python
"""Generate tests/golden/golden_augment.npz by running THE REFERENCE'S OWN train-time augmentations (data_augmentation.py) on
seeded crops with recorded draws.

  python oracle/make_golden_augment.py --ref <checkout of the reference tree>

train.py:85-92's chain -- HSVJitter(15, 15, 15), ChangeBright(mag=[0.5, 1.5]), GaussianNoise(2, 5), GaussianBlur(6),
BlackCover(prob=0.2) -- is imported from the reference unmodified (make_golden.py's stubs) and applied in that order, with
np.random.uniform / normal / randint / choice and random.uniform replaced by a player of recorded draws.  The player also checks
that the reference asks for exactly the draws each case expects, in order, so the fixture pins the chain's order and branch
structure as well as its arithmetic.  Branch tests are answered with prob / 2 (taken) or (1 + prob) / 2 (not taken); GaussianNoise's
fields are standard normals from np.random.default_rng(noise seed) times the std; BlackCover's corners come from each case's list,
as many as the reference's loop asks for.  depthB enters BlackCover as an array that stores a Python int the way numpy 1.x does
(-9999 -> 55537), where numpy 2 raises.

Stored per case: the draws in se3tn_augment_draws' layout (cover fields other than the branch left 0), the corner list, the corners
the reference used, the seeds, and the reference's rgbB / depthB / maskB.  The inputs are regenerated from their seeds by
augment_ref.case_inputs.
"""
import argparse, os, random

import numpy as np

import augment_ref as R
from make_golden import ROOT, import_reference

H_NOISE, BRIGHT_MAG, RGB_NOISE, DEPTH_NOISE, BLUR_MAX, PROB, BLUR_PROB, COVER_PROB = 15, (0.5, 1.5), 2, 5, 6, 0.5, 0.4, 0.2
SEG_KINDS = ('seg', 'none', 'two')

# seed, maskB kind, hsv branches / magnitudes, bright factor, (rgb noise branch, std), (depth noise branch, std), noise seed,
# (rgb blur branch, k), (depth blur branch, k), cover branch, corners
CASES = [
    (1, 'seg', (1, 1, 1), (7.25, -13.9, 4.1), 1.21, (1, 1.7), (1, 4.6), 11, (1, 3), (1, 5), 1, [(90, 80, 1)]),
    (2, 'none', (1, 0, 1), (-14.6, 0.0, 9.9), 0.63, (1, 1.95), (0, 0.0), 12, (0, 0), (1, 7), 1, [(170, 170, 0)]),
    (3, 'two', (0, 1, 0), (0.0, 12.5, 0.0), 1.49, (0, 0.0), (1, 4.9), 13, (1, 7), (0, 0), 1, 'center_then_far'),
    (4, 'seg', (0, 0, 0), (0.0, 0.0, 0.0), 1.37, (0, 0.0), (0, 0.0), 14, (0, 0), (0, 0), 0, []),
    (5, 'none', (1, 1, 0), (3.3, -2.2, 0.0), 0.51, (1, 0.4), (1, 4.99), 15, (1, 5), (1, 3), 1, [(0, 0, 3)]),
    (6, 'seg', (0, 0, 1), (0.0, 0.0, -15.0), 1.0, (1, 2.0), (1, 0.01), 16, (1, 7), (1, 7), 1, 'center_then_far'),
]


def corners_of(spec, mask):
    if spec != 'center_then_far':
        return list(spec)
    ys, xs = np.nonzero(mask == 1)
    return [(int(xs.mean()), int(ys.mean()), 2), (3, 4, 0)]


class Player:
    """Answers the reference's np.random / random calls from a list of (name, args, value), then BlackCover's corners."""
    def __init__(self, calls, corners):
        self.calls, self.corners, self.used, self.pending = list(calls), list(corners), 0, []

    def __call__(self, name, *args):
        if self.calls:
            want, want_args, value = self.calls.pop(0)
            assert (want, want_args) == (name, args), 'the reference asked for %s%s, the case expects %s%s' % (name, args, want, want_args)
            return value
        if name == 'randint' and args == (0, 176):
            if not self.pending:
                u, v, q = self.corners[self.used]
                self.used += 1
                self.pending = [v, q]
                return u
            return self.pending.pop(0)
        assert name == 'choice' and args == ((0, 1, 2, 3),) and len(self.pending) == 1, (name, args)
        return self.pending.pop(0)


class Numpy1Store(np.ndarray):
    """Stores a Python int as numpy 1.x did, wrapping it into the dtype (BlackCover's -9999 into uint16 -> 55537)."""
    def __setitem__(self, key, value):
        if isinstance(value, int):
            value = np.array(value, dtype=np.int64).astype(self.dtype)
        super().__setitem__(key, value)


def run_case(DA, case):
    seed, kind, hb, hm, bright, (nrb, nrs), (ndb, nds), nseed, (brb, brk), (bdb, bdk), cb, cspec = case
    rgbB, depthB, maskB, rgbA = R.case_inputs(seed, kind)
    corners = corners_of(cspec, maskB)
    rng = np.random.default_rng(nseed)
    noise_rgb = rng.standard_normal((176, 176, 3)) * nrs
    noise_depth = rng.standard_normal((176, 176)) * nds
    t = lambda taken, prob: prob / 2 if taken else (1 + prob) / 2
    calls = []
    for c in range(3):
        calls.append(('uniform', (), t(hb[c], PROB)))
        if hb[c]:
            calls.append(('uniform', (-H_NOISE, H_NOISE), hm[c]))
    calls.append(('random.uniform', BRIGHT_MAG, bright))
    for taken, std, lim, field in ((nrb, nrs, RGB_NOISE, noise_rgb), (ndb, nds, DEPTH_NOISE, noise_depth)):
        calls.append(('uniform', (), t(taken, PROB)))
        if taken:
            calls += [('uniform', (0, lim), std), ('normal', (0, std, field.shape), field)]
    for taken, k in ((brb, brk), (bdb, bdk)):
        calls.append(('uniform', (), t(taken, BLUR_PROB)))
        if taken:
            calls.append(('randint', (1, BLUR_MAX // 2 + 1), (k - 1) // 2))
    calls.append(('uniform', (0, 1), t(cb, COVER_PROB)))
    play = Player(calls, corners)

    saved = {k: getattr(np.random, k) for k in ('uniform', 'normal', 'randint', 'choice')}
    saved_random = random.uniform
    np.random.uniform = lambda *a: play('uniform', *a)
    np.random.normal = lambda loc, scale, size: play('normal', loc, scale, tuple(size))
    np.random.randint = lambda lo, hi: play('randint', lo, hi)
    np.random.choice = lambda a: play('choice', tuple(a))
    random.uniform = lambda a, b: play('random.uniform', a, b)
    try:
        chain = [DA.HSVJitter(H_NOISE, H_NOISE, H_NOISE), DA.ChangeBright(prob=0.5, mag=list(BRIGHT_MAG)),
                 DA.GaussianNoise(RGB_NOISE, DEPTH_NOISE), DA.GaussianBlur(BLUR_MAX), DA.BlackCover(prob=COVER_PROB)]
        data = (rgbA, np.zeros((176, 176), np.uint16), rgbB.copy(), depthB.copy(), np.zeros((176, 176), np.uint8), maskB.copy(), np.eye(4))
        for tr in chain:
            if isinstance(tr, DA.BlackCover):
                d = list(data)
                d[3] = np.ascontiguousarray(d[3]).view(Numpy1Store)
                data = tuple(d)
            data = tr(data)
    finally:
        for k, f in saved.items():
            setattr(np.random, k, f)
        random.uniform = saved_random
    assert not play.calls, 'the reference did not ask for %s' % (play.calls,)
    p = np.zeros(R.N_PARAMS)
    p[R.HSV_ON] = 1; p[R.HSV_BRANCH:R.HSV_BRANCH + 3] = hb; p[R.HSV_MAG:R.HSV_MAG + 3] = [m if b else 0 for b, m in zip(hb, hm)]
    p[R.BRIGHT_ON] = 1; p[R.BRIGHT] = bright
    p[R.NOISE_RGB_BRANCH], p[R.NOISE_RGB_STD], p[R.NOISE_DEPTH_BRANCH], p[R.NOISE_DEPTH_STD] = nrb, nrs, ndb, nds
    p[R.BLUR_RGB_BRANCH], p[R.BLUR_RGB_K], p[R.BLUR_DEPTH_BRANCH], p[R.BLUR_DEPTH_K] = brb, brk, bdb, bdk
    p[R.COVER_BRANCH] = cb
    out = [np.asarray(x) for x in data[2:4]] + [np.asarray(data[5])]
    return dict(params=p, corners=np.array(corners, np.int64).reshape(-1, 3), corners_used=np.int64(play.used),
                seed=np.int64(seed), kind=np.int64(SEG_KINDS.index(kind)), noise_seed=np.int64(nseed),
                rgbB=out[0].astype(np.uint8), depthB=out[1].astype(np.uint16), maskB=out[2].astype(np.uint8))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--ref', required=True, help='a checkout of the reference tree (its data_augmentation.py is imported)')
    ap.add_argument('--out', default=os.path.join(ROOT, 'tests', 'golden', 'golden_augment.npz'))
    args = ap.parse_args()
    DA = import_reference(args.ref)[1]
    g = {'n_cases': np.int64(len(CASES))}
    for i, case in enumerate(CASES):
        for k, v in run_case(DA, case).items():
            g['%s_%d' % (k, i)] = v
    np.savez_compressed(args.out, **g)
    print(args.out, os.path.getsize(args.out))


if __name__ == '__main__':
    main()
