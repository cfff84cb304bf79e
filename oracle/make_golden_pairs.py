#!/usr/bin/env python
"""Generate tests/golden/golden_pairs.npz by running THE REFERENCE'S OWN pair-generator arithmetic (Utils.py) on seeded inputs.

  python oracle/make_golden_pairs.py --ref <checkout of the reference tree>

Executed from the reference, unmodified, with make_golden.py's stubs (open3d / transformations stubbed, np.float aliased):
  Utils.random_gaussian_magnitude (and through it Utils.random_direction), after random.seed(s); np.random.seed(s)
  Utils.random_direction on its own
  Utils.crop_bbox(color, depth, bbox, size, seg) with windows inside, across and beyond the frame edges
Inputs are regenerated from seeds in the tests; the seg frame, the windows and every output are stored.
"""
import argparse, os, random

import numpy as np

from make_golden import ROOT, import_reference, synth

# (seed, max_T metres, max_R degrees, draws): dataset_info.yml's 0.02 / 20 and two others
RNG_CASES = ((0, 0.02, 20.0, 40), (7, 0.05, 45.0, 40), (123, 0.01, 5.0, 40))


def seg_frame(h, w, seed):
    """A uint8 label image: background 0 and a few rectangles of labels 1..21 (overlapping)."""
    rng = np.random.default_rng(seed)
    seg = np.zeros((h, w), np.uint8)
    for _ in range(12):
        y0, x0 = rng.integers(0, h), rng.integers(0, w)
        seg[y0:y0 + rng.integers(5, h // 2), x0:x0 + rng.integers(5, w // 2)] = rng.integers(1, 22)
    return seg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--ref', required=True, help='a checkout of the reference tree (its Utils.py is imported)')
    ap.add_argument('--out', default=os.path.join(ROOT, 'tests', 'golden', 'golden_pairs.npz'))
    args = ap.parse_args()
    U = import_reference(args.ref)[0]
    g = {}
    for seed, mt, mr, k in RNG_CASES:
        random.seed(seed); np.random.seed(seed)
        g['rgm_%d' % seed] = np.stack([U.random_gaussian_magnitude(mt, mr) for _ in range(k)])
        random.seed(seed)
        g['dir_%d' % seed] = np.stack([U.random_direction() for _ in range(k)])
    g['rng_cases'] = np.array([[s, mt, mr, k] for s, mt, mr, k in RNG_CASES], dtype=np.float64)
    # crop_bbox with seg on a 120 x 160 frame: windows inside, across each edge, larger than the frame, tiny (upsampled)
    rgb, depth = synth.raw_frame(3, 120, 160)
    seg = seg_frame(120, 160, 5)
    boxes = [((10, 20), (90, 100)), ((-30, -25), (40, 50)), ((60, 100), (150, 200)), ((-50, -60), (170, 220)),
             ((50, 70), (57, 79)), ((-5, 150), (30, 190))]
    g['seg'] = seg
    for i, ((t, l), (b, r)) in enumerate(boxes):
        bb = np.array([[t, l], [b, l], [t, r], [b, r]], dtype=np.int32)
        out_rgb, out_depth, out_seg = U.crop_bbox(rgb, depth, bb, (176, 176), seg)
        g['crop_bb_%d' % i] = bb
        g['crop_rgb_%d' % i] = out_rgb; g['crop_depth_%d' % i] = out_depth; g['crop_seg_%d' % i] = out_seg
    g['n_crops'] = np.int64(len(boxes))
    np.savez_compressed(args.out, **g)
    print(args.out, os.path.getsize(args.out))


if __name__ == '__main__':
    main()
