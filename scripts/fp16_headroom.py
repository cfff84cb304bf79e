"""Headroom of the 'fp16' mode: the largest stored |activation| of every conv output buffer on the test inputs (tensor-regime
pairs, the raw-regime frame of 64 tracks on weight seeds 0 / 1, config 1), against fp16's largest value 65504, which the
saturating encode relies on; and the fraction of the synthetic sets' fp16-held conv weights (layers 2-13) that fall in
fp16's subnormal range (|w| < 2^-14) or flush to zero.  Run from the repo root on the GPU:

    python scripts/fp16_headroom.py
"""
import importlib, json, os, sys
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import layer_ref as R
PKG = 'iros20-6d-pose-tracking_b200'
BUFS = ['P1A', 'P1B', 'T1', 'T2', 'U', 'CAT', 'F1', 'T4', 'F2', 'H1', 'H2']


def stored_max(eng, n):
    out = {}
    for b in BUFS:
        nb = R.floats_per_image(b) * 2
        u = eng.debug_buffer(R.BUF_ID[b], eng.max_batch).view(torch.uint8).reshape(-1)[:n * nb]
        out[b] = float(u.view(torch.float16).float().abs().max())
    return out


def main():
    pkg = importlib.import_module(PKG)
    synth = pkg.synth
    weights = importlib.import_module(PKG + '.weights')
    eng = pkg.Engine(max_batch=64)
    mean, std = synth.default_mean_std()
    for w in (0, 1):
        eng.load_state_dict(synth.make_state_dict(w), w)
    eng.set_stats(mean, std, 0); eng.set_stats(mean + 1.5, std * 1.25, 1)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(eng.device)
    res = {}
    A, B = synth.tensor_pairs(64, seed=2)
    eng.forward(t(A), t(B), precision='fp16'); torch.cuda.synchronize()
    res['tensor regime, 64 pairs'] = stored_max(eng, 64)
    n = 64
    rgb, depth = synth.raw_frame(11); poses = synth.raw_poses(n, seed=11); rgbA, depthA = synth.rendered_views(n, poses, seed=11)
    wid = np.repeat(np.array([0, 1], np.int32), n // 2)
    eng.track_batch(t(rgb), t(depth), synth.CAMERA_K, t(poses), t(np.full(n, 200.0)), t(rgbA), t(depthA), 0.03, 5 * np.pi / 180,
                    weight_ids_host=wid, weight_ids_dev=t(wid), precision='fp16'); torch.cuda.synchronize()
    res['raw regime, 64 tracks, sets 0/1'] = stored_max(eng, 64)
    import cv2
    g = os.path.join(ROOT, 'tests', 'golden')
    ra = cv2.imread(os.path.join(g, 'c1_rgbA.png'))[..., ::-1].copy(); rb = cv2.imread(os.path.join(g, 'c1_rgbB.png'))[..., ::-1].copy()
    tA, tB = eng.normalize(t(ra[None]), t(synth.depth_from_rgb(ra)[None]), t(rb[None]), t(synth.depth_from_rgb(rb)[None]),
                           t(synth.config1_pose()[None]), precision='fp16')
    eng.forward(tA, tB, precision='fp16'); torch.cuda.synchronize()
    res['config 1'] = stored_max(eng, 1)
    eng.close()
    w_off, _, _ = R.blob_offsets()
    sub = {}
    for s in (0, 1):
        blob = weights.pack_state_dict(synth.make_state_dict(s))
        w = np.concatenate([R.layer_weights(blob, li)[0].ravel() for li in range(2, 14)]).astype(np.float32)
        a = np.abs(w)
        sub['set %d' % s] = {'weights': int(w.size), 'subnormal': float(((a < 2.0 ** -14) & (a >= 2.0 ** -25)).mean()),
                             'to_zero': float(((a < 2.0 ** -25) & (a > 0)).mean()), 'max_abs': float(a.max())}
    res['fp16 weights (layers 2-13)'] = sub
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
