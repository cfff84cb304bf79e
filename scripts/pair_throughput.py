#!/usr/bin/env python
"""Pairs per second of the held-out pair generator (produce_train_pair_data.py) on a 480 x 640 frame and a ~20k-face mesh:

  device   Engine.perturb_pairs alone (bbox + pyrender-mode render + crops, one CUDA graph) at n = 1, 16, 64 samples per step,
           CUDA events around `iters` steps after a warm-up
  e2e      ProducerPurturb.generate with its PNG / npz writes (host draws, one step, thread-pool writes), wall clock
  oracle   the CPU oracle's generate loop (oracle/pairs_oracle.py) over a process pool of every host core

    python scripts/pair_throughput.py [--out results.json] [--iters 50] [--e2e_samples 256] [--oracle_samples 8]
"""
import argparse, importlib, json, os, random, sys, tempfile, time
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'oracle'))
PKG = 'iros20-6d-pose-tracking_b200'
H, W = 480, 640


def setup():
    synth = importlib.import_module(PKG + '.synth')
    K = synth.CAMERA_K
    info = {'resolution': 176, 'object_width': 200.0, 'boundingbox': 10, 'max_translation': 0.02, 'max_rotation': 20.0,
            'camera': {'focalX': float(K[0, 0]), 'focalY': float(K[1, 1]), 'centerX': float(K[0, 2]), 'centerY': float(K[1, 2]),
                       'height': H, 'width': W}}
    mesh = synth.mesh(5, seed=1)                                    # 20480 faces
    B = synth.raw_poses(1, seed=2)[0]; B[:3, 3] = (0.01, -0.02, 0.6)
    rgb, depth = synth.raw_frame(7, H, W)
    return synth, info, mesh, B, rgb, depth


def seg_of(B, K, mesh):
    import se3_oracle as O
    _, d = O.render_full_frame_unlit(B, K, mesh, H, W)
    seg = np.zeros((H, W), np.uint8); seg[d > 0] = 1
    return seg


def oracle_one(args):
    import pairs_oracle as PO
    seed, B, rgb, depth, seg, K32, mesh = args
    random.seed(seed); np.random.seed(seed)
    return len(PO.generate(B, rgb, depth, seg, 1, 1, K32, 200.0, 0.02, 20.0, mesh))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='also write the JSON result to this file (it is always printed)')
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--e2e_samples', type=int, default=256)
    ap.add_argument('--oracle_samples', type=int, default=8)
    args = ap.parse_args()
    import torch
    PP = importlib.import_module(PKG + '.produce_train_pair_data')
    synth, info, mesh, B, rgb, depth = setup()
    K32 = PP._cam_K32(info)
    seg = seg_of(B, K32.astype(np.float64), mesh)
    res = {'gpu': torch.cuda.get_device_name(0), 'frame': [H, W], 'mesh_faces': int(len(mesh['faces'])), 'host_cores': os.cpu_count()}
    try:
        import subprocess
        res['power_limit_and_max_sm_clock'] = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                                                             capture_output=True, text=True).stdout.strip()
    except OSError:
        res['power_limit_and_max_sm_clock'] = 'unknown'
    prod = PP.ProducerPurturb(info, model=mesh, max_batch=64)
    eng = prod.engine
    frame = PP.frame_to_device(eng, rgb, depth, seg)
    random.seed(0); np.random.seed(0)
    draws = [A for A, ok in prod.draw(B, 64) if ok]
    while len(draws) < 64:
        draws.append(draws[len(draws) % 8])
    dev = eng.device
    for n in (1, 16, 64):
        A = torch.from_numpy(np.stack(draws[:n])).to(dev)
        ow = torch.full((n,), 200.0, dtype=torch.float64, device=dev)
        cid = torch.ones(n, dtype=torch.int32, device=dev)
        out = eng.perturb_pairs(*frame, K32, A, ow, cid)
        for _ in range(5):
            eng.perturb_pairs(*frame, K32, A, ow, cid, out=out)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(args.iters):
            eng.perturb_pairs(*frame, K32, A, ow, cid, out=out)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.iters
        res['device_n%d' % n] = {'ms_per_step': ms, 'pairs_per_s': n / ms * 1e3, 'graph': eng.last_step_was_graph()}
    # end to end: generate with its writes, 64 samples per call
    with tempfile.TemporaryDirectory() as tmp:
        random.seed(1); np.random.seed(1)
        prod.generate(tmp + '/', B, rgb, depth, 64, 1, current_seg=seg)        # warm-up
        c0 = prod.count
        t = time.perf_counter()
        for _ in range(max(1, args.e2e_samples // 64)):
            prod.generate(tmp + '/', B, rgb, depth, 64, 1, current_seg=seg)
        dt = time.perf_counter() - t
        written = prod.count - c0
        # the same pairs' PNG encoding alone, on the same thread-pool width
        from PIL import Image
        from concurrent.futures import ThreadPoolExecutor
        imgs = [np.asarray(Image.open(os.path.join(tmp, '%07drgbA.png' % i))) for i in range(min(written, 64))]
        t = time.perf_counter()
        with ThreadPoolExecutor(prod.workers) as pool:
            list(pool.map(lambda im: Image.fromarray(im).save(os.path.join(tmp, 'x%d.png' % id(im)), optimize=True), imgs * 2))
        png_s = (time.perf_counter() - t) / len(imgs)               # two optimize=True rgb PNGs per pair
    res['e2e'] = {'pairs': written, 's': dt, 'pairs_per_s': written / dt, 'write_threads': prod.workers,
                  'rgb_png_optimize_pairs_per_s_alone': 1.0 / png_s}
    # CPU oracle on every host core
    K32c = K32
    jobs = [(s, B, rgb, depth, seg, K32c, mesh) for s in range(args.oracle_samples)]
    t = time.perf_counter()
    with ProcessPoolExecutor(os.cpu_count()) as pool:
        n = sum(pool.map(oracle_one, jobs))
    dt = time.perf_counter() - t
    res['oracle_cpu'] = {'samples': n, 's': dt, 'pairs_per_s': n / dt, 'processes': os.cpu_count()}
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
