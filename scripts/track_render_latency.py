"""Per-frame cost of rendering input A inside the tracking step, against rendering it first and passing it in.

One object, one 480 x 640 frame per call (the reference's calling pattern, numpy in, numpy out):
  old  ra, da = Tracker.render_window(p); Tracker.on_track(p, rgb, depth, rgbA=ra, depthA=da)
       (render, two device -> host copies of input A, then se3tn_track_host uploads it again)
  new  Tracker.on_track(p, rgb, depth)                  (se3tn_track_render_host: one call, input A stays on the device)
Wall clock per frame over 300 frames after warm-up, the two alternated four times in one process.
Then 64 tracks per step on device tensors, pairs/s: Engine.render + Engine.track_batch against Engine.track_render, with a
device synchronise at the end of each window.  Every track is tracked from the same previous pose in every frame, so both
variants do the same work each time.

    python scripts/track_render_latency.py [--level 5] [--frames 300] [--steps 200] [--rounds 4]
"""
import argparse, importlib, os, subprocess, sys, tempfile, time
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
pkg = importlib.import_module('iros20-6d-pose-tracking_b200'); synth = pkg.synth
mio = importlib.import_module('iros20-6d-pose-tracking_b200.mesh_io')

ap = argparse.ArgumentParser()
ap.add_argument('--level', type=int, default=5, help='icosphere subdivisions of the synthetic model: 20 * 4**level faces')
ap.add_argument('--frames', type=int, default=300)
ap.add_argument('--steps', type=int, default=200)
ap.add_argument('--rounds', type=int, default=4)
args = ap.parse_args()

if not torch.cuda.is_available():
    raise SystemExit('needs a CUDA device')
try:
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                         capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    smi = 'nvidia-smi unavailable'
print('device: %s | nvidia-smi name, power limit, max SM clock: %s' % (torch.cuda.get_device_name(), smi))

K = synth.CAMERA_K
TN, RN = 0.03, 5 * np.pi / 180
mesh = synth.mesh(args.level, seed=0)
print('model: %d vertices, %d faces' % (len(mesh['pos']), len(mesh['faces'])))
info = {'resolution': 176, 'boundingbox': 10, 'object_width': 200.0,
        'camera': {'focalX': K[0, 0], 'focalY': K[1, 1], 'centerX': K[0, 2], 'centerY': K[1, 2], 'height': 480, 'width': 640}}
mean, std = synth.default_mean_std()
with tempfile.TemporaryDirectory() as tmp:                      # the Tracker reads the model file only while it is built
    ply = os.path.join(tmp, 'model.ply')
    mio.save_ply_mesh(ply, mesh)
    trk = pkg.Tracker(info, mean, std, {'state_dict': synth.make_state_dict(0)}, model_path=ply, max_batch=64)
rgb, depth = synth.raw_frame(0)
p = np.eye(4); p[:3, 3] = (0.02, -0.01, 0.6)


def old_frame():
    ra, da = trk.render_window(p)
    return trk.on_track(p, rgb, depth, rgbA=ra, depthA=da)


def new_frame():
    return trk.on_track(p, rgb, depth)


assert np.array_equal(old_frame(), new_frame()), 'the two sequences must give the same pose'
med = {'old': [], 'new': []}
for r in range(args.rounds):
    for name, fn in (('old', old_frame), ('new', new_frame)):
        for _ in range(30):
            fn()
        t = np.empty(args.frames)
        for i in range(args.frames):
            t0 = time.perf_counter(); fn(); t[i] = time.perf_counter() - t0
        med[name].append(np.median(t) * 1e3)
        print('round %d %-3s one object: median %.3f ms per frame (min %.3f, max %.3f over %d frames)'
              % (r, name, med[name][-1], t.min() * 1e3, t.max() * 1e3, args.frames))
for name, label in (('old', 'render_window + on_track(rgbA, depthA)'), ('new', 'on_track, render inside the step   ')):
    print('one object, %s: median per frame %.3f ms, range of the %d round medians %.3f-%.3f ms'
          % (label, float(np.median(med[name])), args.rounds, min(med[name]), max(med[name])))

# ---- 64 tracks per step, device tensors ----
eng, dev, n = trk.engine, trk.engine.device, 64
R, D = torch.from_numpy(rgb).to(dev), torch.from_numpy(depth).to(dev)
P = torch.from_numpy(synth.raw_poses(n, seed=1)).to(dev)
ow = torch.full((n,), 200.0, dtype=torch.float64, device=dev)
ra, da = torch.empty(n, 176, 176, 3, dtype=torch.uint8, device=dev), torch.empty(n, 176, 176, dtype=torch.uint16, device=dev)
outs = {v: dict(out_poses=torch.empty_like(P), out_trans=torch.empty(n, 3, device=dev), out_rot=torch.empty(n, 3, device=dev)) for v in ('old', 'new')}


def old_step():
    eng.render(K, P, ow, out_rgb=ra, out_depth=da)
    eng.track_batch(R, D, K, P, ow, ra, da, TN, RN, **outs['old'])


def new_step():
    eng.track_render(R, D, K, P, ow, TN, RN, **outs['new'])


old_step(); new_step(); torch.cuda.synchronize()
assert torch.equal(outs['old']['out_poses'], outs['new']['out_poses']), 'the two steps must give the same poses'
rate = {'old': [], 'new': []}
for r in range(args.rounds):
    for name, fn in (('old', old_step), ('new', new_step)):
        for _ in range(20):
            fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.steps):
            fn()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        rate[name].append(n * args.steps / dt)
        print('round %d %-3s %d tracks: %.0f pairs/s (%.3f ms per step)' % (r, name, n, rate[name][-1], dt / args.steps * 1e3))
for name, label in (('old', 'render + track_batch'), ('new', 'track_render        ')):
    print('%d tracks, %s: %.0f-%.0f pairs/s over %d rounds' % (n, label, min(rate[name]), max(rate[name]), args.rounds))
eng.close()
