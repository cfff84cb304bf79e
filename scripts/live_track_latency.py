"""Per-frame cost of hole-filling a live sensor's depth inside the tracking step, against the reference ROS node's sequence.

One object, one 480 x 640 raw depth frame per call (numpy in, numpy out), input A rendered inside the step in both:
  ros   depth = (Utils.fill_depth(raw / 1e3, max_depth=2.0) * 1000).astype(uint16); Tracker.on_track(p, rgb, depth)
        (fill: pageable upload of the raw frame, 8 launches, 1.2 MB of float32 metres back, a host multiply and cast; then
        on_track uploads the crop window of the filled frame)
  step  Tracker(fill_depth=True).on_track(p, rgb, raw)  (se3tn_track_render_host: the raw frame goes up once, the fill runs
        inside the step's graph)
Wall clock per frame over --frames frames after warm-up, the two alternated --rounds times in one process.
Then 64 tracks per step on device tensors, pairs/s: Engine.fill_depth + Engine.track_render against Engine.track_render with
fill_depth=True, with a device synchronise at the end of each window.  Every track is tracked from the same previous pose in
every frame, so both variants do the same work each time.

    python scripts/live_track_latency.py [--level 5] [--frames 300] [--steps 200] [--rounds 4]
"""
import argparse, importlib, os, subprocess, sys, tempfile, time
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
pkg = importlib.import_module('iros20-6d-pose-tracking_b200'); synth = pkg.synth
mio = importlib.import_module('iros20-6d-pose-tracking_b200.mesh_io')
U = importlib.import_module('iros20-6d-pose-tracking_b200.Utils')

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
    ros = pkg.Tracker(info, mean, std, {'state_dict': synth.make_state_dict(0)}, model_path=ply, max_batch=64)
    live = pkg.Tracker(info, mean, std, {'state_dict': synth.make_state_dict(0)}, model_path=ply, engine=ros.engine, fill_depth=True)
U.set_engine(ros.engine)
rgb, raw = synth.raw_frame(0)
raw[raw > 2000] = 0                                             # no negative filled metres: numpy's cast of those to uint16 is undefined
raw[220:260, 300:340] = 0                                       # a hole in the object's window
p = np.eye(4); p[:3, 3] = (0.02, -0.01, 0.6)


def ros_frame():
    depth = (U.fill_depth(raw / 1e3, max_depth=2.0) * 1000).astype(np.uint16)
    return ros.on_track(p, rgb, depth)


def step_frame():
    return live.on_track(p, rgb, raw)


assert np.array_equal(ros_frame(), step_frame()), 'the two sequences must give the same pose'
med = {'ros': [], 'step': []}
for r in range(args.rounds):
    for name, fn in (('ros', ros_frame), ('step', step_frame)):
        for _ in range(30):
            fn()
        t = np.empty(args.frames)
        for i in range(args.frames):
            t0 = time.perf_counter(); fn(); t[i] = time.perf_counter() - t0
        med[name].append(np.median(t) * 1e3)
        print('round %d %-4s one object: median %.3f ms per frame (min %.3f, max %.3f over %d frames)'
              % (r, name, med[name][-1], t.min() * 1e3, t.max() * 1e3, args.frames))
for name, label in (('ros', 'Utils.fill_depth -> cast -> on_track'), ('step', 'on_track(raw), fill inside the step ')):
    print('one object, %s: median per frame %.3f ms, range of the %d round medians %.3f-%.3f ms'
          % (label, float(np.median(med[name])), args.rounds, min(med[name]), max(med[name])))

# ---- 64 tracks per step, device tensors ----
eng, dev, n = ros.engine, ros.engine.device, 64
R, D = torch.from_numpy(rgb).to(dev), torch.from_numpy(raw).to(dev)
P = torch.from_numpy(synth.raw_poses(n, seed=1)).to(dev)
ow = torch.full((n,), 200.0, dtype=torch.float64, device=dev)
outs = {v: dict(out_poses=torch.empty_like(P), out_trans=torch.empty(n, 3, device=dev), out_rot=torch.empty(n, 3, device=dev)) for v in ('ros', 'step')}
filled = torch.empty_like(D)


def ros_step():
    filled.copy_(eng.fill_depth(D))
    eng.track_render(R, filled, K, P, ow, TN, RN, **outs['ros'])


def fill_step():
    eng.track_render(R, D, K, P, ow, TN, RN, fill_depth=True, **outs['step'])


ros_step(); fill_step(); torch.cuda.synchronize()
assert torch.equal(outs['ros']['out_poses'], outs['step']['out_poses']), 'the two steps must give the same poses'
rate = {'ros': [], 'step': []}
for r in range(args.rounds):
    for name, fn in (('ros', ros_step), ('step', fill_step)):
        for _ in range(20):
            fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.steps):
            fn()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        rate[name].append(n * args.steps / dt)
        print('round %d %-4s %d tracks: %.0f pairs/s (%.3f ms per step)' % (r, name, n, rate[name][-1], dt / args.steps * 1e3))
for name, label in (('ros', 'fill_depth + track_render     '), ('step', 'track_render(fill_depth=True)')):
    print('%d tracks, %s: %.0f-%.0f pairs/s over %d rounds' % (n, label, min(rate[name]), max(rate[name]), args.rounds))
eng.close()
