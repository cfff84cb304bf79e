"""Cost per frame of re-initialising lost tracks through Tracker.on_track_batch (device route: CUDA poses, numpy frame), 8
objects of one synthetic 480 x 640 frame (oracle/init_ref.py labelled_scene) tracked with a checkpoint whose head outputs zero,
so poses stay where they are put.  Rows: re-initialisation off (the fit check on at the same tau, so the step is the same);
on with nothing lost (the loss check and its one synchronisation); on with 1, 4 or 8 tracks restarted every frame at the init
defaults (those tracks are fed 0.3 m off their objects; below 0.1, after 1).  Prints the card's name and power limit read in the same
run, then one JSON line per row: mean ms per frame over `--frames` frames after `--warmup`, wall clock to a synchronisation.
Then the same rows through the one-pass loop of the YCB-Video driver (one_pass), per frame over the whole sequence, decoding
and first-frame graph captures included.

    python scripts/reinit_latency.py [--frames 50] [--warmup 5]"""
import argparse, importlib, json, os, subprocess, sys, tempfile, time
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import init_ref  # noqa: E402
PKG = 'iros20-6d-pose-tracking_b200'
N = 8


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    print(subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip())
    pkg = importlib.import_module(PKG)
    synth = pkg.synth
    K = synth.CAMERA_K
    mesh, gts, _, depth, seg = init_ref.labelled_scene(synth, N, seed=0)
    info = {'resolution': 176, 'boundingbox': 10, 'object_width': 200.0,
            'camera': {'focalX': K[0, 0], 'focalY': K[1, 1], 'centerX': K[0, 2], 'centerY': K[1, 2], 'height': 480, 'width': 640}}
    mean, std = synth.default_mean_std()
    sd = synth.make_state_dict(0)
    for k in ('trans_out.0.weight', 'trans_out.0.bias', 'rot_out.0.weight', 'rot_out.0.bias'):
        sd[k] = torch.zeros_like(sd[k])
    rgb = np.zeros((480, 640, 3), np.uint8)
    labels = list(range(1, N + 1))
    tau = importlib.import_module(PKG + '.predict').FIT_TAU_DEFAULT
    path = os.path.join(tempfile.mkdtemp(), 'model.ply')
    importlib.import_module(PKG + '.mesh_io').save_ply_mesh(path, mesh)
    # below 0.1: the scene's objects at the edge of the frame fit well above it, and a track fed off its object fits nothing
    for name, reinit, lost in (('off', None, 0), ('on, none lost', dict(below=0.1, after=1), 0),
                               ('on, 1 restarted', dict(below=0.1, after=1), 1), ('on, 4 restarted', dict(below=0.1, after=1), 4),
                               ('on, 8 restarted', dict(below=0.1, after=1), 8)):
        trk = pkg.Tracker(info, mean, std, {'state_dict': sd}, model_path=path, renderer='cuda', max_batch=N, fit=tau, reinit=reinit,
                          engine=pkg.Engine(max_batch=N * 8))
        start = gts.copy()
        start[:lost, 0, 3] += 0.3
        start = torch.from_numpy(start).cuda()
        poses = start.clone()                            # one input buffer: the step's graph is replayed frame after frame
        kw = {} if reinit is None else dict(seg=seg, labels=labels)
        for f in range(args.warmup + args.frames):
            if f == args.warmup:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
            poses.copy_(start)
            trk.on_track_batch(poses, rgb, depth, **kw)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1000 / args.frames
        ev = None if trk.last_reinit is None else trk.last_reinit.cpu().numpy().tolist()
        print(json.dumps({'route': 'on_track_batch', 'row': name, 'n': N, 'ms_per_frame': round(ms, 3), 'last_events': ev}))
        trk.engine.close()
    one_pass(pkg, mesh, gts, depth, seg, info, mean, std, sd, path, tau, args)


def one_pass(pkg, mesh, gts, depth, seg, info, mean, std, sd, path, tau, args):
    """The same rows through the YCB-Video one-pass loop (predict._track_sequences, the frames decoded from PNG files through
    its ring): one sequence of warmup + frames frames, the 8 objects under weight ids (= labels) 1..8.  The tracks start where
    they are put and the restarted ones 0.3 m off.  The loop carries the poses from frame to frame, so those are restarted in
    the first frame and then stay where the start put them: these rows measure the loop with the check on, one restart per
    displaced track, and the decoding of every frame's three PNG files, which bounds the loop here."""
    import cv2
    pr = importlib.import_module(PKG + '.predict')
    d = tempfile.mkdtemp()
    frames = args.warmup + args.frames
    rgb_files, depth_files, seg_files = [], [], []
    for t in range(frames):
        rgb_files.append(os.path.join(d, '%06d-color.png' % t)); cv2.imwrite(rgb_files[-1], np.zeros((480, 640, 3), np.uint8))
        depth_files.append(os.path.join(d, '%06d-depth.png' % t)); cv2.imwrite(depth_files[-1], depth)
        seg_files.append(os.path.join(d, '%06d-label.png' % t)); cv2.imwrite(seg_files[-1], seg)
    ids = tuple(range(1, N + 1))
    for name, reinit, lost in (('off', None, 0), ('on, none lost', dict(below=0.1, after=1), 0),
                               ('on, 1 restarted', dict(below=0.1, after=1), 1), ('on, 8 restarted', dict(below=0.1, after=1), 8)):
        opts = pr.step_options(fit=tau, reinit=reinit)
        eng = pkg.Engine(max_batch=N * pr.reinit_keep(opts))
        trackers = {w: pkg.Tracker(info, mean, std, {'state_dict': sd}, model_path=path, renderer='cuda', engine=eng, weight_id=w)
                    for w in ids}
        start = gts.copy()
        start[:lost, 0, 3] += 0.3
        seq = (rgb_files, depth_files, ids, start) + (() if reinit is None else (seg_files,))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = next(pr._track_sequences(eng, trackers, [seq], (('bf16x3', 1),), 2, 2, None, opts, [0]))
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1000 / frames
        ev = None if reinit is None else res[2][('bf16x3', 1)][-1].tolist()
        print(json.dumps({'route': 'one-pass loop', 'row': name, 'n': N, 'ms_per_frame': round(ms, 3), 'frames': frames,
                          'last_events': ev}))
        eng.close()


if __name__ == '__main__':
    main()
