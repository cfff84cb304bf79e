"""YCB-Video evaluation throughput: predict.getResultsYcbAll (every class of a test sequence in one step per frame, each frame
decoded once) against the loop of per-class predict.getResultsYcb runs it replaces (one class per run, every frame decoded once
per object, one synchronous n = 1 step per frame), over the same data set.  The two alternate `--rounds` times in one process,
each call timed whole (engine set-up, weight and mesh upload, decoding, tracking, writing the pose files); the card's name and
power limit are read in the same run.

    python scripts/ycb_all_throughput.py [--frames 100] [--rounds 3] [--precision bf16x3] [--video]

--video times three legs instead, alternating in the same way: getResultsYcbAll without videos; with video=True (every track
drawn on the device, written by the video sink); and without videos followed by the reference's own way of making them (the CPU
oracle's cv2 drawing of every track in every frame on the host, encoding on a writer thread), from frames decoded before the
timer starts.  It reports the model point counts drawn.

The data set is written to a temporary directory, seeded, and removed afterwards: test sequences 0048..0050 with 5 objects each,
480 x 640 colour and depth PNGs, synthetic weights, statistics and meshes per class.  Rates: frames/s counts each sequence frame
once; objects x frames/s counts each tracked object in each frame.
"""
import argparse, importlib, json, os, subprocess, sys, tempfile, time
from concurrent.futures import ThreadPoolExecutor
import cv2
import numpy as np
import torch
import yaml
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
PKG = 'iros20-6d-pose-tracking_b200'
SEQS = {48: (1, 2, 3, 4, 5), 49: (2, 3, 4, 5, 6), 50: (1, 3, 5, 6, 7)}


def smooth(rng, shape, lo, hi, dtype):
    """A frame with some structure (a blurred random field plus noise), so the PNGs compress like camera images, not like noise."""
    small = rng.uniform(lo, hi, (shape[0] // 16, shape[1] // 16) + shape[2:])
    img = cv2.resize(small, (shape[1], shape[0]), interpolation=cv2.INTER_CUBIC) + rng.normal(0, (hi - lo) * 0.02, shape)
    return np.clip(img, lo, hi).astype(dtype)


def write_tree(tmp, frames, synth, seqs=SEQS):
    """The data set of {sequence id: class ids} `seqs` under tmp -> (ycb dir, path templates, class ids)."""
    mio = importlib.import_module(PKG + '.mesh_io')
    rng = np.random.default_rng(0)
    ycb, cfg = os.path.join(tmp, 'ycb'), os.path.join(tmp, 'cfg')
    classes = sorted(set(c for cls in seqs.values() for c in cls))
    K = synth.CAMERA_K
    cam = {'focalX': float(K[0, 0]), 'focalY': float(K[1, 1]), 'centerX': float(K[0, 2]), 'centerY': float(K[1, 2]), 'height': 480, 'width': 640}
    mean, std = synth.default_mean_std()
    for c in classes:
        d = os.path.join(cfg, 'c%d' % c)
        os.makedirs(os.path.join(d, 'train'))
        yaml.safe_dump({'resolution': 176, 'object_width': 150.0 + 10 * c, 'boundingbox': 10, 'camera': cam}, open(os.path.join(d, 'dataset_info.yml'), 'w'))
        np.save(os.path.join(d, 'mean.npy'), mean + c); np.save(os.path.join(d, 'std.npy'), std)
        torch.save({'epoch': 1, 'state_dict': synth.make_state_dict(c), 'best_prec': 0.0}, os.path.join(d, 'model_best_val.pth.tar'))
        mio.save_ply_mesh(os.path.join(d, 'textured.ply'), synth.mesh(3, seed=c))
    for k in range(1, 22):
        os.makedirs(os.path.join(ycb, 'CADmodels', '%03d_obj' % k))
    for seq, cls in seqs.items():
        base = os.path.join(ycb, 'data_organized', '%04d' % seq)
        for sub in ['color', 'depth_filled'] + ['pose_gt/%d' % c for c in cls]:
            os.makedirs(os.path.join(base, sub))
        for i in range(frames):
            cv2.imwrite(os.path.join(base, 'color', '%06d-color.png' % (i + 1)), smooth(rng, (480, 640, 3), 0, 255, np.uint8))
            cv2.imwrite(os.path.join(base, 'depth_filled', '%06d-depth.png' % (i + 1)), smooth(rng, (480, 640), 400, 1500, np.uint16))
        for c in cls:
            p = synth.raw_poses(1, seed=10 * seq + c)[0]
            for i in range(frames):
                q = p.copy(); q[:3, 3] += 0.001 * i
                np.savetxt(os.path.join(base, 'pose_gt', str(c), '%06d.txt' % (i + 1)), q)
    templates = {'train_data_path': os.path.join(cfg, 'c{class_id}', 'train'), 'mean_std_path': os.path.join(cfg, 'c{class_id}'),
                 'ckpt_dir': os.path.join(cfg, 'c{class_id}', 'model_best_val.pth.tar'),
                 'model_path': os.path.join(cfg, 'c{class_id}', 'textured.ply')}
    return ycb, templates, classes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=100, help='frames per sequence')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--precision', default='bf16x3')
    ap.add_argument('--video', action='store_true', help='time the result videos: device drawing against host drawing')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    pkg = importlib.import_module(PKG)
    pr = importlib.import_module(PKG + '.predict')
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    with tempfile.TemporaryDirectory() as tmp:
        ycb, templates, classes = write_tree(tmp, args.frames, pkg.synth)
        seq_frames = len(SEQS) * args.frames
        obj_frames = sum(len(cls) for cls in SEQS.values()) * args.frames

        def one_pass(r):
            pr.getResultsYcbAll(ycb, classes, templates, os.path.join(tmp, 'all%d' % r), precision=args.precision)

        def per_class(r):
            for k in pr.ycb_all_classes(ycb, classes, templates, args.precision):
                pr.getResultsYcb(ycb, k['class_id'], k['dataset_info'], k['mean'], k['std'], k['ckpt_dir'], k['model_path'],
                                 os.path.join(tmp, 'pc%d' % r, k['name']), precision=args.precision, max_batch=1)

        def one_pass_video(r):
            pr.getResultsYcbAll(ycb, classes, templates, os.path.join(tmp, 'vid%d' % r), precision=args.precision, video=True)

        points, frames_rgb = {}, {}
        if args.video:
            sys.path.insert(0, os.path.join(ROOT, 'oracle'))
            import overlay_oracle as OV
            points = {c: pr.PointCloud(pr.load_vertices(templates['model_path'].format(class_id=c))).voxel_down_sample(voxel_size=0.005).points
                      for c in classes}
            frames_rgb = {seq: [pr.read_rgb(os.path.join(ycb, 'data_organized', '%04d' % seq, 'color', '%06d-color.png' % (i + 1)))
                                for i in range(args.frames)] for seq in SEQS}

        def one_pass_host_video(r):
            out = os.path.join(tmp, 'host%d' % r)
            res = pr.getResultsYcbAll(ycb, classes, templates, out, precision=args.precision)
            names = pr.ycb_class_names(ycb)
            jobs = []
            with ThreadPoolExecutor(max_workers=1) as writer:
                for seq, cls in SEQS.items():
                    vids = [cv2.VideoWriter(os.path.join(pr.ycb_all_res_dir(out, names[c - 1]), 'seq%d.mp4' % seq),
                                            cv2.VideoWriter_fourcc(*'mp4v'), 30, (320, 240)) for c in cls]
                    for i in range(1, args.frames):
                        drawn = [OV.draw_track(frames_rgb[seq][i], synth_K, res[c][seq][i], points[c], 'frame:%d' % (i + 1), 'under')
                                 for c in cls]
                        jobs.append(writer.submit(lambda d=drawn, v=vids: [w.write(f) for w, f in zip(v, d)]))
                    jobs.append(writer.submit(lambda v=vids: [w.release() for w in v]))
            for j in jobs:
                j.result()

        synth_K = pkg.synth.CAMERA_K
        legs = ((('one_pass', one_pass), ('one_pass_video', one_pass_video), ('one_pass_host_video', one_pass_host_video)) if args.video
                else (('one_pass', one_pass), ('per_class', per_class)))
        times = {name: [] for name, _ in legs}
        for r in range(args.rounds + 1):                             # round 0 warms every leg up and is not counted
            for name, fn in legs:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn(r)
                torch.cuda.synchronize()
                if r > 0:
                    times[name].append(time.perf_counter() - t0)
    out = {'gpu': gpu, 'torch_device': torch.cuda.get_device_name(0), 'precision': args.precision, 'sequences': len(SEQS),
           'objects_per_sequence': [len(c) for c in SEQS.values()], 'frames_per_sequence': args.frames, 'rounds': args.rounds}
    if points:
        out['model_points'] = {c: len(p) for c, p in points.items()}
    for name, ts in times.items():
        out[name] = {'seconds': [round(t, 3) for t in ts],
                     'frames_per_s': [round(seq_frames / t, 1) for t in ts],
                     'object_frames_per_s': [round(obj_frames / t, 1) for t in ts]}
        print('%-19s frames/s %s (%.1f-%.1f)   objects x frames/s %s' % (name, out[name]['frames_per_s'], min(out[name]['frames_per_s']),
                                                                         max(out[name]['frames_per_s']), out[name]['object_frames_per_s']))
    print('card (name, power limit, max SM clock): %s' % gpu)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
