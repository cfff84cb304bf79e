"""Validation on perturbed YCB-Video key frames, file route against one pass, on a synthetic YCB-Video layout:

  * file route: `produce_train_pair_data --mode ycbv` (produce_ycbv: PNG / npz pair files), then problems.evaluate on each
    class's folder;
  * one pass: problems.validate_ycbv, the same key-frame loop with each class's kept pairs appended to device queues and scored
    there.

The layout is built from seeds in a temporary directory: `--frames` 480 x 640 key frames, 5 classes with 20,480-face meshes
(synth.mesh level 5), each labelled in the seg image by a box around its projected centre, and one synthetic checkpoint per
class.  The two routes alternate `--rounds` times in one process, each in a fresh output folder; the script checks that they
give the same losses and prints pairs/s and key frames/s as JSON (also to `--out`), with the card's name and power limit read in
the same run.

    python scripts/perturbed_validate_throughput.py [--frames 200] [--num_sample 10] [--rounds 2] [--precision bf16x3] [--out FILE]
"""
import argparse, importlib, json, os, shutil, subprocess, sys, tempfile, time
from concurrent.futures import ThreadPoolExecutor
import cv2
import numpy as np
import torch
import yaml
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
PKG = 'iros20-6d-pose-tracking_b200'
H, W = 480, 640
CLASSES = (1, 2, 3, 4, 5)


def build_layout(root, synth, mesh_io, n_frames, seed=0):
    """<root>/ycb (data_organized/0048, image_sets/keyframe.txt, CADmodels/) and <root>/cfg/c<id> -> the four path templates."""
    rng = np.random.default_rng(seed)
    K = synth.CAMERA_K
    cam = {'focalX': float(K[0, 0]), 'focalY': float(K[1, 1]), 'centerX': float(K[0, 2]), 'centerY': float(K[1, 2]), 'height': H, 'width': W}
    mean, std = synth.default_mean_std()
    for c in CLASSES:
        d = os.path.join(root, 'cfg', 'c%d' % c)
        os.makedirs(os.path.join(d, 'train'))
        info = {'resolution': 176, 'object_width': 120.0, 'boundingbox': 10, 'max_translation': 0.02, 'max_rotation': 15.0, 'camera': cam}
        with open(os.path.join(d, 'dataset_info.yml'), 'w') as f:
            yaml.safe_dump(info, f)
        mesh_io.save_ply_mesh(os.path.join(d, 'textured.ply'), synth.mesh(5, seed=c))
        torch.save({'state_dict': synth.make_state_dict(c)}, os.path.join(d, 'model_best_val.pth.tar'))
        np.save(os.path.join(d, 'mean.npy'), mean); np.save(os.path.join(d, 'std.npy'), std)
    for c in range(1, 6):
        os.makedirs(os.path.join(root, 'ycb', 'CADmodels', '%03d_obj' % c))
    base = os.path.join(root, 'ycb', 'data_organized', '0048')
    for sub in ['color', 'depth_filled', 'seg'] + ['pose_gt/%d' % c for c in CLASSES]:
        os.makedirs(os.path.join(base, sub))
    centres = {c: np.array([-0.2 + 0.1 * k, 0.08 * (-1) ** k, 0.8]) for k, c in enumerate(CLASSES)}

    def frame(i):
        rgb, depth = synth.raw_frame(1000 + i, H, W)
        seg = np.zeros((H, W), np.uint8)
        for c in CLASSES:
            B = synth.raw_poses(1, seed=100 * i + c)[0]
            B[:3, 3] = centres[c] + np.random.default_rng(100 * i + c).normal(0, 0.005, 3)
            u = int(K[0, 0] * B[0, 3] / B[2, 3] + K[0, 2]); v = int(K[1, 1] * B[1, 3] / B[2, 3] + K[1, 2])
            seg[max(0, v - 30):v + 30, max(0, u - 40):u + 40] = c
            np.savetxt(os.path.join(base, 'pose_gt', str(c), '%06d.txt' % (i + 1)), B)
        cv2.imwrite(os.path.join(base, 'color', '%06d-color.png' % (i + 1)), rgb[..., ::-1])
        cv2.imwrite(os.path.join(base, 'depth_filled', '%06d-depth.png' % (i + 1)), depth)
        cv2.imwrite(os.path.join(base, 'seg', '%06d-label.png' % (i + 1)), seg)

    with ThreadPoolExecutor(max_workers=min(16, os.cpu_count() or 4)) as pool:
        list(pool.map(frame, range(n_frames)))
    os.makedirs(os.path.join(root, 'ycb', 'image_sets'))
    with open(os.path.join(root, 'ycb', 'image_sets', 'keyframe.txt'), 'w') as f:
        f.write(''.join('0048/%06d\n' % (i + 1) for i in range(n_frames)))
    cfg = os.path.join(root, 'cfg', 'c{class_id}')
    return {'train_data_path': os.path.join(cfg, 'train'), 'model_path': os.path.join(cfg, 'textured.ply'),
            'ckpt_dir': os.path.join(cfg, 'model_best_val.pth.tar'), 'mean_std_path': cfg}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=200)
    ap.add_argument('--num_sample', type=int, default=10)
    ap.add_argument('--batch_size', type=int, default=200)
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--precision', default='bf16x3')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    pkg = importlib.import_module(PKG)
    PP = importlib.import_module(PKG + '.produce_train_pair_data'); P = importlib.import_module(PKG + '.problems')
    D = importlib.import_module(PKG + '.datasets'); E = importlib.import_module(PKG + '.engine')
    mesh_io = importlib.import_module(PKG + '.mesh_io')
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    with tempfile.TemporaryDirectory() as root:
        tpl = build_layout(root, pkg.synth, mesh_io, args.frames)
        ycb = os.path.join(root, 'ycb')

        def file_route():
            out = os.path.join(root, 'pairs')
            shutil.rmtree(out, ignore_errors=True)
            counts = PP.produce_ycbv(ycb, CLASSES, tpl, out, num_sample=args.num_sample, seed=0)
            eng = E.Engine(max_batch=args.batch_size)
            res = {}
            for c in CLASSES:
                d = tpl['mean_std_path'].format(class_id=c)
                info = yaml.safe_load(open(os.path.join(d, 'dataset_info.yml')))
                ds = D.TrackDataset(os.path.join(out, '%03d_obj' % c), 'val', np.load(os.path.join(d, 'mean.npy')),
                                    np.load(os.path.join(d, 'std.npy')), dataset_info=info, trans_normalizer=info['max_translation'],
                                    rot_normalizer=info['max_rotation'] * np.pi / 180)
                model = pkg.Se3TrackNet(engine=eng, weight_id=0)
                model.load_state_dict(torch.load(tpl['ckpt_dir'].format(class_id=c), map_location='cpu')['state_dict'])
                r = P.evaluate(model, ds, args.batch_size, precision=args.precision)
                res[c] = (counts[c], r['trans'], r['rot'])
            eng.close()
            return res

        def one_pass():
            r = P.validate_ycbv(ycb, CLASSES, tpl, num_sample=args.num_sample, seed=0, batch_size=args.batch_size,
                                max_batch=args.batch_size, precisions=[args.precision])
            return {c: (r[c][args.precision]['pairs'], r[c][args.precision]['trans'], r[c][args.precision]['rot']) for c in CLASSES}

        times = {'file_route': [], 'one_pass': []}
        results = {}
        for _ in range(args.rounds):
            for name, fn in (('file_route', file_route), ('one_pass', one_pass)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                results[name] = fn()
                torch.cuda.synchronize()
                times[name].append(time.perf_counter() - t0)
    pairs = sum(n for n, _, _ in results['one_pass'].values())
    out = dict(gpu=gpu, frames=args.frames, frame_hw=[H, W], classes=len(CLASSES), mesh_faces=20 * 4 ** 5, num_sample=args.num_sample,
               batch_size=args.batch_size, precision=args.precision, pairs=pairs,
               identical=results['file_route'] == results['one_pass'])
    for name, ts in times.items():
        out[name] = dict(seconds=[round(t, 3) for t in ts], pairs_per_s=[round(pairs / t, 1) for t in ts],
                         key_frames_per_s=[round(args.frames / t, 2) for t in ts])
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
