"""YCBInEOAT evaluation throughput, two comparisons on one seeded synthetic data set in the YCBInEOAT layout:

  tracking  predict.getResultsYcbInEOAT (every video in one pass: one Engine, each object's weights loaded once, frames decoded
            --decode_ahead ahead by a thread pool) against the loop it replaces, one predictSequenceYcbInEOAT run per video (a new
            Tracker per run, each frame decoded on the calling thread before its step).
  scoring   the eval_ycbineoat drop-in (one add_adi_sets launch, one vocap_sets call per metric) against its CPU restatement
            (oracle/ycbineoat_oracle.py: Utils.add / Utils.adi with scipy's cKDTree per pose, as the reference scores).

Each leg is timed whole (set-up, weight and mesh upload, decoding, tracking, writing or reading the pose files) and the legs of
a comparison alternate `--rounds` times in one process after one warm-up round; the card's name and power limit are read in the
same run.

    python scripts/ycbineoat_all_throughput.py [--frames 100] [--rounds 3] [--decode_ahead 4] [--precision bf16x3]

The data set is written to a temporary directory and removed afterwards: 5 videos of 3 objects (two videos of the bleach bottle,
two of the sugar box), 480 x 640 colour and depth PNGs, synthetic weights, statistics, meshes and model points per object.
"""
import argparse, contextlib, importlib, io, json, os, subprocess, sys, tempfile, time
import cv2
import numpy as np
import torch
import yaml
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'oracle'))
PKG = 'iros20-6d-pose-tracking_b200'
VIDEOS = {'bleach0': 'bleach', 'bleach_hard_00_03': 'bleach', 'sugar_box1': 'sugar', 'sugar_box_yalehand0': 'sugar',
          'cracker_box_reorient': 'cracker'}
CAD = {'cracker': '003_cracker_box', 'sugar': '004_sugar_box', 'bleach': '021_bleach_cleanser'}


def smooth(rng, shape, lo, hi, dtype):
    """A frame with some structure (a blurred random field plus noise), so the PNGs compress like camera images, not like noise."""
    small = rng.uniform(lo, hi, (shape[0] // 16, shape[1] // 16) + shape[2:])
    img = cv2.resize(small, (shape[1], shape[0]), interpolation=cv2.INTER_CUBIC) + rng.normal(0, (hi - lo) * 0.02, shape)
    return np.clip(img, lo, hi).astype(dtype)


def write_tree(tmp, frames, synth, videos=VIDEOS):
    """The data set of {video folder: object} `videos` under tmp -> path templates."""
    mio = importlib.import_module(PKG + '.mesh_io')
    rng = np.random.default_rng(0)
    K = synth.CAMERA_K
    cam = {'focalX': float(K[0, 0]), 'focalY': float(K[1, 1]), 'centerX': float(K[0, 2]), 'centerY': float(K[1, 2]), 'height': 480, 'width': 640}
    mean, std = synth.default_mean_std()
    for j, obj in enumerate(CAD):
        d = os.path.join(tmp, 'cfg', obj)
        os.makedirs(os.path.join(d, 'train'))
        yaml.safe_dump({'resolution': 176, 'object_width': 160.0 + 20 * j, 'boundingbox': 10, 'camera': cam}, open(os.path.join(d, 'dataset_info.yml'), 'w'))
        np.save(os.path.join(d, 'mean.npy'), mean + j); np.save(os.path.join(d, 'std.npy'), std)
        torch.save({'epoch': 1, 'state_dict': synth.make_state_dict(j + 1), 'best_prec': 0.0}, os.path.join(d, 'model_best_val.pth.tar'))
        mio.save_ply_mesh(os.path.join(d, 'textured.ply'), synth.mesh(3, seed=j + 1))
        os.makedirs(os.path.join(tmp, 'ycb', 'CADmodels', CAD[obj]))
        np.savetxt(os.path.join(tmp, 'ycb', 'CADmodels', CAD[obj], 'points.xyz'), synth.mesh(4, seed=j + 1)['pos'].astype(np.float64))
    for v_i, v in enumerate(videos):
        base = os.path.join(tmp, 'data', v)
        for sub in ('rgb', 'depth_filled', 'annotated_poses'):
            os.makedirs(os.path.join(base, sub))
        p = synth.raw_poses(1, seed=10 + v_i)[0]
        for i in range(frames):
            cv2.imwrite(os.path.join(base, 'rgb', '%07d.png' % i), smooth(rng, (480, 640, 3), 0, 255, np.uint8))
            cv2.imwrite(os.path.join(base, 'depth_filled', '%07d.png' % i), smooth(rng, (480, 640), 400, 1500, np.uint16))
            q = p.copy(); q[:3, 3] += 0.001 * i
            np.savetxt(os.path.join(base, 'annotated_poses', '%07d.txt' % i), q)
    templates = {'train_data_path': os.path.join(tmp, 'cfg', '{object}', 'train'), 'mean_std_path': os.path.join(tmp, 'cfg', '{object}'),
                 'ckpt_dir': os.path.join(tmp, 'cfg', '{object}', 'model_best_val.pth.tar'),
                 'model_path': os.path.join(tmp, 'cfg', '{object}', 'textured.ply')}
    return templates


def alternate(legs, rounds):
    """{name: [seconds per round]}: the legs run in turn, round 0 warms them up and is not counted."""
    times = {name: [] for name, _ in legs}
    for r in range(rounds + 1):
        for name, fn in legs:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            with contextlib.redirect_stdout(io.StringIO()):
                fn(r)
            torch.cuda.synchronize()
            if r > 0:
                times[name].append(time.perf_counter() - t0)
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=100, help='frames per video')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--decode_ahead', type=int, default=4)
    ap.add_argument('--precision', default='bf16x3')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    pkg = importlib.import_module(PKG)
    pr = importlib.import_module(PKG + '.predict')
    ev = importlib.import_module(PKG + '.eval_ycbineoat')
    import ycbineoat_oracle as YO
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    with tempfile.TemporaryDirectory() as tmp:
        templates = write_tree(tmp, args.frames, pkg.synth)
        data, ycb = os.path.join(tmp, 'data'), os.path.join(tmp, 'ycb')
        frames = len(VIDEOS) * args.frames

        def one_pass(r):
            pr.getResultsYcbInEOAT(data, templates, os.path.join(tmp, 'all%d' % r), precision=args.precision, decode_ahead=args.decode_ahead)

        def per_video(r):
            objs = pr.ycbineoat_objects(sorted(set(VIDEOS.values())), templates, precision=args.precision)
            for v, o in VIDEOS.items():
                k = objs[o]
                pr.predictSequenceYcbInEOAT(os.path.join(data, v), k['dataset_info'], k['mean'], k['std'], k['ckpt_dir'], k['model_path'],
                                            os.path.join(tmp, 'pv%d' % r, v), precision=args.precision, max_batch=1)

        track = alternate([('one_pass', one_pass), ('per_video', per_video)], args.rounds)
        res = argparse.Namespace(res_dir=os.path.join(tmp, 'all0') + '/', YCBInEOAT_dir=data, ycb_dir=ycb)
        score = alternate([('drop_in', lambda r: ev.eval_all(res)), ('cpu_restatement', lambda r: YO.eval_all(res.res_dir, data, ycb))], args.rounds)
        with contextlib.redirect_stdout(io.StringIO()):
            got = ev.eval_all(res)
        want = YO.eval_all(res.res_dir, data, ycb)
    out = {'gpu': gpu, 'torch_device': torch.cuda.get_device_name(0), 'precision': args.precision, 'videos': len(VIDEOS),
           'objects': len(CAD), 'frames_per_video': args.frames, 'decode_ahead': args.decode_ahead, 'rounds': args.rounds,
           'model_points': int(pkg.synth.mesh(4, seed=1)['pos'].shape[0]),
           'auc_drop_in_vs_cpu': [got[1], want[2], got[2], want[3]]}
    for name, ts in list(track.items()) + list(score.items()):
        out[name] = {'seconds': [round(t, 3) for t in ts], 'frames_per_s': [round(frames / t, 1) for t in ts]}
        print('%-16s frames/s %s' % (name, out[name]['frames_per_s']))
    print('decode ahead: %d frames; card (name, power limit, max SM clock): %s' % (args.decode_ahead, gpu))
    print(json.dumps(out))


if __name__ == '__main__':
    main()
