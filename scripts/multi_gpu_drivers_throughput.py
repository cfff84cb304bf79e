"""The one-pass drivers on several GPUs: predict.getResultsYcbAll and getResultsYcbInEOAT with gpus = 1, 2, 4, 8 (those of them
up to the number of visible GPUs), the counts alternating `--rounds` times in one process after one warm-up round, each call timed
whole (process start, engine set-up, weight and mesh upload, decoding, tracking, writing the pose files).  The card's name and
power limit, the GPU count and the host CPU count are read in the same run, and every tree a multi-GPU call writes is checked,
file for file and byte for byte, against the tree of the 1-GPU call of the same round.

    python scripts/multi_gpu_drivers_throughput.py [--frames 60] [--rounds 2] [--precision bf16x3]

The data sets are those of scripts/ycb_all_throughput.py and scripts/ycbineoat_all_throughput.py with 8 sequences each, so that
each of 8 ranks has work: YCB-Video test sequences 0048..0055 with 5 objects each, 8 YCBInEOAT videos of 3 objects; 480 x 640
colour and depth PNGs, seeded, in a temporary directory removed afterwards.  Rates count each sequence frame once.
"""
import argparse, contextlib, importlib, io, json, os, subprocess, sys, tempfile, time
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'scripts'))
PKG = 'iros20-6d-pose-tracking_b200'
import ycb_all_throughput as YA            # noqa: E402
import ycbineoat_all_throughput as YE      # noqa: E402

SEQS = {48: (1, 2, 3, 4, 5), 49: (2, 3, 4, 5, 6), 50: (1, 3, 5, 6, 7), 51: (1, 2, 4, 6, 7), 52: (2, 3, 5, 6, 7),
        53: (1, 2, 3, 6, 7), 54: (3, 4, 5, 6, 7), 55: (1, 2, 4, 5, 7)}
VIDEOS = {'bleach0': 'bleach', 'bleach_hard_00_03': 'bleach', 'bleach_hard_00_03_chaitanya': 'bleach', 'cracker_box_reorient': 'cracker',
          'cracker_box_yalehand0': 'cracker', 'sugar_box1': 'sugar', 'sugar_box_yalehand0': 'sugar', 'sugar_box_hand1': 'sugar'}


def tree(root):
    out = {}
    for d, _, fs in os.walk(root):
        for f in fs:
            with open(os.path.join(d, f), 'rb') as x:
                out[os.path.relpath(os.path.join(d, f), root)] = x.read()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=60, help='frames per sequence or video')
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--precision', default='bf16x3')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    pkg = importlib.import_module(PKG)
    pr = importlib.import_module(PKG + '.predict')
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    visible = torch.cuda.device_count()
    counts = [g for g in (1, 2, 4, 8) if g <= visible] + ([visible] if visible not in (1, 2, 4, 8) and visible > 1 else [])
    out = {'gpu': gpu, 'gpus_visible': visible, 'host_cpus': os.cpu_count(), 'precision': args.precision,
           'frames_per_sequence': args.frames, 'rounds': args.rounds, 'sequences': len(SEQS), 'videos': len(VIDEOS)}
    with tempfile.TemporaryDirectory() as tmp:
        ycb, ycb_tpl, classes = YA.write_tree(os.path.join(tmp, 'ycbv'), args.frames, pkg.synth, SEQS)
        eoat = os.path.join(tmp, 'eoat')
        eoat_tpl = YE.write_tree(eoat, args.frames, pkg.synth, VIDEOS)
        drivers = {
            'ycbv_all': (len(SEQS) * (args.frames - 1),                        # YCB-Video tracks from the second frame
                         lambda g, o: pr.getResultsYcbAll(ycb, classes, ycb_tpl, o, precision=args.precision, gpus=g)),
            'ycbineoat_all': (len(VIDEOS) * args.frames,
                              lambda g, o: pr.getResultsYcbInEOAT(os.path.join(eoat, 'data'), eoat_tpl, o, precision=args.precision, gpus=g))}
        for name, (frames, run) in drivers.items():
            times = {g: [] for g in counts}
            same = True
            for r in range(args.rounds + 1):                            # round 0 warms every count up and is not counted
                for g in counts:
                    o = os.path.join(tmp, 'out', '%s_r%d_g%d' % (name, r, g))
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    with contextlib.redirect_stdout(io.StringIO()):
                        run(g, o)
                    torch.cuda.synchronize()
                    if r > 0:
                        times[g].append(time.perf_counter() - t0)
                one = tree(os.path.join(tmp, 'out', '%s_r%d_g1' % (name, r)))
                for g in counts[1:]:
                    same = same and tree(os.path.join(tmp, 'out', '%s_r%d_g%d' % (name, r, g))) == one
            base = min(times[1])
            out[name] = {'frames': frames, 'trees_equal_to_1_gpu': same,
                         'per_gpus': {g: {'seconds': [round(t, 3) for t in ts], 'frames_per_s': [round(frames / t, 1) for t in ts],
                                          'speedup_best_vs_best_1_gpu': round(base / min(ts), 2)} for g, ts in times.items()}}
            for g, row in out[name]['per_gpus'].items():
                print('%-14s gpus=%d  frames/s %s  speed-up %.2fx' % (name, g, row['frames_per_s'], row['speedup_best_vs_best_1_gpu']))
            print('%-14s every multi-GPU tree equals the 1-GPU tree: %s' % (name, same))
    print('card (name, power limit, max SM clock): %s; %d GPUs visible, %d host CPUs' % (gpu, visible, os.cpu_count()))
    print(json.dumps(out))


if __name__ == '__main__':
    main()
