"""Precision sweep throughput: one pass of a one-pass driver over several precision modes (every frame decoded once, one tracking
step per mode) against one single-mode run per mode, on the seeded synthetic data sets of scripts/ycbineoat_all_throughput.py
(5 videos of 3 objects) and scripts/ycb_all_throughput.py (3 test sequences of 5 objects).

    python scripts/precision_sweep_throughput.py [--frames 60] [--rounds 2] [--ycbineoat_modes bf16x3,bf16,fp16,fp8]
                                                 [--ycbv_modes bf16x3,bf16,fp8] [--data ycbineoat,ycbv]

For each data set the legs (the sweep, then each mode alone) run in turn `--rounds` times in one process after one warm-up round,
each call timed whole (engine set-up, weight and mesh upload, decoding, tracking, writing the pose files).  frames/s counts each
video or sequence frame once, whatever the number of modes.  Each call also reports the host seconds spent in np.savetxt (the pose
files, one set per mode) and an upper bound on its tracking steps' device time (Split).  The card's name and power limit are read
in the same run; nothing is changed on the device.  The data sets are written to a temporary directory and removed afterwards.
"""
import argparse, importlib.util, json, os, subprocess, sys, tempfile, time
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
PKG = 'iros20-6d-pose-tracking_b200'


def script(name):
    """A sibling script as a module: its write_tree builds the synthetic data set."""
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, 'scripts', name + '.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class Split:
    """Where a leg's time goes: host seconds inside np.savetxt (the pose files), and the sum over its tracking steps of the CUDA
    event time from before a step's enqueue to its end -- an upper bound on the steps' device time (it also counts any stretch in
    which the stream waits for the host to enqueue)."""
    def __init__(self, Engine):
        self.Engine, self.write_s, self.events = Engine, 0.0, []

    def __enter__(self):
        self.track, self.savetxt = self.Engine.track_render, np.savetxt
        track, savetxt, split = self.track, self.savetxt, self

        def timed_track(eng, *a, **kw):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = track(eng, *a, **kw)
            e1.record()
            split.events.append((e0, e1))
            return out

        def timed_savetxt(*a, **kw):
            t0 = time.perf_counter()
            savetxt(*a, **kw)
            split.write_s += time.perf_counter() - t0
        self.Engine.track_render, np.savetxt = timed_track, timed_savetxt
        return self

    def __exit__(self, *exc):
        self.Engine.track_render, np.savetxt = self.track, self.savetxt
        torch.cuda.synchronize()
        self.step_s = sum(a.elapsed_time(b) for a, b in self.events) / 1000


def alternate(legs, rounds, Engine):
    """{name: [(seconds, savetxt seconds, step seconds) per round]}: the legs run in turn, round 0 warms them up and is not
    counted."""
    times = {name: [] for name, _ in legs}
    for r in range(rounds + 1):
        for name, fn in legs:
            torch.cuda.synchronize()
            with Split(Engine) as split:
                t0 = time.perf_counter()
                fn(r)
                torch.cuda.synchronize()
                t = time.perf_counter() - t0
            if r > 0:
                times[name].append((t, split.write_s, split.step_s))
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=60, help='frames per video / sequence')
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--ycbineoat_modes', default='bf16x3,bf16,fp16,fp8')
    ap.add_argument('--ycbv_modes', default='bf16x3,bf16,fp8')
    ap.add_argument('--data', default='ycbineoat,ycbv')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    pkg = importlib.import_module(PKG)
    pr = importlib.import_module(PKG + '.predict')
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    out = {'gpu': gpu, 'torch_device': torch.cuda.get_device_name(0), 'frames': args.frames, 'rounds': args.rounds}
    for data in args.data.split(','):
        with tempfile.TemporaryDirectory() as tmp:
            if data == 'ycbineoat':
                s = script('ycbineoat_all_throughput')
                templates = s.write_tree(tmp, args.frames, pkg.synth)
                modes = args.ycbineoat_modes.split(',')
                frames = len(s.VIDEOS) * args.frames
                run = lambda precision, dest: pr.getResultsYcbInEOAT(os.path.join(tmp, 'data'), templates, dest, precision=precision)
            elif data == 'ycbv':
                s = script('ycb_all_throughput')
                ycb, templates, classes = s.write_tree(tmp, args.frames, pkg.synth)
                modes = args.ycbv_modes.split(',')
                frames = len(s.SEQS) * args.frames
                run = lambda precision, dest: pr.getResultsYcbAll(ycb, classes, templates, dest, precision=precision)
            else:
                raise SystemExit('--data: ycbineoat and / or ycbv, not %r' % data)
            legs = [('sweep', lambda r: run(modes, os.path.join(tmp, 'sweep%d' % r)))]
            legs += [(m, lambda r, m=m: run(m, os.path.join(tmp, '%s%d' % (m, r)))) for m in modes]
            times = alternate(legs, args.rounds, pr.Engine)
        res = out[data] = {'modes': modes, 'frames_per_round': frames}
        for name, ts in times.items():
            res[name] = {'seconds': [round(t, 3) for t, _, _ in ts], 'frames_per_s': [round(frames / t, 1) for t, _, _ in ts],
                         'savetxt_seconds': [round(w, 3) for _, w, _ in ts], 'step_seconds': [round(s, 3) for _, _, s in ts]}
            print('%-9s %-7s frames/s %s   seconds %s, in np.savetxt %s, steps (device, upper bound) %s'
                  % (data, name, res[name]['frames_per_s'], res[name]['seconds'], res[name]['savetxt_seconds'], res[name]['step_seconds']))
        single = sum(min(t for t, _, _ in times[m]) for m in modes)
        print('%-9s sweep of %d modes: best %.2f s, against %.2f s for the best single-mode runs of all of them in a row'
              % (data, len(modes), min(t for t, _, _ in times['sweep']), single))
    print('card (name, power limit, max SM clock): %s' % gpu)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
