"""ICP alone on synthetic frames: a zero head (the network leaves every pose as it is), 8 tracks started 5-10 mm and 2-5 degrees
off the poses that drew the frame (oracle/icp_ref.py synthetic_scene, the pyrender-mode rasteriser's depth), M = 10 iterations in
one pyrender-mode step.  Prints the card's name and power limit read in the same run, then one JSON line per iteration with
every track's ADD (mm, on synth.model_points) and rotation error (degrees), and their mean and max.

    python scripts/icp_convergence.py [--seed 0]"""
import argparse, importlib, json, os, subprocess, sys
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import icp_ref  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--seed', type=int, default=0)
    args = ap.parse_args()
    print(subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip())
    pkg = importlib.import_module('iros20-6d-pose-tracking_b200')
    synth = pkg.synth
    mesh, gts, starts, D = icp_ref.synthetic_scene(synth, 8, seed=args.seed)
    e = pkg.Engine(max_batch=8)
    sd = synth.make_state_dict(2)
    for k in ('trans_out.0.weight', 'trans_out.0.bias', 'rot_out.0.weight', 'rot_out.0.bias'):
        sd[k] = torch.zeros_like(sd[k])
    mean, std = synth.default_mean_std()
    e.load_state_dict(sd, 0); e.set_mesh(mesh, 0); e.set_stats(mean, std, 0)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    slots = torch.empty(10, 8, 4, 4, dtype=torch.float64, device='cuda')
    e.track_render(dev(synth.raw_frame(3)[0]), dev(D), synth.CAMERA_K, dev(starts), torch.full((8,), 200.0, dtype=torch.float64, device='cuda'),
                   0.03, 5 * np.pi / 180, mode='pyrender', image_hw=D.shape, icp=10, out_icp_poses=slots)
    pts = synth.model_points()

    def err(p, g):
        add = np.linalg.norm(pts @ p[:3, :3].T + p[:3, 3] - pts @ g[:3, :3].T - g[:3, 3], axis=1).mean() * 1000
        return add, np.degrees(np.arccos(np.clip((np.trace(p[:3, :3].T @ g[:3, :3]) - 1) / 2, -1, 1)))
    poses = [starts] + list(slots.cpu().numpy())
    for m, P in enumerate(poses):
        ev = np.array([err(P[i], gts[i]) for i in range(8)])
        print(json.dumps({'iteration': m, 'n': 8, 'add_mm': np.round(ev[:, 0], 3).tolist(), 'rot_deg': np.round(ev[:, 1], 3).tolist(),
                          'add_mean': round(float(ev[:, 0].mean()), 3), 'add_max': round(float(ev[:, 0].max()), 3),
                          'rot_mean': round(float(ev[:, 1].mean()), 3), 'rot_max': round(float(ev[:, 1].max()), 3)}))
    e.close()


if __name__ == '__main__':
    main()
